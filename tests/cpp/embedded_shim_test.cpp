// embedded_shim_test.cpp — plans with strides through include/dfft.hpp's setStrides.
//   - one rank (MPIcuFFT_Slab<double>, C2C, 16 x 32 x 64): the caller's arrays have two ghost layers on every side; execC2C
//     both ways on the interiors is compared by memcmp with a plan without strides on dense arrays, and every ghost
//     element of both arrays must keep its value;
//   - the plan reports the strides (dfft_plan_get_strides), and strides set after the first exec are refused.
// Build (tests/test_gpu_embedded.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include
//        embedded_shim_test.cpp -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    const size_t nx = 16, ny = 32, nz = 64, h = 2, es = 16;
    const size_t ex = nx + 2 * h, ey = ny + 2 * h, ez = nz + 2 * h;  // the caller's arrays, interior at (h, h, h)
    const long long st[3] = {(long long)(ex * ey * ez), (long long)(ey * ez), (long long)ez};
    const size_t lead = (h * ey * ez + h * ez + h) * es, dense = nx * ny * nz * es, full = ex * ey * ez * es;
    bool ok = true;
    {
        GlobalSize gs(nx, ny, nz);
        MPIcuFFT_Slab<double> plan(cfg, comm, -1, DFFT_C2C);
        plan.initFFT(&gs, nullptr);
        plan.setStrides(st, st);
        long long gi[3], go[3];
        ok = ok && dfft_plan_get_strides(plan.handle(), gi, go) == DFFT_SUCCESS && std::memcmp(gi, st, sizeof st) == 0 &&
             std::memcmp(go, st, sizeof st) == 0;
        dfft_plan_t c = nullptr;
        dfft_config ccfg{};
        if (dfft_plan_create(comm, &ccfg, DFFT_SLAB_ZY_THEN_X, DFFT_F64, DFFT_C2C, nx, ny, nz, 1, 1, 1, &c) != DFFT_SUCCESS) return 1;
        std::vector<unsigned char> h_in(full), h_out(full, 0xAB), a(full), b(dense);
        for (size_t k = 0; k < full; ++k) h_in[k] = (unsigned char)((k * 2654435761u) >> 13);
        for (size_t k = 7; k < full; k += 8) h_in[k] = 0x3f;  // finite doubles
        void *x, *y, *xd, *yd;
        if (cudaMalloc(&x, full) || cudaMalloc(&y, full) || cudaMalloc(&xd, dense) || cudaMalloc(&yd, dense)) return 1;
        cudaMemcpy(x, h_in.data(), full, cudaMemcpyHostToDevice);
        cudaMemcpy(y, h_out.data(), full, cudaMemcpyHostToDevice);
        // the dense copy of the interior
        cudaMemcpy3DParms p{};
        p.srcPtr = make_cudaPitchedPtr(static_cast<char*>(x) + lead, ez * es, ez * es, ey);
        p.dstPtr = make_cudaPitchedPtr(xd, nz * es, nz * es, ny);
        p.extent = make_cudaExtent(nz * es, ny, nx);
        p.kind = cudaMemcpyDeviceToDevice;
        cudaMemcpy3D(&p);
        for (int direction : {DFFT_FORWARD, DFFT_INVERSE}) {
            plan.execC2C(static_cast<char*>(y) + lead, static_cast<char*>(x) + lead, direction);
            if (dfft_exec_c2c(c, yd, xd, direction) != DFFT_SUCCESS || cudaDeviceSynchronize() != cudaSuccess) { ok = false; break; }
            cudaMemcpy(a.data(), y, full, cudaMemcpyDeviceToHost);
            cudaMemcpy(b.data(), yd, dense, cudaMemcpyDeviceToHost);
            bool same = true, ghosts = true;
            for (size_t i = 0; i < ex; ++i)
                for (size_t j = 0; j < ey; ++j) {
                    const unsigned char* row = a.data() + (i * ey + j) * ez * es;
                    const bool inside = i >= h && i < h + nx && j >= h && j < h + ny;
                    for (size_t k = 0; k < ez * es; ++k) {
                        const bool in_row = inside && k >= h * es && k < (h + nz) * es;
                        if (in_row) same = same && row[k] == b[(((i - h) * ny + (j - h)) * nz) * es + (k - h * es)];
                        else ghosts = ghosts && row[k] == 0xAB;
                    }
                }
            std::vector<unsigned char> back(full);
            cudaMemcpy(back.data(), x, full, cudaMemcpyDeviceToHost);
            const bool input_kept = std::memcmp(back.data(), h_in.data(), full) == 0;
            std::printf("direction %d: interior %s, output ghosts %s, input array %s\n", direction, same ? "identical" : "DIFFERENT",
                        ghosts ? "kept" : "WRITTEN", input_kept ? "kept" : "CHANGED");
            ok = ok && same && ghosts && input_kept;
        }
        const bool refused = dfft_plan_set_strides(plan.handle(), st, nullptr) == DFFT_ERR_STATE;
        std::printf("strides after an exec: %s\n", refused ? "refused" : "ACCEPTED");
        ok = ok && refused;
        cudaFree(x); cudaFree(y); cudaFree(xd); cudaFree(yd);
        dfft_plan_destroy(c);
    }
    dfft_comm_destroy(comm);
    std::printf("%s\n", ok ? "PASSED" : "FAILED");
    return ok ? 0 : 1;
}
