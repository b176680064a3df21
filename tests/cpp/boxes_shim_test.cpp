// boxes_shim_test.cpp — box plans through include/dfft.hpp's initFFT(global_size, partition, in_boxes, out_boxes).
//   - geometry-only plans of 4 ranks (MPIcuFFT_Pencil<double>, 2 x 2): the getters report each rank's bricks;
//   - one rank (MPIcuFFT_Slab<double>, C2C): with the whole grid as its boxes the plan is the natural one, and execC2C both
//     ways is compared by memcmp with dfft_plan_create through the C ABI.
// Build (tests/test_gpu_boxes.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include
//        boxes_shim_test.cpp -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

static bool bricks() {
    // 2 x 2 x 1 bricks of 8 x 8 x 16 in, 1 x 2 x 2 of the output
    const size_t in[24] = {0, 0, 0, 4, 4, 16, 0, 4, 0, 4, 8, 16, 4, 0, 0, 8, 4, 16, 4, 4, 0, 8, 8, 16};
    const size_t out[24] = {0, 0, 0, 8, 4, 8, 0, 0, 8, 8, 4, 16, 0, 4, 0, 8, 8, 8, 0, 4, 8, 8, 8, 16};
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    bool ok = true;
    for (int r = 0; r < 4; ++r) {
        dfft_comm_t comm;
        if (dfft_comm_create_dry(r, 4, &comm) != DFFT_SUCCESS) return false;
        {
            GlobalSize gs(8, 8, 16);
            Pencil_Partition part(2, 2);
            MPIcuFFT_Pencil<double> plan(cfg, comm, -1, DFFT_C2C);
            plan.initFFT(&gs, &part, in, out);
            size_t is[3], io[3], os[3], oo[3];
            plan.getInSize(is); plan.getInStart(io); plan.getOutSize(os); plan.getOutStart(oo);
            for (int a = 0; a < 3; ++a) {
                ok = ok && io[a] == in[6 * r + a] && is[a] == in[6 * r + 3 + a] - in[6 * r + a];
                ok = ok && oo[a] == out[6 * r + a] && os[a] == out[6 * r + 3 + a] - out[6 * r + a];
            }
            std::printf("rank %d: in [%zu %zu %zu]+[%zu %zu %zu], out [%zu %zu %zu]+[%zu %zu %zu]\n", r, io[0], io[1], io[2], is[0], is[1], is[2], oo[0],
                        oo[1], oo[2], os[0], os[1], os[2]);
        }
        dfft_comm_destroy(comm);
    }
    return ok;
}

static bool one_rank() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return false;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    const size_t nx = 16, ny = 32, nz = 64, whole[6] = {0, 0, 0, nx, ny, nz};
    bool ok = true;
    {
        GlobalSize gs(nx, ny, nz);
        MPIcuFFT_Slab<double> plan(cfg, comm, -1, DFFT_C2C);
        plan.initFFT(&gs, nullptr, whole, whole);
        dfft_plan_t c = nullptr;
        dfft_config ccfg{};
        if (dfft_plan_create(comm, &ccfg, DFFT_SLAB_ZY_THEN_X, DFFT_F64, DFFT_C2C, nx, ny, nz, 1, 1, 1, &c) != DFFT_SUCCESS) return false;
        const size_t bytes = nx * ny * nz * 16;
        std::vector<unsigned char> h(bytes), a(bytes), b(bytes);
        for (size_t k = 0; k < bytes; ++k) h[k] = (unsigned char)((k * 2654435761u) >> 13);
        for (size_t k = 7; k < bytes; k += 8) h[k] = 0x3f;  // finite doubles
        void *x, *y1, *y2;
        if (cudaMalloc(&x, bytes) || cudaMalloc(&y1, bytes) || cudaMalloc(&y2, bytes)) return false;
        cudaMemcpy(x, h.data(), bytes, cudaMemcpyHostToDevice);
        for (int direction : {DFFT_FORWARD, DFFT_INVERSE}) {
            plan.execC2C(y1, x, direction);
            if (dfft_exec_c2c(c, y2, x, direction) != DFFT_SUCCESS || cudaDeviceSynchronize() != cudaSuccess) { ok = false; break; }
            cudaMemcpy(a.data(), y1, bytes, cudaMemcpyDeviceToHost);
            cudaMemcpy(b.data(), y2, bytes, cudaMemcpyDeviceToHost);
            const bool same = std::memcmp(a.data(), b.data(), bytes) == 0, moved = std::memcmp(a.data(), h.data(), bytes) != 0;
            std::printf("one rank, direction %d: %s\n", direction, same && moved ? "identical" : "DIFFERENT");
            ok = ok && same && moved;
        }
        cudaFree(x); cudaFree(y1); cudaFree(y2);
        dfft_plan_destroy(c);
    }
    dfft_comm_destroy(comm);
    return ok;
}

int main() {
    const bool ok = bricks() && one_rank();
    std::printf("%s\n", ok ? "PASSED" : "FAILED");
    return ok ? 0 : 1;
}
