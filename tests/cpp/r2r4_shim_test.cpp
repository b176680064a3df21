// r2r4_shim_test.cpp — per-axis plans with type-IV kinds (DFFT_DCT4 / DFFT_DST4) through include/dfft.hpp:
// MPIcuFFT_Slab<double> and MPIcuFFT_Pencil<float> constructed with kinds (x, y, z), initFFT (the pencil plan batched and in
// place), execR2R forward and inverse; every output is compared by memcmp with the output of the same plan made through the
// C ABI (dfft_plan_create_r2r), and dfft_plan_get_r2r_kinds must return the kinds.
// Build (tests/test_gpu_r2r4.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include r2r4_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

template <typename T, typename Plan>
static bool compare(dfft_comm_t comm, Plan& shim, int decomp, const int (&kinds)[3], size_t nx, size_t ny, size_t nz, size_t batch, bool inplace,
                    int d) {
    const size_t n = nx * ny * nz;
    int got[3] = {0, 0, 0};
    if (dfft_plan_get_r2r_kinds(shim.handle(), got) != DFFT_SUCCESS || got[0] != kinds[0] || got[1] != kinds[1] || got[2] != kinds[2]) {
        std::printf("getR2RKinds mismatch\n");
        return false;
    }
    dfft_plan_t c = nullptr;
    dfft_config cfg{};
    cfg.comm_method = DFFT_PEER2PEER; cfg.comm_method2 = DFFT_PEER2PEER;
    if (dfft_plan_create_r2r(comm, &cfg, decomp, sizeof(T) == 8 ? DFFT_F64 : DFFT_F32, kinds, nx, ny, nz, 1, 1, batch, inplace ? 1 : 0, 1, &c) !=
        DFFT_SUCCESS) {
        std::printf("dfft_plan_create_r2r: %s\n", dfft_last_error_string());
        return false;
    }
    // one field: the larger of the domain and the array; in place, fields are a domain apart
    const size_t field = inplace ? shim.getDomainSize() / sizeof(T) : n;
    const size_t elems = field * batch;
    std::vector<T> h(elems), a(elems), b(elems);
    for (size_t k = 0; k < elems; ++k) h[k] = T(double((k * 2654435761u) % 1000) / 999.0 - 0.5);
    void *x, *y1, *y2;
    if (cudaMalloc(&x, elems * sizeof(T)) || cudaMalloc(&y1, elems * sizeof(T)) || cudaMalloc(&y2, elems * sizeof(T))) return false;
    bool ok = true;
    for (int direction : {DFFT_FORWARD, DFFT_INVERSE}) {
        cudaMemcpy(inplace ? y1 : x, h.data(), elems * sizeof(T), cudaMemcpyHostToDevice);
        shim.execR2R(y1, inplace ? y1 : x, direction, d);
        cudaMemcpy(inplace ? y2 : x, h.data(), elems * sizeof(T), cudaMemcpyHostToDevice);
        const int rc = d == 3 ? dfft_exec_r2r(c, y2, inplace ? y2 : x, direction) : dfft_exec_r2r_partial(c, y2, inplace ? y2 : x, direction, d);
        if (rc != DFFT_SUCCESS || cudaDeviceSynchronize() != cudaSuccess) { std::printf("exec failed\n"); ok = false; break; }
        cudaMemcpy(a.data(), y1, elems * sizeof(T), cudaMemcpyDeviceToHost);
        cudaMemcpy(b.data(), y2, elems * sizeof(T), cudaMemcpyDeviceToHost);
        const bool same = std::memcmp(a.data(), b.data(), elems * sizeof(T)) == 0;
        double mag = 0;
        for (size_t k = 0; k < elems; ++k) mag += double(a[k]) * double(a[k]);
        std::printf("decomp %d kinds (%d, %d, %d) batch %zu inplace %d d %d direction %d: %s (|out|^2 %.3e)\n", decomp, kinds[0], kinds[1], kinds[2], batch,
                    int(inplace), d, direction, same ? "identical" : "DIFFERENT", mag);
        ok = ok && same && mag > 0;
    }
    cudaFree(x); cudaFree(y1); cudaFree(y2);
    dfft_plan_destroy(c);
    return ok;
}

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    bool ok = true;
    {
        const int kinds[3] = {DFFT_DCT4, DFFT_R2HC, DFFT_R2HC};  // a channel with different walls in x, periodic y and z
        GlobalSize gs(32, 64, 128);
        MPIcuFFT_Slab<double> plan(cfg, comm, -1, kinds);
        plan.initFFT(&gs, true);
        ok = compare<double>(comm, plan, DFFT_SLAB_ZY_THEN_X, kinds, 32, 64, 128, 1, false, 3) && ok;
    }
    {
        const int kinds[3] = {DFFT_DST4, DFFT_DCT1, DFFT_DCT4};
        GlobalSize gs(16, 33, 64);
        Pencil_Partition part(1, 1);
        MPIcuFFT_Pencil<float> plan(cfg, comm, -1, kinds);
        plan.initFFT(&gs, &part, true, 2, true);
        ok = compare<float>(comm, plan, DFFT_PENCIL, kinds, 16, 33, 64, 2, true, 3) && ok;
        ok = compare<float>(comm, plan, DFFT_PENCIL, kinds, 16, 33, 64, 2, true, 2) && ok;
    }
    dfft_comm_destroy(comm);
    if (ok) std::printf("PASSED\n");
    return ok ? 0 : 1;
}
