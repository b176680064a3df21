// transform_axes_shim_test.cpp — kept axes through include/dfft.hpp: MPIcuFFT_Slab<double> (C2C) and
// MPIcuFFT_Pencil<float> (per-axis R2R) with setTransformAxes(false, true, true) after initFFT; execC2C / execR2R forward
// and inverse are compared by memcmp with the same plan made through the C ABI with dfft_plan_set_transform_axes, and
// dfft_plan_get_transform_axes must return the axes.
// Build (tests/test_gpu_transform_axes.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include
//        transform_axes_shim_test.cpp -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

// es: bytes per element of the buffers (complex for C2C, real for R2R); kinds == nullptr: a C2C plan
template <typename Plan>
static bool compare(dfft_comm_t comm, Plan& shim, int decomp, int prec, const int* kinds, size_t es, size_t nx, size_t ny, size_t nz) {
    const int axes[3] = {0, 1, 1};
    int got[3] = {1, 1, 1};
    if (dfft_plan_get_transform_axes(shim.handle(), got) != DFFT_SUCCESS || got[0] != 0 || got[1] != 1 || got[2] != 1) {
        std::printf("getTransformAxes mismatch\n");
        return false;
    }
    dfft_plan_t c = nullptr;
    dfft_config cfg{};
    cfg.comm_method = DFFT_PEER2PEER; cfg.comm_method2 = DFFT_PEER2PEER;
    const int rc0 = kinds ? dfft_plan_create_r2r(comm, &cfg, decomp, prec, kinds, nx, ny, nz, 1, 1, 1, 0, 1, &c)
                          : dfft_plan_create(comm, &cfg, decomp, prec, DFFT_C2C, nx, ny, nz, 1, 1, 1, &c);
    if (rc0 != DFFT_SUCCESS || dfft_plan_set_transform_axes(c, axes) != DFFT_SUCCESS) {
        std::printf("C ABI plan: %s\n", dfft_last_error_string());
        return false;
    }
    const size_t bytes = nx * ny * nz * es;
    std::vector<unsigned char> h(bytes), a(bytes), b(bytes);
    for (size_t k = 0; k < bytes; ++k) h[k] = (unsigned char)((k * 2654435761u) >> 13);
    if (prec == DFFT_F64)  // finite doubles: keep every exponent byte small
        for (size_t k = 7; k < bytes; k += 8) h[k] = 0x3f;
    else
        for (size_t k = 3; k < bytes; k += 4) h[k] = 0x3f;
    void *x, *y1, *y2;
    if (cudaMalloc(&x, bytes) || cudaMalloc(&y1, bytes) || cudaMalloc(&y2, bytes)) return false;
    cudaMemcpy(x, h.data(), bytes, cudaMemcpyHostToDevice);
    bool ok = true;
    for (int direction : {DFFT_FORWARD, DFFT_INVERSE}) {
        if (kinds) shim.execR2R(y1, x, direction);
        else shim.execC2C(y1, x, direction);
        const int rc = kinds ? dfft_exec_r2r(c, y2, x, direction) : dfft_exec_c2c(c, y2, x, direction);
        if (rc != DFFT_SUCCESS || cudaDeviceSynchronize() != cudaSuccess) { std::printf("exec failed\n"); ok = false; break; }
        cudaMemcpy(a.data(), y1, bytes, cudaMemcpyDeviceToHost);
        cudaMemcpy(b.data(), y2, bytes, cudaMemcpyDeviceToHost);
        const bool same = std::memcmp(a.data(), b.data(), bytes) == 0;
        const bool moved = std::memcmp(a.data(), h.data(), bytes) != 0;  // y and z were transformed
        std::printf("decomp %d prec %d %s direction %d: %s\n", decomp, prec, kinds ? "r2r" : "c2c", direction, same && moved ? "identical" : "DIFFERENT");
        ok = ok && same && moved;
    }
    // the setter refuses once a schedule exists
    if (dfft_plan_set_transform_axes(c, axes) != DFFT_ERR_STATE) { std::printf("no DFFT_ERR_STATE after an exec\n"); ok = false; }
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
        GlobalSize gs(32, 64, 128);
        MPIcuFFT_Slab<double> plan(cfg, comm, -1, DFFT_C2C);
        plan.initFFT(&gs, true);
        plan.setTransformAxes(false, true, true);
        ok = compare(comm, plan, DFFT_SLAB_ZY_THEN_X, DFFT_F64, nullptr, 16, 32, 64, 128) && ok;
    }
    {
        const int kinds[3] = {DFFT_DCT, DFFT_R2HC, DFFT_R2HC};
        GlobalSize gs(64, 32, 16);
        Pencil_Partition part(1, 1);
        MPIcuFFT_Pencil<float> plan(cfg, comm, -1, kinds);
        plan.initFFT(&gs, &part, true);
        plan.setTransformAxes(false, true, true);
        ok = compare(comm, plan, DFFT_PENCIL, DFFT_F32, kinds, 4, 64, 32, 16) && ok;
    }
    dfft_comm_destroy(comm);
    if (ok) std::printf("PASSED\n");
    return ok ? 0 : 1;
}
