// half_shim_test.cpp — 16-bit plans through include/dfft.hpp: MPIcuFFT_Slab<__half> (C2C, both directions) and
// MPIcuFFT_Pencil<__nv_bfloat16> (R2C / C2R) on one rank against the C ABI plans of DFFT_F16 / DFFT_BF16 on the same input,
// byte for byte (memcmp).  dfft.hpp includes no CUDA header: the prec<__half> / prec<__nv_bfloat16> specialisations exist
// because this file includes cuda_fp16.h / cuda_bf16.h first.
// Build (tests/test_gpu_half.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include half_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

static_assert(dfft_shim::prec<__half>::value == DFFT_F16 && dfft_shim::prec<__nv_bfloat16>::value == DFFT_BF16, "16-bit shim precisions");

// finite 16-bit values of both signs, magnitudes in [2^-3, 1): the same bits serve as FP16 and as BF16 numbers
static std::vector<uint16_t> values(size_t count, uint16_t exp_base) {
    std::vector<uint16_t> v(count);
    for (size_t i = 0; i < count; ++i) {
        const uint32_t h = uint32_t(i * 2654435761u) >> 7;
        v[i] = uint16_t((h & 1u) << 15) | uint16_t(exp_base + (h >> 1) % 0x0300u);
    }
    return v;
}

static bool same(const void* a, const void* b, size_t bytes, const char* what) {
    std::vector<unsigned char> ha(bytes), hb(bytes);
    cudaMemcpy(ha.data(), a, bytes, cudaMemcpyDeviceToHost);
    cudaMemcpy(hb.data(), b, bytes, cudaMemcpyDeviceToHost);
    if (std::memcmp(ha.data(), hb.data(), bytes) == 0) return true;
    std::printf("%s: the shim's output differs from the C ABI plan's\n", what);
    return false;
}

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    const size_t nx = 32, ny = 64, nz = 128, pts = nx * ny * nz, nzc = nz / 2 + 1, spec = nx * ny * nzc;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(nx, ny, nz);
    int rc = 0;
    void *in, *a, *b, *back_a, *back_b;
    if (cudaMalloc(&in, pts * 4) || cudaMalloc(&a, pts * 4) || cudaMalloc(&b, pts * 4) || cudaMalloc(&back_a, pts * 4) || cudaMalloc(&back_b, pts * 4))
        return 1;
    {   // FP16 C2C slab: 4-byte (re, im) pairs
        const std::vector<uint16_t> x = values(2 * pts, 0x3000);  // FP16 exponents 12..14
        cudaMemcpy(in, x.data(), pts * 4, cudaMemcpyHostToDevice);
        MPIcuFFT_Slab<__half> shim(cfg, comm, -1, DFFT_C2C);
        shim.initFFT(&gs, nullptr, true);
        dfft_plan_t plan;
        if (dfft_plan_create(comm, nullptr, DFFT_SLAB_ZY_THEN_X, DFFT_F16, DFFT_C2C, nx, ny, nz, 1, 1, 1, &plan) != DFFT_SUCCESS) return 1;
        if (dfft_get_domain_size(plan) != pts * 4) { std::printf("FP16 domain size %zu\n", dfft_get_domain_size(plan)); rc = 1; }
        shim.execC2C(a, in, DFFT_FORWARD);
        if (dfft_exec_c2c(plan, b, in, DFFT_FORWARD) != DFFT_SUCCESS) return 1;
        rc |= !same(a, b, pts * 4, "FP16 slab forward");
        shim.execC2C(back_a, a, DFFT_INVERSE);
        if (dfft_exec_c2c(plan, back_b, b, DFFT_INVERSE) != DFFT_SUCCESS) return 1;
        rc |= !same(back_a, back_b, pts * 4, "FP16 slab inverse");
        dfft_plan_destroy(plan);
    }
    {   // BF16 R2C / C2R pencil on a 1 x 1 grid: 2-byte reals, 4-byte complex pairs
        const std::vector<uint16_t> x = values(pts, 0x3E00);  // BF16 exponents 124..126
        cudaMemcpy(in, x.data(), pts * 2, cudaMemcpyHostToDevice);
        Pencil_Partition part(1, 1);
        MPIcuFFT_Pencil<__nv_bfloat16> shim(cfg, comm, -1, DFFT_R2C);
        shim.initFFT(&gs, &part, true);
        dfft_plan_t plan;
        if (dfft_plan_create(comm, nullptr, DFFT_PENCIL, DFFT_BF16, DFFT_R2C, nx, ny, nz, 1, 1, 1, &plan) != DFFT_SUCCESS) return 1;
        shim.execR2C(a, in);
        if (dfft_exec_r2c(plan, b, in) != DFFT_SUCCESS) return 1;
        rc |= !same(a, b, spec * 4, "BF16 pencil R2C");
        shim.execC2R(back_a, a);
        if (dfft_exec_c2r(plan, back_b, b) != DFFT_SUCCESS) return 1;
        rc |= !same(back_a, back_b, pts * 2, "BF16 pencil C2R");
        dfft_plan_destroy(plan);
    }
    cudaFree(in); cudaFree(a); cudaFree(b); cudaFree(back_a); cudaFree(back_b);
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
