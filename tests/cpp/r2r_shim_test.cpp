// r2r_shim_test.cpp — a DCT round trip through MPIcuFFT_Slab<double> of include/dfft.hpp: execR2R forward (DCT-II), then
// inverse (DCT-III) with setScale(1, 1 / (8 N)), compared with the input; then the same for a DST plan, partial d = 1.
// Build (tests/test_gpu_r2r.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include r2r_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <vector>

#include "dfft.hpp"

static double round_trip(dfft_comm_t comm, int transform, int d) {
    const size_t nx = 64, ny = 32, nz = 128, n = nx * ny * nz;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(nx, ny, nz);
    MPIcuFFT_Slab<double> plan(cfg, comm, -1, transform);
    plan.initFFT(&gs, true);
    const double lens[3] = {double(nz), double(ny), double(nx)};
    double round = 1;
    for (int k = 0; k < d; ++k) round *= 2 * lens[k];
    plan.setScale(1.0, 1.0 / round);
    std::vector<double> h(n), back(n);
    for (size_t k = 0; k < n; ++k) h[k] = double((k * 2654435761u) % 1000) / 999.0 - 0.5;
    void *x, *spec, *y;
    if (cudaMalloc(&x, n * 8) || cudaMalloc(&spec, plan.getDomainSize()) || cudaMalloc(&y, n * 8)) return 1e9;
    cudaMemcpy(x, h.data(), n * 8, cudaMemcpyHostToDevice);
    plan.execR2R(spec, x, DFFT_FORWARD, d);
    plan.execR2R(y, spec, DFFT_INVERSE, d);
    cudaMemcpy(back.data(), y, n * 8, cudaMemcpyDeviceToHost);
    double num = 0, den = 0;
    for (size_t k = 0; k < n; ++k) { num += (back[k] - h[k]) * (back[k] - h[k]); den += h[k] * h[k]; }
    cudaFree(x); cudaFree(spec); cudaFree(y);
    return std::sqrt(num / den);
}

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    int rc = 0;
    const double e_dct = round_trip(comm, DFFT_DCT, 3), e_dst = round_trip(comm, DFFT_DST, 1);
    std::printf("DCT round trip rel-L2 %.3e, DST (d = 1) %.3e\n", e_dct, e_dst);
    if (!(e_dct <= 1e-12) || !(e_dst <= 1e-12)) rc = 1;
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
