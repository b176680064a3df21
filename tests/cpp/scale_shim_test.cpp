// scale_shim_test.cpp — the reference's testcase 3 (execR2C, then execC2R, compare with the input) through
// MPIcuFFT_Slab<double> of include/dfft.hpp, with setScale(1, 1.0 / N): the round trip gives back the input with no
// scaling by the caller.
// Build (tests/test_gpu_scale.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include scale_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <vector>

#include "dfft.hpp"

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    const size_t nx = 64, ny = 32, nz = 128, n = nx * ny * nz;
    int rc = 0;
    {
        Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
        GlobalSize gs(nx, ny, nz);
        MPIcuFFT_Slab<double> plan(cfg, comm, -1, DFFT_R2C);
        plan.initFFT(&gs, true);
        double f = 0, i = 0;
        plan.getScale(f, i);
        if (f != 1.0 || i != 1.0) { std::printf("default scale (%g, %g)\n", f, i); return 1; }
        plan.setScale(1.0, 1.0 / double(n));
        plan.getScale(f, i);
        if (f != 1.0 || i != 1.0 / double(n)) { std::printf("getScale (%g, %g)\n", f, i); return 1; }
        std::vector<double> h(n), back(n);
        for (size_t k = 0; k < n; ++k) h[k] = double((k * 2654435761u) % 1000) / 999.0;
        void *x, *spec, *y;
        if (cudaMalloc(&x, n * 8) || cudaMalloc(&spec, plan.getDomainSize()) || cudaMalloc(&y, n * 8)) return 1;
        cudaMemcpy(x, h.data(), n * 8, cudaMemcpyHostToDevice);
        plan.execR2C(spec, x);
        plan.execC2R(y, spec);
        cudaMemcpy(back.data(), y, n * 8, cudaMemcpyDeviceToHost);
        double num = 0, den = 0;
        for (size_t k = 0; k < n; ++k) { num += (back[k] - h[k]) * (back[k] - h[k]); den += h[k] * h[k]; }
        const double err = std::sqrt(num / den);
        std::printf("round trip rel-L2 %.3e\n", err);
        if (!(err <= 1e-12)) rc = 1;
        cudaFree(x); cudaFree(spec); cudaFree(y);
    }
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
