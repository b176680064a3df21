// components_shim_test.cpp — initFFTInterleaved of include/dfft.hpp: MPIcuFFT_Slab<double> C2C and R2C plans of a 16x32x64
// grid with 3 components per point, against the batched plan (batch = 3) on the component-major copy of the same data,
// byte for byte (memcmp) in both directions, plus getComponents and the sizes.
// Build (tests/test_gpu_components.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include components_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

// [P][C] (interleaved) <-> [C][P] (component-major), P points of `bytes` each
static std::vector<char> transpose(const std::vector<char>& a, size_t rows, size_t cols, size_t bytes) {
    std::vector<char> b(a.size());
    for (size_t r = 0; r < rows; ++r)
        for (size_t c = 0; c < cols; ++c) std::memcpy(&b[(c * rows + r) * bytes], &a[(r * cols + c) * bytes], bytes);
    return b;
}

static int run(int transform, dfft_comm_t comm) {
    const size_t C = 3, n[3] = {16, 32, 64};
    const bool real = transform == DFFT_R2C;
    const size_t pin = n[0] * n[1] * n[2], pout = n[0] * n[1] * (real ? n[2] / 2 + 1 : n[2]);
    const size_t bin = real ? 8 : 16, bout = 16;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(n[0], n[1], n[2]);
    MPIcuFFT_Slab<double> ilv(cfg, comm, -1, transform), bat(cfg, comm, -1, transform);
    ilv.initFFTInterleaved(&gs, nullptr, C, true);
    bat.initFFT(&gs, nullptr, true, C);
    int rc = 0;
    if (ilv.getComponents() != C || bat.getComponents() != 1) { std::printf("getComponents\n"); rc = 1; }
    if (ilv.getDomainSize() != C * bat.getDomainSize()) { std::printf("domain size\n"); rc = 1; }
    size_t a[3], b[3];
    ilv.getOutSize(a);
    bat.getOutSize(b);
    if (std::memcmp(a, b, sizeof a) != 0) { std::printf("out size\n"); rc = 1; }
    std::vector<char> x(C * pin * bin);
    for (size_t i = 0; i < x.size() / 8; ++i) {
        const double v = double((i * 2654435761u) % 1000) / 7.0 - 70.0;
        std::memcpy(&x[8 * i], &v, 8);
    }
    const std::vector<char> xc = transpose(x, pin, C, bin);
    void *d_in, *d_out, *d_back;
    if (cudaMalloc(&d_in, x.size()) || cudaMalloc(&d_out, C * pout * bout) || cudaMalloc(&d_back, x.size())) return 1;
    std::vector<char> yi(C * pout * bout), yb(yi.size()), bi(x.size()), bb(x.size());
    // interleaved forward and inverse
    cudaMemcpy(d_in, x.data(), x.size(), cudaMemcpyHostToDevice);
    if (real) ilv.execR2C(d_out, d_in); else ilv.execC2C(d_out, d_in, DFFT_FORWARD);
    cudaMemcpy(yi.data(), d_out, yi.size(), cudaMemcpyDeviceToHost);
    if (real) ilv.execC2R(d_back, d_out); else ilv.execC2C(d_back, d_out, DFFT_INVERSE);
    cudaMemcpy(bi.data(), d_back, bi.size(), cudaMemcpyDeviceToHost);
    // batched, component-major
    cudaMemcpy(d_in, xc.data(), xc.size(), cudaMemcpyHostToDevice);
    if (real) bat.execR2C(d_out, d_in); else bat.execC2C(d_out, d_in, DFFT_FORWARD);
    cudaMemcpy(yb.data(), d_out, yb.size(), cudaMemcpyDeviceToHost);
    if (real) bat.execC2R(d_back, d_out); else bat.execC2C(d_back, d_out, DFFT_INVERSE);
    cudaMemcpy(bb.data(), d_back, bb.size(), cudaMemcpyDeviceToHost);
    cudaFree(d_in); cudaFree(d_out); cudaFree(d_back);
    if (!real) {  // the C2C passes run the same arithmetic per line: byte for byte
        if (std::memcmp(transpose(yi, pout, C, bout).data(), yb.data(), yb.size()) != 0) { std::printf("C2C forward differs\n"); rc = 1; }
        if (std::memcmp(transpose(bi, pin, C, bin).data(), bb.data(), bb.size()) != 0) { std::printf("C2C inverse differs\n"); rc = 1; }
        return rc;
    }
    // R2C / C2R: the paired z pass is other arithmetic than the half-length kernel; within 1e-12 of the batched plan
    auto close = [&](const std::vector<char>& u, const std::vector<char>& v) {
        double num = 0, den = 0;
        for (size_t i = 0; i < u.size() / 8; ++i) {
            double p, q;
            std::memcpy(&p, &u[8 * i], 8);
            std::memcpy(&q, &v[8 * i], 8);
            num += (p - q) * (p - q);
            den += q * q;
        }
        return num <= 1e-24 * den;
    };
    if (!close(transpose(yi, pout, C, bout), yb)) { std::printf("R2C forward differs\n"); rc = 1; }
    if (!close(transpose(bi, pin, C, bin), bb)) { std::printf("C2R inverse differs\n"); rc = 1; }
    return rc;
}

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    int rc = 0;
    try {
        rc = run(DFFT_C2C, comm) | run(DFFT_R2C, comm);
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        rc = 1;
    }
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
