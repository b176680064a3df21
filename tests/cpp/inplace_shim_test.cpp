// inplace_shim_test.cpp — the in-place initFFT overload of include/dfft.hpp: MPIcuFFT_Slab<double> plans created with
// initFFT(gs, partition, allocate, batch, inplace = true), C2C 64^3 and R2C / C2R 32x16x64 with padded real rows,
// compared byte for byte (memcmp) with the out-of-place plan on the same input.
// Build (tests/test_gpu_inplace.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include inplace_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

static bool same(const void* dev_a, const void* dev_b, size_t bytes) {
    std::vector<char> a(bytes), b(bytes);
    cudaMemcpy(a.data(), dev_a, bytes, cudaMemcpyDeviceToHost);
    cudaMemcpy(b.data(), dev_b, bytes, cudaMemcpyDeviceToHost);
    return std::memcmp(a.data(), b.data(), bytes) == 0;
}

static int c2c(dfft_comm_t comm) {
    const size_t n = 64, elems = n * n * n, bytes = elems * 16;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(n, n, n);
    MPIcuFFT_Slab<double> ip(cfg, comm, -1, DFFT_C2C), oop(cfg, comm, -1, DFFT_C2C);
    ip.initFFT(&gs, nullptr, true, 1, true);
    oop.initFFT(&gs, true);
    if (!ip.isInPlace() || oop.isInPlace() || ip.getWorkSizeDevice() * 2 != oop.getWorkSizeDevice()) { std::printf("c2c: plan getters\n"); return 1; }
    std::vector<double> h(2 * elems);
    for (size_t i = 0; i < h.size(); ++i) h[i] = double((i * 2654435761u) % 1000) / 7.0;
    void *x, *buf, *ref;
    if (cudaMalloc(&x, bytes) || cudaMalloc(&buf, bytes) || cudaMalloc(&ref, bytes)) return 1;
    cudaMemcpy(x, h.data(), bytes, cudaMemcpyHostToDevice);
    for (int dir : {DFFT_FORWARD, DFFT_INVERSE}) {
        oop.execC2C(ref, x, dir);
        cudaMemcpy(buf, x, bytes, cudaMemcpyDeviceToDevice);
        ip.execC2C(buf, buf, dir);
        if (!same(buf, ref, bytes)) { std::printf("c2c direction %d: in-place output differs\n", dir); return 1; }
    }
    cudaFree(x); cudaFree(buf); cudaFree(ref);
    return 0;
}

static int r2c(dfft_comm_t comm) {
    const size_t nx = 32, ny = 16, nz = 64, nzc = nz / 2 + 1, rows = nx * ny;
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(nx, ny, nz);
    MPIcuFFT_Slab<double> ip(cfg, comm), oop(cfg, comm);
    ip.initFFT(&gs, nullptr, true, 1, true);
    oop.initFFT(&gs, true);
    if (ip.getDomainSize() != rows * nzc * 16) { std::printf("r2c: domain size\n"); return 1; }
    std::vector<double> real(rows * nz), padded(rows * 2 * nzc, 0.0);
    for (size_t i = 0; i < real.size(); ++i) real[i] = double((i * 2246822519u) % 997) / 13.0;
    for (size_t r = 0; r < rows; ++r) std::memcpy(&padded[r * 2 * nzc], &real[r * nz], nz * sizeof(double));
    void *x, *spec, *back, *buf;
    const size_t rbytes = rows * nz * 8, cbytes = rows * nzc * 16;
    if (cudaMalloc(&x, rbytes) || cudaMalloc(&spec, cbytes) || cudaMalloc(&back, rbytes) || cudaMalloc(&buf, cbytes)) return 1;
    cudaMemcpy(x, real.data(), rbytes, cudaMemcpyHostToDevice);
    cudaMemcpy(buf, padded.data(), cbytes, cudaMemcpyHostToDevice);
    oop.execR2C(spec, x);
    ip.execR2C(buf, buf);
    if (!same(buf, spec, cbytes)) { std::printf("r2c: in-place spectrum differs\n"); return 1; }
    oop.execC2R(back, spec);
    ip.execC2R(buf, buf);
    std::vector<double> got(rows * 2 * nzc), want(rows * nz);
    cudaMemcpy(got.data(), buf, cbytes, cudaMemcpyDeviceToHost);
    cudaMemcpy(want.data(), back, rbytes, cudaMemcpyDeviceToHost);
    for (size_t r = 0; r < rows; ++r)
        if (std::memcmp(&got[r * 2 * nzc], &want[r * nz], nz * sizeof(double)) != 0) { std::printf("c2r: row %zu differs\n", r); return 1; }
    cudaFree(x); cudaFree(spec); cudaFree(back); cudaFree(buf);
    return 0;
}

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    int rc = c2c(comm) | r2c(comm);
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
