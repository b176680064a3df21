// batch_shim_test.cpp — the batched initFFT overload of include/dfft.hpp: a C2C MPIcuFFT_Slab<double> of 4 fields of 64^3
// (one launch) and of 3 fields of 16^3 (per field), forward and inverse, compared byte for byte (memcmp) with the
// unbatched plan run on every field.
// Build (tests/test_gpu_batch.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include batch_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

static int run(size_t n, size_t batch, dfft_comm_t comm) {
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(n, n, n);
    MPIcuFFT_Slab<double> batched(cfg, comm, -1, DFFT_C2C), single(cfg, comm, -1, DFFT_C2C);
    batched.initFFT(&gs, nullptr, true, batch);
    single.initFFT(&gs, true);
    if (batched.getBatch() != batch || single.getBatch() != 1) { std::printf("getBatch\n"); return 1; }
    const size_t field = n * n * n, bytes = batch * field * 16;
    std::vector<double> h(2 * batch * field);
    for (size_t i = 0; i < h.size(); ++i) h[i] = double((i * 2654435761u) % 1000) / 7.0;
    void *x, *a, *b;
    if (cudaMalloc(&x, bytes) || cudaMalloc(&a, bytes) || cudaMalloc(&b, bytes)) return 1;
    cudaMemcpy(x, h.data(), bytes, cudaMemcpyHostToDevice);
    std::vector<char> ha(bytes), hb(bytes);
    for (int dir : {DFFT_FORWARD, DFFT_INVERSE}) {
        batched.execC2C(a, x, dir);
        for (size_t f = 0; f < batch; ++f) single.execC2C((char*)b + f * field * 16, (const char*)x + f * field * 16, dir);
        cudaMemcpy(ha.data(), a, bytes, cudaMemcpyDeviceToHost);
        cudaMemcpy(hb.data(), b, bytes, cudaMemcpyDeviceToHost);
        if (std::memcmp(ha.data(), hb.data(), bytes) != 0) {
            std::printf("n=%zu batch=%zu direction %d: batched output differs from the per-field output\n", n, batch, dir);
            return 1;
        }
    }
    cudaFree(x); cudaFree(a); cudaFree(b);
    return 0;
}

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    int rc = run(64, 4, comm) | run(16, 3, comm);
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
