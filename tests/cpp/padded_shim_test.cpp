// padded_shim_test.cpp — the padded initFFT overload of include/dfft.hpp: an MPIcuFFT_Slab<double> C2C plan of a 16x32x64
// grid keeping 11x21x43 modes, against the ordinary plan of the grid.  Forward: the kept modes of the ordinary output,
// gathered through the index map, byte for byte (memcmp).  Inverse: the ordinary inverse of the zero-embedded spectrum,
// byte for byte (the padded passes load zeros where the ordinary ones read them).
// Build (tests/test_gpu_padded.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include padded_shim_test.cpp
//        -Ldistributedfft_b200 -ldfft -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,<repo>/distributedfft_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.hpp"

// line position of spectral index m of a K-point spectrum on an N-point axis (numpy's fftfreq(K) * K mod N)
static size_t pos(size_t m, size_t k, size_t n) { return m < (k + 1) / 2 ? m : m + n - k; }

int main() {
    dfft_comm_t comm;
    if (dfft_comm_create(0, 1, nullptr, 0, &comm) != DFFT_SUCCESS) return 1;
    const size_t n[3] = {16, 32, 64}, k[3] = {11, 21, 43};
    const size_t full = n[0] * n[1] * n[2], kept = k[0] * k[1] * k[2];
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(n[0], n[1], n[2]), ks(k[0], k[1], k[2]);
    int rc = 0;
    {
        MPIcuFFT_Slab<double> pad(cfg, comm, -1, DFFT_C2C), ord(cfg, comm, -1, DFFT_C2C);
        pad.initFFT(&gs, &ks, nullptr, true);
        ord.initFFT(&gs, true);
        size_t sk[3], os[3];
        pad.getSpectralSize(sk);
        pad.getOutSize(os);
        for (int a = 0; a < 3; ++a)
            if (sk[a] != k[a] || os[a] != k[a]) { std::printf("spectral size / out size of axis %d\n", a); rc = 1; }
        std::vector<double> x(2 * full);
        for (size_t i = 0; i < x.size(); ++i) x[i] = double((i * 2654435761u) % 1000) / 7.0 - 70.0;
        void *dx, *dfull, *dkept, *dback, *dref;
        if (cudaMalloc(&dx, full * 16) || cudaMalloc(&dfull, full * 16) || cudaMalloc(&dkept, kept * 16) || cudaMalloc(&dback, full * 16) ||
            cudaMalloc(&dref, full * 16))
            return 1;
        cudaMemcpy(dx, x.data(), full * 16, cudaMemcpyHostToDevice);
        ord.execC2C(dfull, dx, DFFT_FORWARD);
        pad.execC2C(dkept, dx, DFFT_FORWARD);
        std::vector<double> hf(2 * full), hk(2 * kept), want(2 * kept), emb(2 * full, 0.0);
        cudaMemcpy(hf.data(), dfull, full * 16, cudaMemcpyDeviceToHost);
        cudaMemcpy(hk.data(), dkept, kept * 16, cudaMemcpyDeviceToHost);
        for (size_t i = 0; i < k[0]; ++i)
            for (size_t j = 0; j < k[1]; ++j)
                for (size_t l = 0; l < k[2]; ++l) {
                    const size_t src = (pos(i, k[0], n[0]) * n[1] + pos(j, k[1], n[1])) * n[2] + pos(l, k[2], n[2]), dst = (i * k[1] + j) * k[2] + l;
                    std::memcpy(&want[2 * dst], &hf[2 * src], 16);
                    std::memcpy(&emb[2 * src], &hk[2 * dst], 16);
                }
        if (std::memcmp(hk.data(), want.data(), kept * 16) != 0) { std::printf("forward: the kept modes differ\n"); rc = 1; }
        cudaMemcpy(dfull, emb.data(), full * 16, cudaMemcpyHostToDevice);
        ord.execC2C(dref, dfull, DFFT_INVERSE);
        pad.execC2C(dback, dkept, DFFT_INVERSE);
        std::vector<double> a(2 * full), b(2 * full);
        cudaMemcpy(a.data(), dback, full * 16, cudaMemcpyDeviceToHost);
        cudaMemcpy(b.data(), dref, full * 16, cudaMemcpyDeviceToHost);
        if (std::memcmp(a.data(), b.data(), full * 16) != 0) { std::printf("inverse: differs from the zero-embedded inverse\n"); rc = 1; }
        cudaFree(dx); cudaFree(dfull); cudaFree(dkept); cudaFree(dback); cudaFree(dref);
    }
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
