// pruned_shim_test.cpp — the pruned initFFT overload of include/dfft.hpp: an MPIcuFFT_Slab<double> C2C plan of a 16x32x64
// transform grid whose field is a 9x17x30 block at the origin, keeping 11x21x43 modes, against the ordinary plan of the
// grid on the zero-embedded field.  Forward: the kept modes of the ordinary output, gathered through the index map, byte
// for byte (memcmp).  Inverse: the data block of the ordinary inverse of the zero-embedded spectrum, byte for byte (the
// pruned passes take zeros where the ordinary ones load them).
// Build (tests/test_gpu_pruned.py does it): g++ -std=c++17 -Iinclude -I/usr/local/cuda/include pruned_shim_test.cpp
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
    const size_t n[3] = {16, 32, 64}, m[3] = {9, 17, 30}, k[3] = {11, 21, 43};
    const size_t full = n[0] * n[1] * n[2], block = m[0] * m[1] * m[2], kept = k[0] * k[1] * k[2];
    Configurations cfg{false, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
    GlobalSize gs(n[0], n[1], n[2]), ms(m[0], m[1], m[2]), ks(k[0], k[1], k[2]);
    int rc = 0;
    {
        MPIcuFFT_Slab<double> pr(cfg, comm, -1, DFFT_C2C), ord(cfg, comm, -1, DFFT_C2C);
        pr.initFFT(&gs, &ms, &ks, nullptr, true);
        ord.initFFT(&gs, true);
        size_t dm[3], sk[3], is[3], os[3];
        pr.getDataSize(dm);
        pr.getSpectralSize(sk);
        pr.getInSize(is);
        pr.getOutSize(os);
        for (int a = 0; a < 3; ++a)
            if (dm[a] != m[a] || is[a] != m[a] || sk[a] != k[a] || os[a] != k[a]) { std::printf("data / spectral / in / out size of axis %d\n", a); rc = 1; }
        // the field: the m-block, and the same values zero-embedded in the n grid
        std::vector<double> x(2 * block), emb_x(2 * full, 0.0);
        for (size_t i = 0; i < m[0]; ++i)
            for (size_t j = 0; j < m[1]; ++j)
                for (size_t l = 0; l < m[2]; ++l) {
                    const size_t b = (i * m[1] + j) * m[2] + l, f = (i * n[1] + j) * n[2] + l;
                    for (int c = 0; c < 2; ++c) x[2 * b + c] = emb_x[2 * f + c] = double(((2 * b + c) * 2654435761u) % 1000) / 7.0 - 70.0;
                }
        void *dx, *dex, *dfull, *dkept, *dback, *dref;
        if (cudaMalloc(&dx, block * 16) || cudaMalloc(&dex, full * 16) || cudaMalloc(&dfull, full * 16) || cudaMalloc(&dkept, kept * 16) ||
            cudaMalloc(&dback, block * 16) || cudaMalloc(&dref, full * 16))
            return 1;
        cudaMemcpy(dx, x.data(), block * 16, cudaMemcpyHostToDevice);
        cudaMemcpy(dex, emb_x.data(), full * 16, cudaMemcpyHostToDevice);
        ord.execC2C(dfull, dex, DFFT_FORWARD);
        pr.execC2C(dkept, dx, DFFT_FORWARD);
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
        pr.execC2C(dback, dkept, DFFT_INVERSE);
        std::vector<double> a(2 * block), b(2 * full), wb(2 * block);
        cudaMemcpy(a.data(), dback, block * 16, cudaMemcpyDeviceToHost);
        cudaMemcpy(b.data(), dref, full * 16, cudaMemcpyDeviceToHost);
        for (size_t i = 0; i < m[0]; ++i)
            for (size_t j = 0; j < m[1]; ++j)
                std::memcpy(&wb[2 * (i * m[1] + j) * m[2]], &b[2 * (i * n[1] + j) * n[2]], m[2] * 16);
        if (std::memcmp(a.data(), wb.data(), block * 16) != 0) { std::printf("inverse: differs from the zero-embedded inverse\n"); rc = 1; }
        cudaFree(dx); cudaFree(dex); cudaFree(dfull); cudaFree(dkept); cudaFree(dback); cudaFree(dref);
    }
    dfft_comm_destroy(comm);
    if (rc == 0) std::printf("PASSED\n");
    return rc;
}
