// bluestein.hpp — host tables of the Bluestein pass (fft_bluestein_kernel), shared with tests/emu_bluestein.cpp.
//
// A line of n points (n not a power of two) is transformed through two FFTs of length M = 2^bluestein_log2m(n) >= 2n - 1:
//   c_k  = exp(-pi i k^2 / n)                         (the chirp, k < n)
//   h_k  = conj(c_|k|) for |k| < n, indices mod M; 0 elsewhere
//   K^   = FFT_M(h) / M                               (the kernel spectrum; 1/M is the inverse FFT's normalisation)
//   X_k  = c_k * IFFT_M(FFT_M(x * c) * K^)_k           (IFFT_M unnormalised)
// Everything is evaluated in long double and rounded to the plan's precision once: k^2 mod 2n exactly in 64-bit integers,
// K^ with a long-double radix-2 FFT on exactly evaluated twiddles.
#pragma once
#include <cmath>
#include <cstddef>
#include <utility>
#include <vector>

#include "fft_core.cuh"

namespace dfft {

// log2 of the smallest power of two >= 2n - 1
inline int bluestein_log2m(size_t n) {
    int l = 0;
    while ((size_t(1) << l) < 2 * n - 1) ++l;
    return l;
}

// [K^ (M entries)][chirp (n entries)] in the precision T
template <typename T>
std::vector<cx<T>> bluestein_table(size_t n) {
    typedef long double R;
    const R pi = 3.14159265358979323846264338327950288L;
    const int lg = bluestein_log2m(n);
    const size_t M = size_t(1) << lg;
    std::vector<R> cr(n), ci(n);
    for (size_t k = 0; k < n; ++k) {
        const unsigned long long q = (unsigned long long)k * k % (2ull * n);  // exp(-pi i k^2 / n) has period 2n in k^2
        const R a = -pi * R(q) / R(n);
        cr[k] = cosl(a);
        ci[k] = sinl(a);
    }
    std::vector<R> hr(M, 0), hi(M, 0);
    for (size_t k = 0; k < n; ++k) {
        hr[k] = cr[k]; hi[k] = -ci[k];
        if (k) { hr[M - k] = cr[k]; hi[M - k] = -ci[k]; }
    }
    // iterative radix-2 DIT FFT in long double: bit-reversed input order, then log2 M butterfly levels
    for (size_t i = 0; i < M; ++i) {
        const size_t r = size_t(bitrev_c(int(i), lg));
        if (r > i) { std::swap(hr[i], hr[r]); std::swap(hi[i], hi[r]); }
    }
    std::vector<R> wr(M / 2 + 1), wi(M / 2 + 1);
    for (size_t m = 0; m <= M / 2; ++m) {
        const R a = -2 * pi * R(m) / R(M);
        wr[m] = cosl(a);
        wi[m] = sinl(a);
    }
    for (size_t len = 2; len <= M; len <<= 1) {
        const size_t half = len / 2, step = M / len;
        for (size_t b = 0; b < M; b += len)
            for (size_t q = 0; q < half; ++q) {
                const R xr = wr[q * step], xi = wi[q * step];
                const size_t i0 = b + q, i1 = i0 + half;
                const R tr = hr[i1] * xr - hi[i1] * xi, ti = hr[i1] * xi + hi[i1] * xr;
                hr[i1] = hr[i0] - tr; hi[i1] = hi[i0] - ti;
                hr[i0] += tr; hi[i0] += ti;
            }
    }
    std::vector<cx<T>> out(M + n);
    for (size_t m = 0; m < M; ++m) out[m] = cx<T>{T(hr[m] / R(M)), T(hi[m] / R(M))};
    for (size_t k = 0; k < n; ++k) out[M + k] = cx<T>{T(cr[k]), T(ci[k])};
    return out;
}

}  // namespace dfft
