// r2r.hpp — per-point arithmetic of the real-to-real pass (fft_r2r_kernel), shared with tests/emu_r2r.cpp.
//
// Two real N-point lines a and b are transformed through one complex N-point FFT (CtaFft's stages):
//   perm:     v[n] = x[2n],  v[N-1-n] = x[2n+1]  (n < N/2);  z = v_a + i v_b
//   DCT-II:   Z = DFT_N(z),  w_k = exp(-i pi k / 2N)
//             X_a[k] = Re(w_k (Z[k] + conj Z[-k mod N])),  X_b[k] = Im(w_k (Z[k] - conj Z[-k mod N]))
//   DCT-III:  V(X)[k] = conj(w_k) (X[k] - i X[N-k]),  X[N] := 0;  Z = V(X_a) + i V(X_b)
//             z = unnormalised inverse DFT_N(Z);  x_a = perm^-1(Re z),  x_b = perm^-1(Im z)
//   DST-II(x) = reverse(DCT-II((-1)^n x)),  DST-III(X) = (-1)^n DCT-III(reverse(X))
// Unnormalised like FFTW's REDFT10 / REDFT01 / RODFT10 / RODFT01: DCT-III(DCT-II(x)) = 2N x.
#pragma once
#include "fft_core.cuh"

namespace dfft {

// index of the real input (forward) or output (inverse) held by point n of the packed line
DFFT_HD int r2r_perm(int n, int N) { return n < N / 2 ? 2 * n : 2 * (N - 1 - n) + 1; }

// (-1)^m for DST, 1 for DCT
template <typename T>
DFFT_HD T r2r_sign(int m, int dst) { return (dst && (m & 1)) ? T(-1) : T(1); }

// forward: coefficient k of both lines from Z[k] and Z[-k mod N]; w = w_k
template <typename T>
DFFT_HD cx<T> r2r_split(cx<T> zk, cx<T> zm, cx<T> w) {
    const cx<T> c = cconj(zm);
    const cx<T> s = cadd(zk, c), d = csub(zk, c);
    return cx<T>{w.x * s.x - w.y * s.y, w.x * d.y + w.y * d.x};  // {X_a[k], X_b[k]}
}

// forward: position of coefficient k in the output line (DST: reversed)
DFFT_HD int r2r_out_index(int k, int N, int dst) { return dst ? N - 1 - k : k; }

// inverse: positions in the input line of X[k] and X[N-k] (DST: of the reversed line); -1 for the X[N] := 0 term
DFFT_HD int r2r_in_k(int k, int N, int dst) { return dst ? N - 1 - k : k; }
DFFT_HD int r2r_in_nk(int k, int N, int dst) { return k == 0 ? -1 : (dst ? k - 1 : N - k); }

// inverse: Z[k] = V(X_a)[k] + i V(X_b)[k] from X_a[k], X_a[N-k], X_b[k], X_b[N-k]; w = w_k
template <typename T>
DFFT_HD cx<T> r2r_build(T ak, T am, T bk, T bm, cx<T> w) {
    const cx<T> wc = cconj(w);
    const cx<T> va = cmul(wc, cx<T>{ak, -am}), vb = cmul(wc, cx<T>{bk, -bm});
    return cx<T>{va.x - vb.y, va.y + vb.x};
}

}  // namespace dfft
