// r2r.hpp — per-point arithmetic of the real-to-real passes (fft_r2r_kernel, fft_r2hc_kernel, fft_r2r1_kernel,
// fft_r2r4_kernel), shared with tests/emu_r2r.cpp, tests/emu_r2hc.cpp, tests/emu_r2r1.cpp and tests/emu_r2r4.cpp.
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
#include <cmath>
#include <vector>

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

// ---- R2HC / HC2R (fft_r2hc_kernel): the same pairing without permutation or w_k ----------------------------------------
// Halfcomplex line of X = DFT_N(x) (FFTW's R2HC format): hc[k] = Re X[k] for k <= N/2, hc[N-k] = Im X[k] for 0 < k < N/2.
//   R2HC:  z = a + i b in natural order,  Z = DFT_N(z);  with m = -k mod N, A = (Z[k] + conj Z[m]) / 2 = X_a[k] and
//          B = (Z[k] - conj Z[m]) / 2i = X_b[k], so hc_a[k] = Re A (k <= N/2) or Im A[m] (k > N/2), and likewise hc_b.
//   HC2R:  Z[k] = X_a[k] + i X_b[k], the full spectra rebuilt from hc[k] and hc[N-k];  z = unnormalised inverse DFT_N(Z),
//          a = Re z, b = Im z.
// Unnormalised like FFTW's R2HC / HC2R: HC2R(R2HC(x)) = N x.

// forward: halfcomplex point k of both lines from Z[k] and Z[-k mod N] (the halving is exact)
template <typename T>
DFFT_HD cx<T> r2hc_split(cx<T> zk, cx<T> zm, int k, int N) {
    if (2 * k <= N) return cx<T>{T(0.5) * (zk.x + zm.x), T(0.5) * (zk.y + zm.y)};
    return cx<T>{T(0.5) * (zm.y - zk.y), T(0.5) * (zk.x - zm.x)};  // {hc_a[k], hc_b[k]}
}

// inverse: position in the input line of hc[N-k], the other half of X[k]; -1 when X[k] is real (k = 0 and k = N/2)
DFFT_HD int r2hc_in_nk(int k, int N) { return k == 0 || 2 * k == N ? -1 : N - k; }

// inverse: Z[k] = X_a[k] + i X_b[k] from hc[k] (ak, bk) and hc[N-k] (am, bm; 0 when X[k] is real)
template <typename T>
DFFT_HD cx<T> r2hc_build(T ak, T am, T bk, T bm, int k, int N) {
    // X[k] = hc[k] + i hc[N-k] for k <= N/2, conj X[N-k] = hc[N-k] - i hc[k] above
    const bool lo = 2 * k <= N;
    const cx<T> xa = lo ? cx<T>{ak, am} : cx<T>{am, -ak}, xb = lo ? cx<T>{bk, bm} : cx<T>{bm, -bk};
    return cx<T>{xa.x - xb.y, xa.y + xb.x};
}

// ---- DCT-I / DST-I (fft_r2r1_kernel): one real line per complex N-point FFT ------------------------------------------------
// FFTW's REDFT00 (L = N + 1 points) and RODFT00 (L = N - 1) are DFTs of the line's 2N-point extension e:
//   DCT-I, even:  e = x_0 .. x_N, x_{N-1} .. x_1          DST-I, odd:  e = 0, x_0 .. x_{N-2}, 0, -x_{N-2} .. -x_0
// e is read as N complex points z_m = e_{2m} + i e_{2m+1}, Z = DFT_N(z), and split as the R2C pass does, W = exp(-i pi / N):
//   E_k = (Z_k + conj Z_{N-k}) / 2 - i W^k (Z_k - conj Z_{N-k}) / 2,   k = 0 .. N,  Z_N := Z_0
//   DCT-I:  y_k = Re E_k (k = 0 .. N)          DST-I:  y_k = -Im E_{k+1} (k = 0 .. N - 2)
// (E = DFT_2N(e).)  One line per FFT: pairing two lines as z = e_a + i e_b would need a 2N-point FFT per pair and would tie
// each line's error to its partner's norm.  Unnormalised like scipy's dct / dst with type=1: each is its own inverse up to 2N.

// x index feeding point i < 2N of the extension, -1 where e_i is zero; neg: e_i = -x
DFFT_HD int r2r1_ext(int i, int N, int dst, bool& neg) {
    neg = false;
    if (!dst) return i <= N ? i : 2 * N - i;
    if (i == 0 || i == N) return -1;
    if (i < N) return i - 1;
    neg = true;
    return 2 * N - 1 - i;
}

// E_k and E_{N-k} from Z[k], Z[-k mod N] and w = W^k (W^{N-k} = -conj W^k, so one twiddle of k <= N/2 serves both)
template <typename T>
DFFT_HD void r2r1_split(cx<T> zk, cx<T> zm, cx<T> w, cx<T>& ek, cx<T>& enk) {
    const cx<T> c = cconj(zm);
    const cx<T> xe{T(0.5) * (zk.x + c.x), T(0.5) * (zk.y + c.y)};
    const cx<T> d = csub(zk, c);
    const cx<T> tt = cmul(w, cx<T>{T(0.5) * d.y, T(-0.5) * d.x});  // W^k (-i/2) d
    ek = cadd(xe, tt);
    enk = cconj(csub(xe, tt));
}

// position of E_k's output in the line: k (DCT-I), k - 1 (DST-I), -1 for E_0 and E_N of the DST-I
DFFT_HD int r2r1_out_index(int k, int N, int dst) { return !dst ? k : (k == 0 || k == N ? -1 : k - 1); }
template <typename T>
DFFT_HD T r2r1_value(cx<T> e, int dst) { return dst ? -e.y : e.x; }

// ---- DCT-IV / DST-IV (fft_r2r4_kernel): one real line per complex M-point FFT, M = N/2 -----------------------------------
// FFTW's REDFT11 / RODFT11 of N points, unnormalised like scipy's dct / dst with type=4:
//   DCT-IV:  y_k = 2 sum_{n<N} x_n cos(pi (2n+1)(2k+1) / 4N)        DST-IV:  the same with sin
// Point m < M packs the reals x_{2m} and x_{N-1-2m}; with p_m = exp(-i pi (4m+1) / 4N) and q_k = exp(-i pi k / N):
//   v_m = (x_{2m} + i x_{N-1-2m}) p_m,  V = DFT_M(v),  c_k = V_k q_k,  y_{2k} = 2 Re c_k,  y_{N-1-2k} = -2 Im c_k
// DST-IV(x)_k = (-1)^k DCT-IV(reverse x)_k: the packed point takes its two reals swapped and y_{N-1-2k} = +2 Im c_k.
// Point k's outputs sit at the same index pair as point m's inputs, so each point stores its own results.  One line per
// FFT (no pairing): each line's error follows its own norm.  Each transform is its own inverse up to 2N.

// the reals of packed point m (and outputs of point k): x_{2m} and x_{N-1-2m}
DFFT_HD int r2r4_lo(int m) { return 2 * m; }
DFFT_HD int r2r4_hi(int m, int N) { return N - 1 - 2 * m; }

// v_m from x_{2m} (lo), x_{N-1-2m} (hi) and p = p_m
template <typename T>
DFFT_HD cx<T> r2r4_pre(T lo, T hi, cx<T> p, int dst) { return cmul(dst ? cx<T>{hi, lo} : cx<T>{lo, hi}, p); }

// y_{2k} (lo) and y_{N-1-2k} (hi) from V_k and q = q_k
template <typename T>
DFFT_HD void r2r4_post(cx<T> v, cx<T> q, int dst, T& lo, T& hi) {
    const cx<T> c = cmul(v, q);
    lo = T(2) * c.x;
    hi = (dst ? T(2) : T(-2)) * c.y;
}

// The type-IV table of N-point lines: [p_m (M entries)][q_k (M entries)], evaluated in long double and rounded once
template <typename T>
std::vector<cx<T>> r2r4_table(int N) {
    const int M = N / 2;
    const long double pi = 3.14159265358979323846264338327950288L;
    std::vector<cx<T>> h(size_t(2) * M);
    for (int m = 0; m < M; ++m) {
        const long double a = -pi * (4.0L * m + 1.0L) / (4.0L * N), b = -pi * m / N;
        h[m] = cx<T>{T(cosl(a)), T(sinl(a))};
        h[M + m] = cx<T>{T(cosl(b)), T(sinl(b))};
    }
    return h;
}

// ---- R2C / C2R z pass of interleaved plans (fft_rc_ilv_kernel)---------------------------------------------------------------
// Every component runs its own complex Nz-point line z = x + 0i.  (Two components sharing one line as z = x_a + i x_b would
// halve the arithmetic, but the split then leaves X_b with an error of u |x_a| rather than u |x_b|: components are
// independent fields, so a small one next to a large one would lose its digits.)  Z = DFT_N(z), m = -k mod N:
//   R2C, k = 0 .. N/2:  X[k] = (Z[k] + conj Z[m]) / 2  (the real part of z's spectrum, Hermitian by construction)
//   C2R:  Z[k] = X[k], with X[k] = conj X[N-k] above N/2 and the imaginary parts of X[0], X[N/2] dropped (as numpy's irfft
//         does);  z = unnormalised inverse DFT_N(Z),  x = Re z.
// Unnormalised like cuFFT: C2R(R2C(x)) = N x.

// forward: X[k] from Z[k] and Z[-k mod N] (the halving is exact)
template <typename T>
DFFT_HD cx<T> rc_line_split(cx<T> zk, cx<T> zm) {
    return cx<T>{T(0.5) * (zk.x + zm.x), T(0.5) * (zk.y - zm.y)};
}

// inverse: Z[k] for k in [0, N) from the stored half spectrum: x = X[k] for k <= N/2 (load at k), else X[N-k] (load at N - k)
DFFT_HD int rc_line_in_k(int k, int N) { return 2 * k <= N ? k : N - k; }
template <typename T>
DFFT_HD cx<T> rc_line_build(cx<T> x, int k, int N) {
    if (k == 0 || 2 * k == N) x.y = T(0);
    else if (2 * k > N) x.y = -x.y;
    return x;
}

}  // namespace dfft
