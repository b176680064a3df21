// CPU emulation of the paired R2C / C2R z pass of interleaved plans (fft_rc_ilv_kernel): runs its per-line steps — two real
// components packed as z = x_a + i x_b, fft_core.cuh's stage arithmetic "one thread at a time" with the kernels'
// shared-memory layout, the split through Z[-k mod N] and the inverse build from X[k] / conj X[N-k] — through the helpers of
// r2r.hpp, and checks both components against a naive long-double R2C / C2R for every N = 4..8192, both directions, f64 and
// f32, with a partner (even C) and with a zero partner (the last component of an odd C).  Built and run by
// tests/test_components.py (no GPU needed).  Prints the worst rel-L2 error per precision; exit code 0 = every case passes.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../distributedfft_b200/csrc/r2r.hpp"

using namespace dfft;

// One CONTIG line (TB = 1) through the stages, with the shared-memory exchange of the kernels' SmemLayout.
template <typename T, int LOG2N, int LOG2E, int ST>
struct RunStages {
    using Core = FftCore<T, LOG2N, LOG2E>;
    using L = SmemLayout<LOG2N, LOG2E, 1, false, int(sizeof(cx<T>))>;
    static void run(std::vector<cx<T>>& regs, std::vector<cx<T>>& smem, const cx<T>* tw) {
        constexpr int E = Core::E, TPL = Core::TPL, NST = Core::NST;
        for (int j = 0; j < TPL; ++j) {
            cx<T>(&v)[E] = *reinterpret_cast<cx<T>(*)[E]>(&regs[size_t(j) * E]);
            Core::template stage_compute<ST>(v, j, tw);
        }
        if constexpr (ST + 1 < NST) {
            for (int j = 0; j < TPL; ++j) {
                const int sb = L::idx(Core::template scatter_base<ST>(j), 0);
                for (int e = 0; e < E; ++e) smem[sb + L::off(Core::template scatter_off<ST>(e))] = regs[size_t(j) * E + e];
            }
            for (int j = 0; j < TPL; ++j)
                for (int e = 0; e < E; ++e) regs[size_t(j) * E + e] = smem[L::idx(j + e * TPL, 0)];
            RunStages<T, LOG2N, LOG2E, ST + 1>::run(regs, smem, tw);
        }
    }
};

// Forward: reals a, b (b absent: zero partner) -> half spectra A, B (N/2 + 1 points).  Inverse: half spectra -> reals.
template <typename T, int LOG2N>
void pair_line(const std::vector<T>& a, const std::vector<T>& b, const std::vector<cx<T>>& A, const std::vector<cx<T>>& B, bool has_b,
               std::vector<T>& ya, std::vector<T>& yb, std::vector<cx<T>>& YA, std::vector<cx<T>>& YB, const std::vector<cx<T>>& tw, bool inverse) {
    constexpr int LOG2E = LOG2N < 4 ? LOG2N : 4;
    using Core = FftCore<T, LOG2N, LOG2E>;
    using L = SmemLayout<LOG2N, LOG2E, 1, false, int(sizeof(cx<T>))>;
    constexpr int N = Core::N, E = Core::E, TPL = Core::TPL;
    std::vector<cx<T>> regs(size_t(TPL) * E), smem(L::ELEMS);
    const cx<T> zero{T(0), T(0)};
    if (!inverse) {
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) regs[size_t(j) * E + e] = cx<T>{a[j + e * TPL], has_b ? b[j + e * TPL] : T(0)};
        RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) smem[L::idx(j + e * TPL, 0)] = regs[size_t(j) * E + Core::final_slot(e)];
        YA.assign(N / 2 + 1, zero);
        YB.assign(N / 2 + 1, zero);
        for (int k = 0; 2 * k <= N; ++k) {
            cx<T> xa, xb;
            rc_pair_split<T>(smem[L::idx(k, 0)], smem[L::idx((N - k) & (N - 1), 0)], xa, xb);
            YA[k] = xa;
            if (has_b) YB[k] = xb;
        }
    } else {
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) {
                const int k = j + e * TPL, m = rc_pair_in_k(k, N);
                regs[size_t(j) * E + e] = cswap(rc_pair_build<T>(A[m], has_b ? B[m] : zero, k, N));
            }
        RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
        ya.assign(N, T(0));
        yb.assign(N, T(0));
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) {
                const cx<T> z = cswap(regs[size_t(j) * E + Core::final_slot(e)]);
                ya[j + e * TPL] = z.x;
                if (has_b) yb[j + e * TPL] = z.y;
            }
    }
}

template <typename T, int LOG2N = 2>
void dispatch(int lg, const std::vector<T>& a, const std::vector<T>& b, const std::vector<cx<T>>& A, const std::vector<cx<T>>& B, bool has_b,
              std::vector<T>& ya, std::vector<T>& yb, std::vector<cx<T>>& YA, std::vector<cx<T>>& YB, const std::vector<cx<T>>& tw, bool inverse) {
    if (lg == LOG2N) pair_line<T, LOG2N>(a, b, A, B, has_b, ya, yb, YA, YB, tw, inverse);
    else if constexpr (LOG2N < 13) dispatch<T, LOG2N + 1>(lg, a, b, A, B, has_b, ya, yb, YA, YB, tw, inverse);
    else abort();
}

template <typename T>
double check(int lg, bool inverse, bool lone) {
    const int N = 1 << lg, H = N / 2 + 1;
    std::vector<cx<T>> tw(N);
    for (int m = 0; m < N; ++m) {
        long double ang = -2.0L * M_PIl * m / N;
        tw[m] = cx<T>{T(cosl(ang)), T(sinl(ang))};
    }
    std::vector<long double> c(N), s(N);
    for (int i = 0; i < N; ++i) { c[i] = cosl(2.0L * M_PIl * i / N); s[i] = sinl(2.0L * M_PIl * i / N); }
    srand(777 + 13 * lg + (inverse ? 1 : 0));
    auto rnd = [] { return rand() / double(RAND_MAX) - 0.5; };
    std::vector<T> a(N), b(N), ya, yb;
    std::vector<cx<T>> A(H), B(H), YA, YB;
    for (int n = 0; n < N; ++n) { a[n] = T(rnd()); b[n] = T(rnd()); }
    // inverse inputs: half spectra of real lines (X[0] and X[N/2] real), as every forward transform produces
    for (int k = 0; k < H; ++k) {
        const bool real = k == 0 || 2 * k == N;
        A[k] = cx<T>{T(rnd()), real ? T(0) : T(rnd())};
        B[k] = cx<T>{T(rnd()), real ? T(0) : T(rnd())};
    }
    dispatch<T>(lg, a, b, A, B, !lone, ya, yb, YA, YB, tw, inverse);
    long double num = 0, den = 0;
    for (int line = 0; line < (lone ? 1 : 2); ++line) {
        if (!inverse) {
            const std::vector<T>& x = line ? b : a;
            const std::vector<cx<T>>& Y = line ? YB : YA;
            for (int k = 0; k < H; ++k) {
                long double re = 0, im = 0;
                for (int n = 0; n < N; ++n) { re += x[n] * c[((long long)k * n) % N]; im -= x[n] * s[((long long)k * n) % N]; }
                num += (Y[k].x - re) * (Y[k].x - re) + (Y[k].y - im) * (Y[k].y - im);
                den += re * re + im * im;
            }
        } else {  // y_n = sum_k X[k] exp(2 pi i k n / N) over the Hermitian extension
            const std::vector<cx<T>>& X = line ? B : A;
            const std::vector<T>& y = line ? yb : ya;
            for (int n = 0; n < N; ++n) {
                long double r = X[0].x + ((n & 1) ? -1 : 1) * (long double)X[N / 2].x;
                for (int k = 1; 2 * k < N; ++k) r += 2 * (X[k].x * c[((long long)k * n) % N] - X[k].y * s[((long long)k * n) % N]);
                num += (y[n] - r) * (y[n] - r);
                den += r * r;
            }
        }
    }
    // a zero partner stores nothing
    if (lone) {
        for (const cx<T>& v : YB) if (v.x != T(0) || v.y != T(0)) return 1.0;
        for (T v : yb) if (v != T(0)) return 1.0;
    }
    return double(sqrtl(num / den));
}

int main() {
    int fails = 0, cases = 0;
    double worst64 = 0, worst32 = 0;
    for (int lg = 2; lg <= 13; ++lg)
        for (int inv = 0; inv < 2; ++inv)
            for (int lone = 0; lone < 2; ++lone) {
                const double e64 = check<double>(lg, inv, lone), e32 = check<float>(lg, inv, lone);
                ++cases;
                worst64 = e64 > worst64 ? e64 : worst64;
                worst32 = e32 > worst32 ? e32 : worst32;
                if (!(e64 <= 1e-15) || !(e32 <= 1e-6)) {
                    printf("N=%d %s%s f64 relL2=%.3e f32 relL2=%.3e FAIL\n", 1 << lg, inv ? "C2R" : "R2C", lone ? " (zero partner)" : "", e64, e32);
                    ++fails;
                }
            }
    printf("cases=%d worst f64 relL2=%.3e worst f32 relL2=%.3e\n", cases, worst64, worst32);
    printf("fails=%d\n", fails);
    return fails ? 1 : 0;
}
