// CPU emulation of the R2C / C2R z pass of interleaved plans (fft_rc_ilv_kernel): runs its per-line steps — one real
// component as z = x + 0i, fft_core.cuh's stage arithmetic "one thread at a time" with the kernels' shared-memory layout,
// the split through Z[-k mod N] and the inverse build from X[k] / conj X[N-k] — through the helpers of r2r.hpp, and checks
// the component against a naive long-double R2C / C2R for every N = 4..8192, both directions, f64 and f32.  (The pass once
// carried two components in one line, z = x_a + i x_b; tests/test_gpu_accuracy.py emulates that split and shows why it
// went: the smaller component inherits the larger one's rounding error.)  Built and run by tests/test_components.py (no
// GPU needed).  Prints the worst rel-L2 error per precision; exit code 0 = every case passes.
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

// Forward: reals a -> half spectrum YA (N/2 + 1 points).  Inverse: half spectrum A -> reals ya.
template <typename T, int LOG2N>
void rc_line(const std::vector<T>& a, const std::vector<cx<T>>& A, std::vector<T>& ya, std::vector<cx<T>>& YA, const std::vector<cx<T>>& tw,
             bool inverse) {
    constexpr int LOG2E = LOG2N < 4 ? LOG2N : 4;
    using Core = FftCore<T, LOG2N, LOG2E>;
    using L = SmemLayout<LOG2N, LOG2E, 1, false, int(sizeof(cx<T>))>;
    constexpr int N = Core::N, E = Core::E, TPL = Core::TPL;
    std::vector<cx<T>> regs(size_t(TPL) * E), smem(L::ELEMS);
    if (!inverse) {
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) regs[size_t(j) * E + e] = cx<T>{a[j + e * TPL], T(0)};
        RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) smem[L::idx(j + e * TPL, 0)] = regs[size_t(j) * E + Core::final_slot(e)];
        YA.assign(N / 2 + 1, cx<T>{T(0), T(0)});
        for (int k = 0; 2 * k <= N; ++k) YA[k] = rc_line_split<T>(smem[L::idx(k, 0)], smem[L::idx((N - k) & (N - 1), 0)]);
    } else {
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) {
                const int k = j + e * TPL;
                regs[size_t(j) * E + e] = cswap(rc_line_build<T>(A[rc_line_in_k(k, N)], k, N));
            }
        RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
        ya.assign(N, T(0));
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) ya[j + e * TPL] = cswap(regs[size_t(j) * E + Core::final_slot(e)]).x;
    }
}

template <typename T, int LOG2N = 2>
void dispatch(int lg, const std::vector<T>& a, const std::vector<cx<T>>& A, std::vector<T>& ya, std::vector<cx<T>>& YA, const std::vector<cx<T>>& tw,
              bool inverse) {
    if (lg == LOG2N) rc_line<T, LOG2N>(a, A, ya, YA, tw, inverse);
    else if constexpr (LOG2N < 13) dispatch<T, LOG2N + 1>(lg, a, A, ya, YA, tw, inverse);
    else abort();
}

template <typename T>
double check(int lg, bool inverse) {
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
    std::vector<T> a(N), ya;
    std::vector<cx<T>> A(H), YA;
    for (int n = 0; n < N; ++n) a[n] = T(rnd());
    // inverse inputs: half spectra of real lines (X[0] and X[N/2] real), as every forward transform produces
    for (int k = 0; k < H; ++k) {
        const bool real = k == 0 || 2 * k == N;
        A[k] = cx<T>{T(rnd()), real ? T(0) : T(rnd())};
    }
    dispatch<T>(lg, a, A, ya, YA, tw, inverse);
    long double num = 0, den = 0;
    if (!inverse) {
        for (int k = 0; k < H; ++k) {
            long double re = 0, im = 0;
            for (int n = 0; n < N; ++n) { re += a[n] * c[((long long)k * n) % N]; im -= a[n] * s[((long long)k * n) % N]; }
            num += (YA[k].x - re) * (YA[k].x - re) + (YA[k].y - im) * (YA[k].y - im);
            den += re * re + im * im;
        }
        // the imaginary parts of X[0] and X[N/2] are exact zeros, as for every real line
        if (YA[0].y != T(0) || YA[N / 2].y != T(0)) return 1.0;
    } else {  // y_n = sum_k X[k] exp(2 pi i k n / N) over the Hermitian extension
        for (int n = 0; n < N; ++n) {
            long double r = A[0].x + ((n & 1) ? -1 : 1) * (long double)A[N / 2].x;
            for (int k = 1; 2 * k < N; ++k) r += 2 * (A[k].x * c[((long long)k * n) % N] - A[k].y * s[((long long)k * n) % N]);
            num += (ya[n] - r) * (ya[n] - r);
            den += r * r;
        }
    }
    return double(sqrtl(num / den));
}

int main() {
    int fails = 0, cases = 0;
    double worst64 = 0, worst32 = 0;
    for (int lg = 2; lg <= 13; ++lg)
        for (int inv = 0; inv < 2; ++inv) {
            const double e64 = check<double>(lg, inv), e32 = check<float>(lg, inv);
            ++cases;
            worst64 = e64 > worst64 ? e64 : worst64;
            worst32 = e32 > worst32 ? e32 : worst32;
            if (!(e64 <= 1e-15) || !(e32 <= 1e-6)) {
                printf("N=%d %s f64 relL2=%.3e f32 relL2=%.3e FAIL\n", 1 << lg, inv ? "C2R" : "R2C", e64, e32);
                ++fails;
            }
        }
    printf("cases=%d worst f64 relL2=%.3e worst f32 relL2=%.3e\n", cases, worst64, worst32);
    printf("fails=%d\n", fails);
    return fails ? 1 : 0;
}
