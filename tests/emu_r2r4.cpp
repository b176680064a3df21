// CPU emulation of the type-IV R2R pass (fft_r2r4_kernel): runs its per-line steps — the loads of x_{2m} and x_{N-1-2m}
// into M = N/2 complex points times p_m, fft_core.cuh's stage arithmetic "one thread at a time" with the kernels'
// shared-memory layout, and the post-twiddle q_k of each point's final slot into y_{2k} and y_{N-1-2k} — through the helpers
// and the host table of r2r.hpp, and checks the line against a naive long-double DCT-IV / DST-IV for every N = 4..8192,
// both kinds, f64 and f32, and that a zero line gives exact zeros.  Built and run by tests/test_r2r4.py (no GPU needed).
// Prints the worst rel-L2 error per precision; exit code 0 = every case passes.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../distributedfft_b200/csrc/r2r.hpp"

using namespace dfft;

// One CONTIG line (TB = 1) through the stages, with the shared-memory exchange of the kernels' SmemLayout.
template <typename T, int LOG2M, int LOG2E, int ST>
struct RunStages {
    using Core = FftCore<T, LOG2M, LOG2E>;
    using L = SmemLayout<LOG2M, LOG2E, 1, false, int(sizeof(cx<T>))>;
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
            RunStages<T, LOG2M, LOG2E, ST + 1>::run(regs, smem, tw);
        }
    }
};

// The kernel's steps on one line x of N = 2M reals; y gets N reals.  tw: the M-point table, w: r2r4_table(N).
template <typename T, int LOG2M>
void r2r4_line(const std::vector<T>& x, std::vector<T>& y, const std::vector<cx<T>>& tw, const std::vector<cx<T>>& w, int dst) {
    constexpr int LOG2E = LOG2M < 4 ? LOG2M : 4;
    using Core = FftCore<T, LOG2M, LOG2E>;
    using L = SmemLayout<LOG2M, LOG2E, 1, false, int(sizeof(cx<T>))>;
    constexpr int M = Core::N, N = 2 * M, E = Core::E, TPL = Core::TPL;
    std::vector<cx<T>> regs(size_t(TPL) * E), smem(L::ELEMS);
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) {
            const int m = j + e * TPL;
            regs[size_t(j) * E + e] = r2r4_pre<T>(x[r2r4_lo(m)], x[r2r4_hi(m, N)], w[m], dst);
        }
    RunStages<T, LOG2M, LOG2E, 0>::run(regs, smem, tw.data());
    y.assign(x.size(), T(-7));  // every output is written once
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            T lo, hi;
            r2r4_post<T>(regs[size_t(j) * E + Core::final_slot(e)], w[M + k], dst, lo, hi);
            y[r2r4_lo(k)] = lo;
            y[r2r4_hi(k, N)] = hi;
        }
}

template <typename T, int LOG2M = 1>
void dispatch(int lg, const std::vector<T>& x, std::vector<T>& y, const std::vector<cx<T>>& tw, const std::vector<cx<T>>& w, int dst) {
    if (lg == LOG2M) r2r4_line<T, LOG2M>(x, y, tw, w, dst);
    else if constexpr (LOG2M < 12) dispatch<T, LOG2M + 1>(lg, x, y, tw, w, dst);
    else abort();
}

// naive long-double DCT-IV / DST-IV (scipy type=4 norm=None, FFTW REDFT11 / RODFT11); c[i] = cos(pi i / 4N),
// s[i] = sin(pi i / 4N) for i < 8N
static long double naive(const std::vector<long double>& x, int k, int N, int dst, const std::vector<long double>& c,
                         const std::vector<long double>& s) {
    long double r = 0;
    for (int n = 0; n < N; ++n) {
        const long long i = (long long)(2 * n + 1) * (2 * k + 1) % (8 * N);
        r += 2 * x[n] * (dst ? s[i] : c[i]);
    }
    return r;
}

template <typename T>
double check(int lg, int dst, bool* zero_ok) {
    const int N = 1 << lg, M = N / 2;
    std::vector<cx<T>> tw(M);
    for (int m = 0; m < M; ++m) {  // Tables::get_tw(log2 M)
        const long double ang = -2.0L * M_PIl * m / M;
        tw[m] = cx<T>{T(cosl(ang)), T(sinl(ang))};
    }
    const std::vector<cx<T>> w = r2r4_table<T>(N);  // Tables::get_r2r4(log2 N)
    std::vector<long double> c(8 * N), s(8 * N);
    for (int i = 0; i < 8 * N; ++i) {
        c[i] = cosl(M_PIl * i / (4.0L * N));
        s[i] = sinl(M_PIl * i / (4.0L * N));
    }
    std::vector<T> x(N), y;
    srand(4321 + 7 * lg + dst);
    for (int n = 0; n < N; ++n) x[n] = T(rand() / double(RAND_MAX) - 0.5);
    dispatch<T>(lg - 1, x, y, tw, w, dst);
    const std::vector<long double> xl(x.begin(), x.end());
    long double num = 0, den = 0;
    for (int k = 0; k < N; ++k) {
        const long double r = naive(xl, k, N, dst, c, s);
        num += (y[k] - r) * (y[k] - r);
        den += r * r;
    }
    // a zero line gives exact zeros
    std::vector<T> z(N, T(0)), yz;
    dispatch<T>(lg - 1, z, yz, tw, w, dst);
    for (int k = 0; k < N; ++k)
        if (yz[k] != T(0)) *zero_ok = false;
    return double(sqrtl(num / den));
}

int main() {
    int fails = 0, cases = 0;
    double worst64 = 0, worst32 = 0;
    static char b64[64] = "", b32[64] = "";
    for (int lg = 2; lg <= 13; ++lg)
        for (int dst = 0; dst < 2; ++dst) {
            bool zero_ok = true;
            const double e64 = check<double>(lg, dst, &zero_ok), e32 = check<float>(lg, dst, &zero_ok);
            ++cases;
            const int N = 1 << lg;
            if (e64 > worst64) { worst64 = e64; snprintf(b64, sizeof b64, "N=%d %s", N, dst ? "DST-IV" : "DCT-IV"); }
            if (e32 > worst32) { worst32 = e32; snprintf(b32, sizeof b32, "N=%d %s", N, dst ? "DST-IV" : "DCT-IV"); }
            if (!(e64 <= 1e-10) || !(e32 <= 1e-5) || !zero_ok) {
                printf("N=%d %s f64 relL2=%.3e f32 relL2=%.3e zero line %s FAIL\n", N, dst ? "DST-IV" : "DCT-IV", e64, e32, zero_ok ? "ok" : "NONZERO");
                ++fails;
            }
        }
    printf("cases=%d worst f64 relL2=%.3e (%s) worst f32 relL2=%.3e (%s)\n", cases, worst64, b64, worst32, b32);
    printf("fails=%d\n", fails);
    return fails ? 1 : 0;
}
