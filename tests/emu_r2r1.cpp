// CPU emulation of the type-I R2R pass (fft_r2r1_kernel): runs its per-line steps — the loads of the line's 2N-point even
// (DCT-I) or odd (DST-I) extension as N complex points, fft_core.cuh's stage arithmetic "one thread at a time" with the
// kernels' shared-memory layout, and the split of Z[k] with Z[N-k] by W^k — through the helpers of r2r.hpp, and checks the
// line against a naive long-double DCT-I / DST-I for every N = 2..8192 (DST-I from 4), both kinds, f64 and f32, and that a
// zero line gives exact zeros.  Built and run by tests/test_r2r1.py (no GPU needed).  Prints the worst rel-L2 error per
// precision; exit code 0 = every case passes.
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

// The kernel's steps on one line x of L = N +- 1 reals; y gets L reals.  w: W^k, k <= N/2.
template <typename T, int LOG2N>
void r2r1_line(const std::vector<T>& x, std::vector<T>& y, const std::vector<cx<T>>& tw, const std::vector<cx<T>>& w, int dst) {
    constexpr int LOG2E = LOG2N < 4 ? LOG2N : 4;
    using Core = FftCore<T, LOG2N, LOG2E>;
    using L = SmemLayout<LOG2N, LOG2E, 1, false, int(sizeof(cx<T>))>;
    constexpr int N = Core::N, E = Core::E, TPL = Core::TPL;
    std::vector<cx<T>> regs(size_t(TPL) * E), smem(L::ELEMS);
    auto ext = [&](int i) {
        bool neg;
        const int m = r2r1_ext(i, N, dst, neg);
        return m < 0 ? T(0) : (neg ? -x[m] : x[m]);
    };
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) {
            const int m = j + e * TPL;
            regs[size_t(j) * E + e] = cx<T>{ext(2 * m), ext(2 * m + 1)};
        }
    RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) smem[L::idx(j + e * TPL, 0)] = regs[size_t(j) * E + Core::final_slot(e)];
    y.assign(x.size(), T(-7));  // every output is written once
    auto store = [&](int k, cx<T> ek) {
        const int o = r2r1_out_index(k, N, dst);
        if (o >= 0) y[o] = r2r1_value<T>(ek, dst);
    };
    for (int k = 0; k <= N / 2; ++k) {  // the kernel's emit(k): k < N/2 over the threads, then N/2
        cx<T> ek, enk;
        r2r1_split<T>(smem[L::idx(k, 0)], smem[L::idx((N - k) & (N - 1), 0)], w[k], ek, enk);
        store(k, ek);
        if (2 * k != N) store(N - k, enk);
    }
}

template <typename T, int LOG2N = 1>
void dispatch(int lg, const std::vector<T>& x, std::vector<T>& y, const std::vector<cx<T>>& tw, const std::vector<cx<T>>& w, int dst) {
    if (lg == LOG2N) r2r1_line<T, LOG2N>(x, y, tw, w, dst);
    else if constexpr (LOG2N < 13) dispatch<T, LOG2N + 1>(lg, x, y, tw, w, dst);
    else abort();
}

// naive long-double DCT-I / DST-I (scipy type=1 norm=None, FFTW REDFT00 / RODFT00); c[i] = cos(pi i / N), s[i] = sin(pi i / N)
// for i < 2N
static long double naive(const std::vector<long double>& x, int k, int N, int dst, const std::vector<long double>& c,
                         const std::vector<long double>& s) {
    long double r = 0;
    if (!dst) {
        r = x[0] + ((k & 1) ? -x[N] : x[N]);
        for (int n = 1; n < N; ++n) r += 2 * x[n] * c[(long long)n * k % (2 * N)];
    } else {
        for (int n = 0; n <= N - 2; ++n) r += 2 * x[n] * s[(long long)(n + 1) * (k + 1) % (2 * N)];
    }
    return r;
}

template <typename T>
double check(int lg, int dst, bool* zero_ok) {
    const int N = 1 << lg, L = dst ? N - 1 : N + 1;
    std::vector<cx<T>> tw(N), w(N / 2 + 1);
    for (int m = 0; m < N; ++m) {
        const long double ang = -2.0L * M_PIl * m / N;
        tw[m] = cx<T>{T(cosl(ang)), T(sinl(ang))};
    }
    for (int k = 0; k <= N / 2; ++k) {  // the host table of the plans: Tables::get_tw2(log2 N) = make_table(N/2 + 1, 2N)
        const long double ang = -2.0L * M_PIl * k / (2.0L * N);
        w[k] = cx<T>{T(cosl(ang)), T(sinl(ang))};
    }
    std::vector<long double> c(2 * N), s(2 * N);
    for (int i = 0; i < 2 * N; ++i) {
        c[i] = cosl(M_PIl * i / N);
        s[i] = sinl(M_PIl * i / N);
    }
    std::vector<T> x(L), y;
    srand(4321 + 7 * lg + dst);
    for (int n = 0; n < L; ++n) x[n] = T(rand() / double(RAND_MAX) - 0.5);
    dispatch<T>(lg, x, y, tw, w, dst);
    const std::vector<long double> xl(x.begin(), x.end());
    long double num = 0, den = 0;
    for (int k = 0; k < L; ++k) {
        const long double r = naive(xl, k, N, dst, c, s);
        num += (y[k] - r) * (y[k] - r);
        den += r * r;
    }
    // a zero line gives exact zeros
    std::vector<T> z(L, T(0)), yz;
    dispatch<T>(lg, z, yz, tw, w, dst);
    for (int k = 0; k < L; ++k)
        if (yz[k] != T(0)) *zero_ok = false;
    return double(sqrtl(num / den));
}

int main() {
    int fails = 0, cases = 0;
    double worst64 = 0, worst32 = 0;
    static char b64[64] = "", b32[64] = "";
    for (int lg = 1; lg <= 13; ++lg)
        for (int dst = 0; dst < 2; ++dst) {
            if (dst && lg < 2) continue;  // DST-I: N >= 4
            bool zero_ok = true;
            const double e64 = check<double>(lg, dst, &zero_ok), e32 = check<float>(lg, dst, &zero_ok);
            ++cases;
            const int L = dst ? (1 << lg) - 1 : (1 << lg) + 1;
            if (e64 > worst64) { worst64 = e64; snprintf(b64, sizeof b64, "L=%d %s", L, dst ? "DST-I" : "DCT-I"); }
            if (e32 > worst32) { worst32 = e32; snprintf(b32, sizeof b32, "L=%d %s", L, dst ? "DST-I" : "DCT-I"); }
            if (!(e64 <= 1e-14) || !(e32 <= 1e-5) || !zero_ok) {
                printf("L=%d %s f64 relL2=%.3e f32 relL2=%.3e zero line %s FAIL\n", L, dst ? "DST-I" : "DCT-I", e64, e32, zero_ok ? "ok" : "NONZERO");
                ++fails;
            }
        }
    printf("cases=%d worst f64 relL2=%.3e (%s) worst f32 relL2=%.3e (%s)\n", cases, worst64, b64, worst32, b32);
    printf("fails=%d\n", fails);
    return fails ? 1 : 0;
}
