// CPU emulation of the R2HC / HC2R pass (fft_r2hc_kernel): runs its per-line steps — two real lines packed as z = a + i b
// in natural order, fft_core.cuh's stage arithmetic "one thread at a time" with the kernels' shared-memory layout, the
// separation through Z[-k mod N], and the inverse build from hc[k] and hc[N-k] — through the helpers of r2r.hpp, and checks
// both lines against a naive long-double R2HC / HC2R (FFTW's halfcomplex format) for every N = 2..8192, both directions,
// f64 and f32, and once more with a zero partner line (an odd line count).  Built and run by tests/test_r2r_mixed.py (no
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

// The kernel's steps on the line pair (a, b); has_b = false: b is a zero partner whose results are dropped.
template <typename T, int LOG2N>
void r2hc_pair(const std::vector<T>& a, const std::vector<T>& b, bool has_b, std::vector<T>& ya, std::vector<T>& yb, const std::vector<cx<T>>& tw,
               bool inverse) {
    constexpr int LOG2E = LOG2N < 4 ? LOG2N : 4;
    using Core = FftCore<T, LOG2N, LOG2E>;
    using L = SmemLayout<LOG2N, LOG2E, 1, false, int(sizeof(cx<T>))>;
    constexpr int N = Core::N, E = Core::E, TPL = Core::TPL;
    std::vector<cx<T>> regs(size_t(TPL) * E), smem(L::ELEMS);
    auto ld = [&](int m, T& va, T& vb) { va = a[m]; vb = has_b ? b[m] : T(0); };
    ya.assign(N, T(0));
    yb.assign(N, T(0));
    if (!inverse) {
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) {
                T va, vb;
                ld(j + e * TPL, va, vb);
                regs[size_t(j) * E + e] = cx<T>{va, vb};
            }
        RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) smem[L::idx(j + e * TPL, 0)] = regs[size_t(j) * E + Core::final_slot(e)];
        for (int k = 0; k < N; ++k) {
            const cx<T> x = r2hc_split<T>(smem[L::idx(k, 0)], smem[L::idx((N - k) & (N - 1), 0)], k, N);
            ya[k] = x.x;
            if (has_b) yb[k] = x.y;
        }
    } else {
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) {
                const int k = j + e * TPL, nk = r2hc_in_nk(k, N);
                T ak, bk, am = T(0), bm = T(0);
                ld(k, ak, bk);
                if (nk >= 0) ld(nk, am, bm);
                regs[size_t(j) * E + e] = cswap(r2hc_build<T>(ak, am, bk, bm, k, N));
            }
        RunStages<T, LOG2N, LOG2E, 0>::run(regs, smem, tw.data());
        for (int j = 0; j < TPL; ++j)
            for (int e = 0; e < E; ++e) {
                const cx<T> z = cswap(regs[size_t(j) * E + Core::final_slot(e)]);
                ya[j + e * TPL] = z.x;
                if (has_b) yb[j + e * TPL] = z.y;
            }
    }
}

template <typename T, int LOG2N = 1>
void dispatch(int lg, const std::vector<T>& a, const std::vector<T>& b, bool has_b, std::vector<T>& ya, std::vector<T>& yb,
              const std::vector<cx<T>>& tw, bool inverse) {
    if (lg == LOG2N) r2hc_pair<T, LOG2N>(a, b, has_b, ya, yb, tw, inverse);
    else if constexpr (LOG2N < 13) dispatch<T, LOG2N + 1>(lg, a, b, has_b, ya, yb, tw, inverse);
    else abort();
}

// naive long-double R2HC / HC2R (FFTW_R2HC / FFTW_HC2R, unnormalised); c[i] = cos(2 pi i / N), s[i] = sin(2 pi i / N)
static long double naive(const std::vector<long double>& x, int k, bool inverse, const std::vector<long double>& c,
                         const std::vector<long double>& s) {
    const int N = int(x.size());
    long double r = 0;
    if (!inverse) {  // hc[k] = Re X[k] (k <= N/2), hc[k] = Im X[N-k] (k > N/2), X[k] = sum x_n exp(-2 pi i k n / N)
        const bool re = 2 * k <= N;
        const long long kk = re ? k : N - k;
        for (int n = 0; n < N; ++n) r += re ? x[n] * c[(kk * n) % N] : -x[n] * s[(kk * n) % N];
    } else {  // y_n = hc[0] + (-1)^n hc[N/2] + 2 sum_{0<j<N/2} (hc[j] cos(2 pi j n / N) - hc[N-j] sin(2 pi j n / N))
        r = x[0];
        if (N > 1) r += ((k & 1) ? -1 : 1) * x[N / 2];
        for (int j = 1; 2 * j < N; ++j) r += 2 * (x[j] * c[((long long)j * k) % N] - x[N - j] * s[((long long)j * k) % N]);
    }
    return r;
}

template <typename T>
double check(int lg, bool inverse, bool lone) {
    const int N = 1 << lg;
    std::vector<cx<T>> tw(N);
    for (int m = 0; m < N; ++m) {
        long double ang = -2.0L * M_PIl * m / N;
        tw[m] = cx<T>{T(cosl(ang)), T(sinl(ang))};
    }
    std::vector<long double> c(N), s(N);
    for (int i = 0; i < N; ++i) { c[i] = cosl(2.0L * M_PIl * i / N); s[i] = sinl(2.0L * M_PIl * i / N); }
    std::vector<T> a(N), b(N), ya, yb;
    srand(4321 + 7 * lg + (inverse ? 1 : 0));
    for (int n = 0; n < N; ++n) {
        a[n] = T(rand() / double(RAND_MAX) - 0.5);
        b[n] = T(rand() / double(RAND_MAX) - 0.5);
    }
    dispatch<T>(lg, a, b, !lone, ya, yb, tw, inverse);
    long double num = 0, den = 0;
    for (int line = 0; line < (lone ? 1 : 2); ++line) {
        const std::vector<T>& x = line ? b : a;
        const std::vector<T>& y = line ? yb : ya;
        std::vector<long double> xl(x.begin(), x.end());
        for (int k = 0; k < N; ++k) {
            const long double r = naive(xl, k, inverse, c, s);
            num += (y[k] - r) * (y[k] - r);
            den += r * r;
        }
    }
    // a zero partner stores nothing
    if (lone)
        for (int k = 0; k < N; ++k)
            if (yb[k] != T(0)) return 1.0;
    return double(sqrtl(num / den));
}

int main() {
    int fails = 0, cases = 0;
    double worst64 = 0, worst32 = 0;
    const char* at64 = "";
    const char* at32 = "";
    static char b64[64], b32[64];
    for (int lg = 1; lg <= 13; ++lg)
        for (int inv = 0; inv < 2; ++inv)
            for (int lone = 0; lone < 2; ++lone) {
                const double e64 = check<double>(lg, inv, lone), e32 = check<float>(lg, inv, lone);
                ++cases;
                if (e64 > worst64) { worst64 = e64; snprintf(b64, sizeof b64, "N=%d %s", 1 << lg, inv ? "HC2R" : "R2HC"); at64 = b64; }
                if (e32 > worst32) { worst32 = e32; snprintf(b32, sizeof b32, "N=%d %s", 1 << lg, inv ? "HC2R" : "R2HC"); at32 = b32; }
                if (!(e64 <= 1e-10) || !(e32 <= 1e-5)) {
                    printf("N=%d %s%s f64 relL2=%.3e f32 relL2=%.3e FAIL\n", 1 << lg, inv ? "HC2R" : "R2HC", lone ? " (zero partner)" : "", e64, e32);
                    ++fails;
                }
            }
    printf("cases=%d worst f64 relL2=%.3e (%s) worst f32 relL2=%.3e (%s)\n", cases, worst64, at64, worst32, at32);
    printf("fails=%d\n", fails);
    return fails ? 1 : 0;
}
