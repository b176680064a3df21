// CPU emulation of the Bluestein pass (fft_bluestein_kernel): runs its per-line steps through fft_core.cuh's stage
// arithmetic "one thread at a time", with the host tables of bluestein.hpp, and checks it against a naive long-double DFT
// in both directions, f64 and f32.  Built and run by tests/test_bluestein.py (no GPU needed).  Prints the worst rel-L2
// error per precision; exit code 0 = every length passes.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../distributedfft_b200/csrc/bluestein.hpp"

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

// The kernel's steps on one line of n points, M = 2^LOG2M.
template <typename T, int LOG2M>
void bluestein_line(const std::vector<cx<T>>& x, std::vector<cx<T>>& out, const std::vector<cx<T>>& table, const std::vector<cx<T>>& tw,
                    bool inverse) {
    constexpr int LOG2E = LOG2M < 4 ? LOG2M : 4;
    using Core = FftCore<T, LOG2M, LOG2E>;
    using L = SmemLayout<LOG2M, LOG2E, 1, false, int(sizeof(cx<T>))>;
    constexpr int M = Core::N, E = Core::E, TPL = Core::TPL;
    const int n = int(x.size());
    const cx<T>* kspec = table.data();
    const cx<T>* chirp = table.data() + M;
    std::vector<cx<T>> regs(size_t(TPL) * E), z(size_t(TPL) * E), smem(L::ELEMS);
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            regs[size_t(j) * E + e] = k < n ? cmul(inverse ? cswap(x[k]) : x[k], chirp[k]) : cx<T>{T(0), T(0)};
        }
    RunStages<T, LOG2M, LOG2E, 0>::run(regs, smem, tw.data());
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) z[size_t(j) * E + e] = cswap(cmul(regs[size_t(j) * E + Core::final_slot(e)], kspec[j + e * TPL]));
    RunStages<T, LOG2M, LOG2E, 0>::run(z, smem, tw.data());
    out.assign(n, cx<T>{T(0), T(0)});
    for (int j = 0; j < TPL; ++j)
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            if (k >= n) continue;
            const cx<T> r = cmul(chirp[k], cswap(z[size_t(j) * E + Core::final_slot(e)]));
            out[k] = inverse ? cswap(r) : r;
        }
}

template <typename T, int LOG2M = 3>
void dispatch(int lg, const std::vector<cx<T>>& x, std::vector<cx<T>>& out, const std::vector<cx<T>>& table, const std::vector<cx<T>>& tw,
              bool inverse) {
    if (lg == LOG2M) bluestein_line<T, LOG2M>(x, out, table, tw, inverse);
    else if constexpr (LOG2M < 13) dispatch<T, LOG2M + 1>(lg, x, out, table, tw, inverse);
    else abort();
}

template <typename T>
double check(int n, bool inverse) {
    const int lg = bluestein_log2m(size_t(n));
    const int M = 1 << lg;
    std::vector<cx<T>> tw(M);
    for (int m = 0; m < M; ++m) {
        long double a = -2.0L * M_PIl * m / M;
        tw[m] = cx<T>{T(cosl(a)), T(sinl(a))};
    }
    const std::vector<cx<T>> table = bluestein_table<T>(size_t(n));
    std::vector<cx<T>> x(n), out;
    srand(777 + n);
    for (auto& c : x) c = cx<T>{T(rand() / double(RAND_MAX) - 0.5), T(rand() / double(RAND_MAX) - 0.5)};
    dispatch<T>(lg, x, out, table, tw, inverse);
    std::vector<long double> ct(n), st(n);
    for (int m = 0; m < n; ++m) {
        long double a = 2.0L * M_PIl * m / n;
        ct[m] = cosl(a);
        st[m] = (inverse ? 1.0L : -1.0L) * sinl(a);
    }
    long double num = 0, den = 0;
    for (int k = 0; k < n; ++k) {
        long double sr = 0, si = 0;
        for (int m = 0; m < n; ++m) {
            const int idx = int((long long)k * m % n);
            sr += x[m].x * ct[idx] - x[m].y * st[idx];
            si += x[m].x * st[idx] + x[m].y * ct[idx];
        }
        num += (out[k].x - sr) * (out[k].x - sr) + (out[k].y - si) * (out[k].y - si);
        den += sr * sr + si * si;
    }
    return double(sqrtl(num / den));
}

int main() {
    std::vector<int> lengths;
    for (int n = 3; n <= 300; ++n) lengths.push_back(n);
    for (int n : {1000, 2047, 2049, 3000, 4093, 4095}) lengths.push_back(n);
    int fails = 0;
    double worst64 = 0, worst32 = 0;
    int at64 = 0, at32 = 0;
    for (int n : lengths)
        for (int inv = 0; inv < 2; ++inv) {
            const double e64 = check<double>(n, inv), e32 = check<float>(n, inv);
            if (e64 > worst64) { worst64 = e64; at64 = n; }
            if (e32 > worst32) { worst32 = e32; at32 = n; }
            if (!(e64 < 1e-10) || !(e32 < 1e-5)) {
                printf("n=%d %s f64 relL2=%.3e f32 relL2=%.3e FAIL\n", n, inv ? "inv" : "fwd", e64, e32);
                ++fails;
            }
        }
    printf("lengths=%zu worst f64 relL2=%.3e (n=%d) worst f32 relL2=%.3e (n=%d)\n", lengths.size(), worst64, at64, worst32, at32);
    printf("fails=%d\n", fails);
    return fails ? 1 : 0;
}
