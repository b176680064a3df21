// dfft_plan.cu — plan construction, step schedule and execution behind include/dfft.h.
//
// A plan is a short list of steps — FFT passes (fft_kernels.cuh), device rendezvous kernels and NCCL
// all-to-all-v exchanges — built once from the partition geometry, replayed by every exec:
//
//   reference call                                              here
//   ------------------------------------------------------------------------------------------------
//   cufftExecR2C/D2Z 2D (y,z)   mpicufft_slab.cpp:788           R2C z pass + C2C y pass (scattering)
//   pack memcpy2D + Alltoallv   mpicufft_slab.cpp:646-661       fused into the y pass' stores (Peer2Peer)
//                                                               or send slots + ncclSend/Recv (All2All)
//   cufftExecZ2Z 1D x           mpicufft_slab.cpp:806           C2C x pass (gathering)
//   pencil transposes 1 and 2   mpicufft_pencil.cpp:858-930,    same mechanism, row / column groups
//                               1490-1576
//
// Peer2Peer: every rank maps the other ranks' work slots with CUDA IPC; an FFT pass writes its output
// rows straight into the layout the receiver's next pass reads (NVLink stores), and ranks meet at tiny
// flag kernels (st.release.sys / ld.acquire.sys on peer-mapped flags) instead of MPI_Waitall.
#include <cuda_runtime.h>
#include <nccl.h>

#include <sys/stat.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <fstream>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "../../include/dfft.h"
#include "bluestein.hpp"
#include "fft_kernels.cuh"
#include "geometry.hpp"

namespace dfft {

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}
#define CK_CUDA(x)                                                                                     \
    do {                                                                                               \
        cudaError_t e_ = (x);                                                                          \
        if (e_ != cudaSuccess)                                                                         \
            return fail(DFFT_ERR_CUDA, std::string(#x) + ": " + cudaGetErrorString(e_) + " (" + __FILE__ + ":" + \
                                           std::to_string(__LINE__) + ")");                            \
    } while (0)
#define CK_NCCL(x)                                                                                     \
    do {                                                                                               \
        ncclResult_t r_ = (x);                                                                         \
        if (r_ != ncclSuccess)                                                                         \
            return fail(DFFT_ERR_NCCL, std::string(#x) + ": " + ncclGetErrorString(r_) + " (" + __FILE__ + ":" + \
                                           std::to_string(__LINE__) + ")");                            \
    } while (0)

static int ilog2_exact(size_t n) {
    if (n == 0 || (n & (n - 1))) return -1;
    int l = 0;
    while ((size_t(1) << l) < n) ++l;
    return l;
}

// ---- twiddle tables ---------------------------------------------------------------------------------
template <typename T>
static cudaError_t make_table(size_t count, size_t denom, void** dev) {
    std::vector<cx<T>> h(count);
    for (size_t m = 0; m < count; ++m) {
        // exact symmetric evaluation in long double
        long double a = -2.0L * 3.14159265358979323846264338327950288L * (long double)m / (long double)denom;
        h[m] = cx<T>{T(cosl(a)), T(sinl(a))};
    }
    cudaError_t e = cudaMalloc(dev, count * sizeof(cx<T>));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*dev, h.data(), count * sizeof(cx<T>), cudaMemcpyHostToDevice);
}

// Type-IV table of N-point real lines: one allocation [p_m (N/2 entries)][q_k (N/2 entries)] (r2r.hpp)
template <typename T>
static cudaError_t make_r2r4_table(int n, void** dev) {
    const std::vector<cx<T>> h = r2r4_table<T>(n);
    cudaError_t e = cudaMalloc(dev, h.size() * sizeof(cx<T>));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*dev, h.data(), h.size() * sizeof(cx<T>), cudaMemcpyHostToDevice);
}

// Twiddle table of 1D plans of N = 2^log2n points (FftPadded::tw1d, DESIGN.md section 3.22): one allocation
// [W_N^l, l < 2^lo][W_N^(h 2^lo), h < N / 2^lo], lo = ceil(log2n / 2), about 2 sqrt(N) entries.  Each entry is evaluated in
// long double from an exact integer numerator and rounded once; a pass multiplies one entry of each half, W_N^m =
// W_N^(m_hi 2^lo) W_N^(m_lo), m = m_hi 2^lo + m_lo reduced mod N in 64-bit integers.
static int tw1d_lo_bits(int log2n) { return (log2n + 1) / 2; }
template <typename T>
static cudaError_t make_tw1d_table(int log2n, void** dev) {
    const int lo = tw1d_lo_bits(log2n);
    const size_t nlo = size_t(1) << lo, nhi = size_t(1) << (log2n - lo);
    std::vector<cx<T>> h(nlo + nhi);
    const long double two_pi = 2.0L * 3.14159265358979323846264338327950288L;
    for (size_t l = 0; l < nlo; ++l) {
        const long double a = -two_pi * (long double)l / (long double)(1ull << log2n);
        h[l] = cx<T>{T(cosl(a)), T(sinl(a))};
    }
    for (size_t k = 0; k < nhi; ++k) {
        const long double a = -two_pi * (long double)k / (long double)nhi;
        h[nlo + k] = cx<T>{T(cosl(a)), T(sinl(a))};
    }
    cudaError_t e = cudaMalloc(dev, h.size() * sizeof(cx<T>));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*dev, h.data(), h.size() * sizeof(cx<T>), cudaMemcpyHostToDevice);
}

// Bluestein table of n-point lines: one allocation [K^ (M entries)][chirp (n entries)] (bluestein.hpp)
template <typename T>
static cudaError_t make_bluestein_table(size_t n, void** dev) {
    const std::vector<cx<T>> h = bluestein_table<T>(n);
    cudaError_t e = cudaMalloc(dev, h.size() * sizeof(cx<T>));
    if (e != cudaSuccess) return e;
    return cudaMemcpy(*dev, h.data(), h.size() * sizeof(cx<T>), cudaMemcpyHostToDevice);
}

// Lengths of C2C axes: powers of two in [2, 2^MAX_LOG2N] (the power-of-two kernels) and any length in [3, BLUESTEIN_MAX_N]
// (the Bluestein pass)
static bool bluestein_length(size_t n) { return ilog2_exact(n) < 0 && n >= 3 && n <= size_t(BLUESTEIN_MAX_N); }
static bool pow2_length(size_t n) { return ilog2_exact(n) >= 1 && ilog2_exact(n) <= MAX_LOG2N; }
static bool c2c_length(size_t n) { return pow2_length(n) || bluestein_length(n); }
// Real-to-real plans: powers of two in [2, 2^MAX_LOG2N].  The transform of a plan from dfft_plan_create_r2r is DFFT_DCT or
// DFFT_DST when all three kinds are that one, DFFT_R2HC for any other combination (its kinds are in dfft_plan_s::kinds).
static bool is_r2r(int transform) { return transform == DFFT_DCT || transform == DFFT_DST || transform == DFFT_R2HC; }
static const char* r2r_name(int k) {
    return k == DFFT_DST    ? "dst"
           : k == DFFT_R2HC ? "r2hc"
           : k == DFFT_DCT1 ? "dct1"
           : k == DFFT_DST1 ? "dst1"
           : k == DFFT_DCT4 ? "dct4"
           : k == DFFT_DST4 ? "dst4"
                            : "dct";
}
static bool r2r_length(size_t n) { return ilog2_exact(n) >= 1 && ilog2_exact(n) <= MAX_LOG2N; }
// Type-I kinds (DFFT_DCT1, DFFT_DST1): axis kinds of per-axis plans (transform DFFT_R2HC) and of dfft_fft1d_r2r only.  An
// axis of L points runs N-point complex lines: L = N + 1 (DCT-I, N in [2, 8192]) or L = N - 1 (DST-I, N in [4, 8192]).
static bool is_type1(int kind) { return kind == DFFT_DCT1 || kind == DFFT_DST1; }
// Type-IV kinds (DFFT_DCT4, DFFT_DST4): axis kinds like type I, of N points, N a power of two in [4, 8192]; a pass runs
// N/2-point complex lines
static bool is_type4(int kind) { return kind == DFFT_DCT4 || kind == DFFT_DST4; }
static bool is_r2r_kind(int kind) { return is_r2r(kind) || is_type1(kind) || is_type4(kind); }
// log2 N of a type-I axis of L points, -1 for a length the kind does not take
static int type1_log2(int kind, size_t L) {
    const int l2 = kind == DFFT_DCT1 ? (L >= 3 ? ilog2_exact(L - 1) : -1) : ilog2_exact(L + 1);
    return l2 >= (kind == DFFT_DCT1 ? 1 : 2) && l2 <= MAX_LOG2N ? l2 : -1;
}
// the lengths an axis of R2R kind `kind` takes
static bool r2r_kind_length(int kind, size_t n) {
    return is_type1(kind) ? type1_log2(kind, n) > 0 : is_type4(kind) ? n >= 4 && r2r_length(n) : r2r_length(n);
}

// One FFT pass of n-point lines (R2C / C2R: n complex points) over the views of prm, its stores scaled by `scale`: the
// power-of-two kernels, or the Bluestein pass when n is not a power of two (prm.tw: the M-point table; blu: the Bluestein
// table of n).  PASS_R2R_*: the R2R kernel of kind r2r (DFFT_DCT, DFFT_DST with prm.tw2 its w_k table, or DFFT_R2HC), or
// the type-I kernel (DFFT_DCT1, DFFT_DST1: n = N +- 1 reals, prm.tw2 the 2N-point table), or the type-IV kernel
// (DFFT_DCT4, DFFT_DST4: n reals through n/2-point lines, prm.tw2 the type-IV table).
// hole: passes of padded and pruned plans that keep part of a side, the holes of their lines (pass_hole): [hole[0],
// hole[1]) on the spectral side, [hole[2], hole[3]) on the physical one; the padded twin of the power-of-two kernel runs
// then, with the physical hole on its loaded side forward and on its stored side inverse.
// w: the spectral weights of the pass's axis (dfft_plan_set_weights), or null.  Weighted passes run the weighted twins:
// of the padded kernels (with hole, empty where the plan keeps a whole side) or of the Bluestein kernel (WEIGHTED = true).
// tw: the twiddle of a pass of a 1D plan (Twiddle1d), or null.  Twiddled passes run the twiddled twin of the padded C2C
// kernel (TWIDDLED = true), with empty holes.
struct Twiddle1d {
    const void* table;              // make_tw1d_table of log2n
    long long line0, c1, mul;       // FftPadded::tw_line0, tw_c1, tw_mul
    int log2n;                      // N = 2^log2n, the signal's length
    long long sB = 0;               // FftPadded::tw_sB: the transposing z pass of natural-order plans; 0 for the others
};
static cudaError_t launch_fft_pass(int prec, PassKind kind, size_t n, const FftParams& prm, const void* blu, double scale, cudaStream_t stream,
                                   int r2r = DFFT_DCT, const int* hole = nullptr, const void* w = nullptr, const Twiddle1d* tw = nullptr) {
    const int log2n = ilog2_exact(n);
    if (hole && log2n >= 0) {
        FftPadded q;
        static_cast<FftParams&>(q) = prm;
        q.scale = scale;
        const int* ld = prm.inverse ? hole : hole + 2;
        const int* st = prm.inverse ? hole + 2 : hole;
        q.ld_lo = ld[0]; q.ld_hi = ld[1];
        q.st_lo = st[0]; q.st_hi = st[1];
        q.w = w;
        q.tw1d = tw ? tw->table : nullptr;
        q.tw_line0 = tw ? tw->line0 : 0;
        q.tw_c1 = tw ? tw->c1 : 0;
        q.tw_mul = tw ? tw->mul : 0;
        q.tw_log2n = tw ? tw->log2n : 0;
        q.tw_lo_bits = tw ? tw1d_lo_bits(tw->log2n) : 0;
        q.tw_sB = tw ? tw->sB : 0;
        return launch_twin(prec, log2n, kind, q, stream);
    }
    if (kind == PASS_R2R_CONTIG || kind == PASS_R2R_TILED) {
        FftR2r r;
        static_cast<FftParams&>(r) = prm;
        r.w = prm.tw2;
        r.dst = r2r == DFFT_DST || r2r == DFFT_DST1 || r2r == DFFT_DST4;
        r.scale = scale;
        if (is_type1(r2r)) return launch_r2r1(prec, type1_log2(r2r, n), kind, r, stream);
        if (is_type4(r2r)) return launch_r2r4(prec, log2n - 1, kind, r, stream);
        return launch_r2r(prec, log2n, kind, r, r2r == DFFT_R2HC, stream);
    }
    if (log2n >= 0) return launch_pass(prec, log2n, kind, prm, scale, stream);
    const int log2m = bluestein_log2m(n);
    FftBluestein b;
    static_cast<FftParams&>(b) = prm;
    b.n = int(n);
    b.kspec = blu;
    b.chirp = blu ? static_cast<const char*>(blu) + (size_t(1) << log2m) * (prec == DFFT_F64 ? 16 : 8) : nullptr;
    b.scale = scale;
    b.w = w;
    return launch_bluestein(prec, log2m, kind, b, stream);
}

// The holes of a pass of n-point lines (R2C / C2R: n complex points, n + 1 spectral ones) that keeps `keep` points of its
// spectral side and `data` points of its physical side (0: all of them).  Spectral, C2C: frequencies 0 .. ceil(K/2) - 1
// and the K - ceil(K/2) negative ones, at the end of the line (numpy's fftfreq(K) * K mod N); R2C / C2R: k = 0 .. keep - 1.
// Physical: positions 0 .. data - 1; R2C / C2R: data reals, the pairs 0 .. data/2 - 1.  hole[0..1] spectral, hole[2..3]
// physical, each empty when lo == hi.
static void pass_hole(PassKind kind, size_t n, size_t keep, size_t data, int hole[4]) {
    const bool half = kind == PASS_R2C || kind == PASS_C2R;
    const size_t full = half ? n + 1 : n, k = keep ? keep : full;
    hole[0] = int(half ? k : (k + 1) / 2);
    hole[1] = int(hole[0] + full - k);
    hole[2] = int(data ? (half ? data / 2 : data) : n);
    hole[3] = int(n);
}

// 16-bit plans (DFFT_F16, DFFT_BF16; DESIGN.md section 3.20): 4-byte complex elements, f32 arithmetic, the sequential schedule
static bool is_half(int prec) { return prec == DFFT_F16 || prec == DFFT_BF16; }
static int refuse_half(const std::string& what) { return fail(DFFT_ERR_UNSUPPORTED, what + " have no 16-bit storage (DFFT_F16 / DFFT_BF16)"); }

// Passes over an axis the plan keeps (dfft_plan_set_transform_axes): the views of the FFT pass they replace, no transform
static bool is_copy(PassKind kind) { return kind == PASS_COPY_CONTIG || kind == PASS_COPY_TILED; }
// one copy pass of n-point lines over the views of prm; real: the real elements of R2R plans
static cudaError_t launch_copy_pass(int prec, bool real, PassKind kind, size_t n, const FftParams& prm, double scale, cudaStream_t stream) {
    FftCopy c;
    static_cast<FftParams&>(c) = prm;
    c.n = int(n);
    c.ltpl = 0;
    c.scale = scale;
    return launch_copy(prec, real, kind, c, stream);
}

struct Tables {
    int prec = DFFT_F64;
    bool dry = false;  // geometry-only plans: no device allocations, segment tables live on the host
    std::map<const void*, std::vector<unsigned char>> host_tabs;  // segment table pointer -> host copy
    std::vector<std::vector<unsigned char>*> dry_store;
    std::map<int, void*> tw;   // log2n -> exp(-2 pi i m / n), m < n
    std::map<int, void*> tw2;  // log2m -> exp(-2 pi i k / 2m), k <= m/2
    std::map<size_t, void*> blu;  // n -> Bluestein table of n-point lines
    std::map<int, void*> r2r4;    // log2 N -> type-IV table of N-point real lines (r2r4_table)
    std::map<int, void*> tw1d;    // log2 N -> twiddle table of 1D plans of N points (make_tw1d_table)
    std::vector<void*> bytes;  // seg_of_n tables
    cudaError_t get_tw(int log2n, void** out) {
        if (dry) { *out = nullptr; return cudaSuccess; }
        auto it = tw.find(log2n);
        if (it == tw.end()) {
            void* d = nullptr;
            size_t n = size_t(1) << log2n;
            cudaError_t e = prec == DFFT_F64 ? make_table<double>(n, n, &d) : make_table<float>(n, n, &d);
            if (e != cudaSuccess) return e;
            it = tw.emplace(log2n, d).first;
        }
        *out = it->second;
        return cudaSuccess;
    }
    cudaError_t get_tw2(int log2m, void** out) {
        if (dry) { *out = nullptr; return cudaSuccess; }
        auto it = tw2.find(log2m);
        if (it == tw2.end()) {
            void* d = nullptr;
            size_t m = size_t(1) << log2m;
            cudaError_t e = prec == DFFT_F64 ? make_table<double>(m / 2 + 1, 2 * m, &d) : make_table<float>(m / 2 + 1, 2 * m, &d);
            if (e != cudaSuccess) return e;
            it = tw2.emplace(log2m, d).first;
        }
        *out = it->second;
        return cudaSuccess;
    }
    cudaError_t get_blu(size_t n, void** out) {
        if (dry) { *out = nullptr; return cudaSuccess; }
        auto it = blu.find(n);
        if (it == blu.end()) {
            void* d = nullptr;
            cudaError_t e = prec == DFFT_F64 ? make_bluestein_table<double>(n, &d) : make_bluestein_table<float>(n, &d);
            if (e != cudaSuccess) return e;
            it = blu.emplace(n, d).first;
        }
        *out = it->second;
        return cudaSuccess;
    }
    cudaError_t get_r2r4(int log2n, void** out) {
        if (dry) { *out = nullptr; return cudaSuccess; }
        auto it = r2r4.find(log2n);
        if (it == r2r4.end()) {
            void* d = nullptr;
            const int n = 1 << log2n;
            cudaError_t e = prec == DFFT_F64 ? make_r2r4_table<double>(n, &d) : make_r2r4_table<float>(n, &d);
            if (e != cudaSuccess) return e;
            it = r2r4.emplace(log2n, d).first;
        }
        *out = it->second;
        return cudaSuccess;
    }
    cudaError_t get_tw1d(int log2n, void** out) {
        if (dry) { *out = nullptr; return cudaSuccess; }
        auto it = tw1d.find(log2n);
        if (it == tw1d.end()) {
            void* d = nullptr;
            cudaError_t e = prec == DFFT_F64 ? make_tw1d_table<double>(log2n, &d) : make_tw1d_table<float>(log2n, &d);
            if (e != cudaSuccess) return e;
            it = tw1d.emplace(log2n, d).first;
        }
        *out = it->second;
        return cudaSuccess;
    }
    cudaError_t seg_table(const Split& s, const unsigned char** out) {
        size_t n = s.start.back() + s.size.back();
        std::vector<unsigned char> h(n);
        for (size_t p = 0; p < s.size.size(); ++p)
            for (size_t k = 0; k < s.size[p]; ++k) h[s.start[p] + k] = (unsigned char)p;
        if (dry) {
            auto* keep = new std::vector<unsigned char>(h);
            dry_store.push_back(keep);
            host_tabs[keep->data()] = h;
            *out = keep->data();
            return cudaSuccess;
        }
        void* d = nullptr;
        cudaError_t e = cudaMalloc(&d, n ? n : 1);
        if (e != cudaSuccess) return e;
        e = cudaMemcpy(d, h.data(), n, cudaMemcpyHostToDevice);
        bytes.push_back(d);
        host_tabs[d] = h;
        *out = (const unsigned char*)d;
        return e;
    }
    // segment tables belong to the schedules: dropped whenever the schedules are rebuilt (dfft_set_work_area)
    void release_seg_tables() {
        for (void* p : bytes) cudaFree(p);
        for (auto* v : dry_store) delete v;
        bytes.clear(); dry_store.clear(); host_tabs.clear();
    }
    void release() {
        for (auto& kv : tw) cudaFree(kv.second);
        for (auto& kv : tw2) cudaFree(kv.second);
        for (auto& kv : blu) cudaFree(kv.second);
        for (auto& kv : r2r4) cudaFree(kv.second);
        for (auto& kv : tw1d) cudaFree(kv.second);
        for (void* p : bytes) cudaFree(p);
        for (auto* v : dry_store) delete v;
        tw.clear(); tw2.clear(); blu.clear(); r2r4.clear(); tw1d.clear(); bytes.clear(); dry_store.clear(); host_tabs.clear();
    }
};

// The power-of-two length a pass of n-point lines runs (R2C / C2R: n complex points): log2 n, or log2 M of the Bluestein
// pass for C2C lengths that are not powers of two, log2 N of type-I R2R passes (r2r: the kind of R2R passes); -1 for lengths
// nothing runs
static int pass_log2(PassKind kind, size_t n, int r2r = 0) {
    if ((kind == PASS_R2R_CONTIG || kind == PASS_R2R_TILED) && is_type1(r2r)) return type1_log2(r2r, n);
    return (kind == PASS_C2C_CONTIG || kind == PASS_C2C_TILED) && bluestein_length(n) ? bluestein_log2m(n) : ilog2_exact(n);
}

// The tables such a pass reads, from T: tw of its power-of-two length, tw2 for R2C / C2R and DCT / DST passes (r2r: the kind
// of R2R passes; DCT / DST take w_k = exp(-i pi k / 2N), k <= N, the R2C table of length 2N), blu for Bluestein lengths.
// Type-I passes take tw and tw2 of log2 N (W^k = exp(-i pi k / N), k <= N/2).  Type-IV passes take tw of log2 N - 1 and, as
// tw2, the type-IV table of N.  One rule for plans and for the single-axis calls.
static int pass_tables(Tables& T, PassKind kind, size_t n, int r2r, void** tw, void** tw2, void** blu) {
    const bool rr = kind == PASS_R2R_CONTIG || kind == PASS_R2R_TILED;
    const bool type1 = rr && is_type1(r2r);
    const int l2 = pass_log2(kind, n, rr ? r2r : 0);
    const bool with_w = rr && r2r != DFFT_R2HC && !type1;
    *tw = *tw2 = *blu = nullptr;
    if (rr && is_type4(r2r)) {
        if (T.get_tw(l2 - 1, tw) != cudaSuccess || T.get_r2r4(l2, tw2) != cudaSuccess) return fail(DFFT_ERR_CUDA, "twiddle table allocation failed");
        return DFFT_SUCCESS;
    }
    if (!type1 && l2 != ilog2_exact(n) && T.get_blu(n, blu) != cudaSuccess) return fail(DFFT_ERR_CUDA, "Bluestein table allocation failed");
    if (T.get_tw(l2, tw) != cudaSuccess) return fail(DFFT_ERR_CUDA, "twiddle table allocation failed");
    if ((kind == PASS_R2C || kind == PASS_C2R || with_w || type1) && T.get_tw2(l2 + (with_w ? 1 : 0), tw2) != cudaSuccess)
        return fail(DFFT_ERR_CUDA, "twiddle table allocation failed");
    return DFFT_SUCCESS;
}

// ---- device rendezvous ---------------------------------------------------------------------------------
// flags layout (uint64): [phase][rank], NPHASE phases.  Thread i handles group member i: publishes my
// epoch in the peer's flag row, then waits for the peer's epoch in mine.
constexpr int NPHASE = 4;
constexpr unsigned long long FLAG_POISON = ~0ull;  // written into every peer's flag rows by a rank that gave up waiting
// A missing peer: the reference would block in MPI_Waitall forever (mpicufft_slab.cpp:802-803).  Here the wait
// gives up after `timeout_cycles` (DFFT_RENDEZVOUS_TIMEOUT_S, default 300 s, 0 = wait forever), records the error
// and POISONS the flag rows of every group member, so that no rank silently continues on half-delivered slots:
// every later rendezvous of every member sees the poison, records an error as well, and dfft_plan_wait returns
// DFFT_ERR_TIMEOUT on all of them (the plan is dead after that and must be destroyed).
__global__ void rendezvous_kernel(unsigned long long* const* peer_flags, unsigned long long* my_flags, const int* group,
                                  int gsize, int me, int nranks, int phase, unsigned long long epoch, int* err,
                                  long long timeout_cycles) {
    const int i = threadIdx.x;
    if (i >= gsize) return;
    const int q = group[i];
    if (q == me) return;
    __threadfence_system();
    unsigned long long* dst = peer_flags[q] + size_t(phase) * nranks + me;
    const unsigned long long* src = my_flags + size_t(phase) * nranks + q;
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(src) : "memory");
    if (v == FLAG_POISON) {  // a peer gave up earlier: do not overwrite its poison with my epoch
        atomicExch(err, 100 + phase);
        return;
    }
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(epoch) : "memory");
    const long long t0 = clock64();
    while (true) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(src) : "memory");
        if (v == FLAG_POISON) {
            atomicExch(err, 100 + phase);
            break;
        }
        if (v >= epoch) break;
        if (timeout_cycles > 0 && clock64() - t0 > timeout_cycles) {
            atomicExch(err, 1 + phase);
            for (int ph = 0; ph < NPHASE; ++ph)
                asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(peer_flags[q] + size_t(ph) * nranks + me), "l"(FLAG_POISON) : "memory");
            break;
        }
        __nanosleep(64);
    }
}


}  // namespace dfft

using namespace dfft;

struct dfft_comm_s {
    int rank = 0, nranks = 1, device = 0;
    ncclComm_t nccl = nullptr;
    bool dry = false;  // geometry-only: plans never touch CUDA (dfft_comm_create_dry)
};

namespace dfft {

enum StepType { STEP_PASS = 0, STEP_RENDEZVOUS = 1, STEP_A2A = 2 };
// the kernel a PASS step launches: one FFT pass, the fused z + y stage or the batched stage of small cubic fields
enum StepKernel { KERNEL_PASS = 0, KERNEL_ZY_FUSED = 1, KERNEL_BATCH_SMALL = 2 };

struct Step {
    StepType type = STEP_PASS;
    const char* phase = nullptr;  // timer section recorded after this step
    const char* label = "";       // short name of the step ("z pass", "y pass", "rendezvous 2", ...)
    // PASS
    StepKernel kernel = KERNEL_PASS;
    PassKind kind = PASS_C2C_CONTIG;
    int log2n = 0;
    // pass length (0: 2^log2n); when it is not 2^log2n the pass runs fft_bluestein_kernel with M = 2^log2n points and the
    // table `blu`
    size_t n = 0;
    const void* blu = nullptr;
    bool bluestein() const { return !is_copy(kind) && n != 0 && n != (size_t(1) << log2n); }
    // PASS_R2R_*: the kind of the axis it transforms (DFFT_DCT, DFFT_DST, DFFT_R2HC, DFFT_DCT1 or DFFT_DST1; type-I passes
    // have n = L reals per line and log2n = log2 N)
    int r2r = 0;
    int axis = 0;  // the axis of the pass: 0 x, 1 y, 2 z (PASS_COPY_*: n is its length, log2n 0)
    // padded plans: the points its spectral side keeps of each line (Kx, Ky, Kz; R2C / C2R: Kz/2 + 1 of the Nz/2 + 1), the
    // rest is the hole (fft_kernels.cuh, FftPadded); 0: the whole line
    size_t keep = 0;
    // pruned plans: the points its physical side holds of each line (Mx, My, Mz; R2C / C2R: Mz reals), the rest is zero
    // (forward: never loaded, inverse: never stored); 0: the whole line
    size_t data = 0;
    // points along n of its input and output views (dfft_debug_run_step and embed_views size views by them)
    void view_lens(size_t* in_len, size_t* out_len) const {
        const size_t len = n ? n : size_t(1) << log2n;
        const size_t phys = data ? (kind == PASS_R2C || kind == PASS_C2R ? data / 2 : data) : len;
        *in_len = prm.inverse ? (keep ? keep : len + (kind == PASS_C2R ? 1 : 0)) : phys;
        *out_len = prm.inverse ? phys : (keep ? keep : len + (kind == PASS_R2C ? 1 : 0));
    }
    FftParams prm{};
    int in_user = 0, out_user = 0;  // 1: patch seg[0].base with the caller's in, 2: with the caller's out
    // RENDEZVOUS
    int group = 0, phase_id = 0;  // group: 0 all, 1 first transposition group, 2 second
    // A2A
    std::vector<size_t> scount, soff, rcount, roff;  // elements, indexed by group member
    int send_slot = 0, recv_slot = 0;
    // overlapped schedules: which plan stream runs the step (0 = caller's stream, 1 = exchange stream,
    // 2 = follow-up stream), events to wait for before it and the event to record after it
    int stream = 0;
    std::vector<int> waits;
    int record = -1;
    // fused z + y stage (KERNEL_ZY_FUSED): prm is the z pass, prm_y the y pass; zyf holds the counters, advanced by every
    // launch on the device
    FftParams prm_y{};
    int y_in_user = 0, y_out_user = 0;  // in_user / out_user of prm_y (in-place plans: its view on the caller's buffer)
    ZyFused zyf{};
    // batched small cubic fields (KERNEL_BATCH_SMALL): one launch for every field; prm.in / prm.out are the caller's
    // buffers, bsf holds the counters
    BatchSmall bsf{};
    // its stores are output values of the exec (the fused and batched stages: those of their last phase), so it runs the
    // scaled twin of its kernel when the plan's output scale for the direction is not 1 (dfft_plan_set_scale)
    bool final_store = false;
    // a copy whose input and output views are the same elements, kept because it stores final values: it only has work to
    // do when the output scale is not 1, and is not launched otherwise (drop_identity_copies)
    bool identity = false;
    // 16-bit plans (split_scale): an FFT pass stores its values times |s|^(share_num / share_den) of the direction's scale s
    // (log2 of its axis length over the sum for the exec's transformed axes), and times the sign of s when `sign`; share_den
    // 0: never scaled (copy passes, other precisions)
    int share_num = 0, share_den = 0;
    bool sign = false;
    // weighted plans (dfft_plan_set_weights): an FFT pass that multiplies its spectral side by the weights of its axis (the
    // plan's pointer for `axis` at exec time, none while it is null): forward its stores, inverse its loads
    bool weighted = false;
    // 1D plans (dfft_plan_create_1d): the twiddled y or z pass ("y" / "z", null for none) and its twiddle; tw.table is
    // null on geometry-only plans
    const char* twiddle = nullptr;
    Twiddle1d tw{};
};

struct Schedule {
    std::vector<Step> steps;
    bool built = false;
    // batched plans: the steps transform one field and run once per field, the caller's buffers shifted by field_in /
    // field_out bytes each time — unless whole_batch, where they cover every field at once
    bool whole_batch = false;
    size_t field_in = 0, field_out = 0;
    // an eager exec has run this schedule: its tables, counters and kernel attributes are set up, so a stream capture
    // may record it (dfft_plan_describe builds schedules without running them)
    bool executed = false;
    bool overlapped = false;  // uses the plan's auxiliary streams
    int nevents = 0;
    int inverse = 0;          // direction (selects the plan's output scale)
};

// The work slots of the schedules, in the order they lie in the work area: D1 and D2 receive the first and the second
// transposition by peer stores (or hold it on a one-member group), SS and SR are the send and receive slots of the
// all-to-all transpositions; -1: the plan has no such slot.  BX: box plans (dfft_plan_create_boxes) only, the staging
// array of their reshape steps, which no pass of the wrapped schedule touches.
struct Slots {
    int D1 = -1, D2 = -1, SS = -1, SR = -1, BX = -1;
    int count = 0;
};
// direct1 / direct2: whether the first / second transposition is direct (peer stores, or a one-member group)
static Slots plan_slots(bool direct1, bool direct2) {
    Slots s;
    if (direct1) s.D1 = s.count++;
    if (direct2) s.D2 = s.count++;
    if (!direct1 || !direct2) { s.SS = s.count++; s.SR = s.count++; }
    return s;
}

}  // namespace dfft

struct dfft_plan_s {
    dfft_comm_t comm = nullptr;
    dfft_config cfg{};
    std::string bench_dir;
    Geometry g;
    int prec = DFFT_F64;
    size_t esize = 16;  // bytes per complex element
    int rank = 0, P = 1;
    int kinds[3] = {0, 0, 0};  // real-to-real plans: the kind of the x, y and z axis
    int taxes[3] = {1, 1, 1};  // dfft_plan_set_transform_axes: 1 transforms the x, y, z axis, 0 keeps it (copy passes)
    bool axes_fixed = false;   // a schedule was built or tuned for taxes: the setter refuses from then on
    size_t batch = 1;         // fields per exec, back to back in every caller buffer (dfft_plan_create_batched)
    size_t comps = 1;         // values per grid point, interleaved (dfft_plan_create_interleaved); esize stays one value's
    double scale[2] = {1.0, 1.0};  // [fwd/inv] output scale (dfft_plan_set_scale), applied by the steps marked final_store
    // dfft_plan_set_weights: the caller's per-axis spectral weights (device pointers, null = all ones), read by the steps
    // marked weighted at every exec.  weighted: the first call came before any schedule was built.
    const void* weights[3] = {nullptr, nullptr, nullptr};
    bool weighted = false;
    // dfft_plan_create_1d: the signal's length N = Nx * Ny * Nz (the factors are the grid), 0 for 3D plans
    size_t n1d = 0;
    // dfft_plan_create_1d_natural: the split of N3 over the ranks, rank r's output chunk [oz.size[r]][N2][N1] from k3 =
    // oz.start[r]; empty for every other plan
    dfft::Split oz;
    // dfft_plan_create_boxes: every rank's box of the physical grid (in_boxes) and of the output grid (out_boxes), in rank
    // order; empty where that side has the natural layout.  box_direct: their reshapes push and gather over peer memory
    // (comm_method Peer2Peer), otherwise they run through an NCCL all-to-all
    std::vector<dfft::Box> in_boxes, out_boxes;
    bool box_direct = false;
    bool boxed() const { return !in_boxes.empty() || !out_boxes.empty(); }
    // dfft_plan_set_strides: the caller's {field, x, y} strides of the physical side (in) and of the output of d = 3 (out),
    // in that side's elements (reals on the real side of R2C / C2R and for R2R plans); z is contiguous.  A side without
    // them is dense.
    long long in_strides[3] = {0, 0, 0}, out_strides[3] = {0, 0, 0};
    bool in_embedded = false, out_embedded = false;
    bool embedded() const { return in_embedded || out_embedded; }
    // dfft_plan_create_inplace: every exec has out == in, fields domain_bytes apart, real rows of R2C / C2R padded to Nzc
    // complex units.  buf_slot: one rank — the schedules' first slot (D1) is the caller's buffer and is not allocated.
    bool inplace = false, buf_slot = false;
    size_t domain_bytes = 0;  // this rank (getDomainSize)
    size_t slot_bytes = 0;    // uniform over ranks
    dfft::Slots slots;        // the schedules' slot ids (plan_slots)
    int nslots = 2;           // slots allocated in the work area
    size_t work_bytes = 0;
    void* work = nullptr;
    bool work_owned = false;
    bool any_direct = false;  // some transposition uses peer stores across >1 ranks
    bool direct1 = true, direct2 = true;
    // peer mapping
    std::vector<std::vector<void*>> slot_ptr;  // [allocated slot][rank]
    // Slot s (Slots) of rank r.  buf_slot: D1 is the caller's buffer, a null base (its views hold byte offsets, which
    // relocate_buffer_views turns into views on the buffer), and the allocated slots start at the next one.
    void* slot(int s, int r) const { return !buf_slot ? slot_ptr[s][r] : s == slots.D1 ? nullptr : slot_ptr[s - 1][r]; }
    std::vector<void*> opened;                 // IPC mappings to close
    unsigned long long* flags = nullptr;       // my flags (NPHASE * P)
    unsigned long long** peer_flags_d = nullptr;
    std::vector<void*> opened_flags;
    int* groups_d = nullptr;  // [3][P] group member lists on device
    std::vector<int> grp[3];
    int* err_d = nullptr;
    size_t l2_bytes = size_t(50) << 20;           // L2 of the plan's GPU (geometry-only plans: an H100's 50 MB)
    unsigned long long epoch = 0;
    unsigned long long ticket[4] = {0, 0, 0, 0};  // per-phase rendezvous counters (same sequence on every rank)
    cudaStream_t aux[2] = {nullptr, nullptr};     // exchange stream (high priority), follow-up stream
    std::vector<cudaEvent_t> sync_events;
    cudaEvent_t fork_ev = nullptr, join_ev[2] = {nullptr, nullptr};
    int xchg_ctas = 0;                            // SMs given to the exchange pass in overlapped schedules
    int tuned_seq[2] = {0, 0};                    // dfft_plan_tune: [fwd/inv] 1 = the sequential schedule won
    int tuned_chunks[2] = {0, 0};                 // dfft_plan_tune: [fwd/inv] z chunks of the winning overlapped schedule (0 = ovl_chunks)
    int tuned_groups_inv = 0;                     // dfft_plan_tune: plane groups of the inverse overlapped pencil schedule (0 = ovl_groups)
    int tuned_ctas[2] = {-2, -2};                 // dfft_plan_tune: [fwd/inv] exchange CTAs of the winning overlapped schedule (-2 = not tuned)
    std::string tune_report;
    int ovl_groups = 4, ovl_chunks = 4;           // overlapped schedules: plane groups of the z pass, z chunks of the y / x passes
    int blocked_ch = 0;                           // > 0: slab forward keeps the y->x intermediate as [b/CH][Nx][CH]
    int single_rank_layout = 1;                   // one rank: hand-over [ny][nzm/CH][nx][CH] (x innermost) instead of [nzm/CH][nx][ny][CH] (DFFT_N1_LAYOUT=0)
    int x_swz = 1;                                // tile-order blocking (log2 G) of passes that read the blocked hand-over layout
    int blocked_inv = 1;                          // the inverse x -> y hand-over is blocked as well (DFFT_BLOCKED_INV=0: plain)
    int xchg_tile_pref = 2;                       // tile preference of passes that store into other GPUs (2 = wide rows)
    long long rendezvous_timeout_cycles = 0;      // device clock cycles a rendezvous waits for a peer (0 = forever)
    int bulk_store = 0;                           // experimental: exchanging y pass stores with cp.async.bulk (DFFT_BULK_STORE=1)
    cudaStream_t own_stream = nullptr, last_stream = nullptr;  // last_stream: stream of the last exec
    cudaEvent_t entry_ev = nullptr;  // synchronous execs: "everything the caller queued on the legacy default stream"
    Tables tabs;
    // schedules: [fwd/inv][d-1]
    Schedule sched[2][3];
    // timing
    bool timing = false;
    std::vector<cudaEvent_t> events;
    std::vector<const char*> ev_names;
    std::vector<int> ev_is_fft;  // 1 fft pass, 0 exchange
    std::vector<const char*> ev_labels;
    int n_events_used = 0;
    // timeline of the last timed exec: one (begin, end) event pair per step, recorded on the step's own stream
    std::vector<cudaEvent_t> tl_events;
    std::vector<const char*> tl_labels;
    std::vector<int> tl_streams;
    int tl_used = 0;
    int last_launches = 0;
    int execs = 0;
    double init_ms = 0;          // "init" section of the reference's CSV
    int csv_warmup_left = 0;     // execs still to be skipped (Configurations::warmup_rounds)
    std::string csv_path;        // empty: no CSV
};

namespace dfft {

// element offset helper
static inline void* eptr(void* base, size_t elems, size_t esize) { return (char*)base + elems * esize; }

static View single_view(void* base, long long sA0, long long sA1, long long sN) {
    View v{};
    v.seg_of_n = nullptr;
    v.nseg = 1;
    v.sN = sN;
    v.seg[0].base = base;
    v.seg[0].sA0 = sA0;
    v.seg[0].sA1 = sA1;
    v.seg[0].n0 = 0;
    return v;
}

}  // namespace dfft

// =====================================================================================================
// Schedule construction
// =====================================================================================================
namespace dfft {

static int build_schedule(dfft_plan_s* p, int inverse, int d, Schedule& sc);
static int build_overlapped_forward(dfft_plan_s* p, Schedule& sc);
static int build_overlapped_slab_inverse(dfft_plan_s* p, Schedule& sc);
static int build_overlapped_pencil_inverse(dfft_plan_s* p, Schedule& sc);
static bool pencil_overlap_enabled();

}  // namespace dfft

static int plan_setup_memory(dfft_plan_s* p, void* user_device);
static void plan_release_memory(dfft_plan_s* p);

// -----------------------------------------------------------------------------------------------------
namespace dfft {

// Fill a segmented view over group members. f(q_pos, rank) returns the segment and the (view-wide) stride
// along the transformed axis.
struct SegN {
    Seg s;
    long long sN;
};
static bool g_view_error = false;
template <typename F>
static void seg_view(View& v, const unsigned char* table, const std::vector<int>& ranks, F f) {
    v.seg_of_n = table;
    v.nseg = int(ranks.size());
    for (size_t q = 0; q < ranks.size(); ++q) {
        SegN sn = f(int(q), ranks[q]);
        v.seg[q] = sn.s;
        if (q == 0) v.sN = sn.sN;
        else if (v.sN != sn.sN) g_view_error = true;
    }
    if (v.nseg == 1) v.seg_of_n = nullptr;
}

static SegN mkseg(void* base, long long sA0, long long sA1, long long sN, size_t n0) {
    SegN r{};
    r.s.base = base; r.s.sA0 = sA0; r.s.sA1 = sA1; r.s.n0 = int(n0);
    r.sN = sN;
    return r;
}

// Whether every axis is a power of two.  Plans with another length run the sequential schedule only: the overlapped
// schedules build their passes for power-of-two lengths.
static bool pow2_axes(const dfft_plan_s* p) { return ilog2_exact(p->g.nx) > 0 && ilog2_exact(p->g.ny) > 0 && ilog2_exact(p->g.nz) > 0; }
// Whether every axis is transformed.  Plans with a kept axis (dfft_plan_set_transform_axes) run the sequential schedule
// only: the overlapped schedules, the fused z + y stage and the batched stage transform every axis they touch.
static bool all_axes(const dfft_plan_s* p) { return p->taxes[0] && p->taxes[1] && p->taxes[2]; }
// Why a plan's features keep it on the sequential schedule, or null: the overlapped schedules, the fused z + y stage and the
// batched stage run none of them.  Their kernels have no 16-bit, weighted or padded twins (FftPadded), and run C2C and
// R2C / C2R passes over every axis.  Interleaved plans (C > 1 values per point): those kernels address one value per
// point.  Plans with a box that is not the natural layout: their reshape steps wrap the sequential schedule (wrap_boxes).
// Embedded plans (dfft_plan_set_strides): the other forms read and write dense caller arrays, and every rank must run the
// same form.  1D plans: their schedule (build_1d) has its own transpositions and twiddled passes.  The text completes
// dfft_plan_tune's report.
static const char* sequential_only(const dfft_plan_s* p) {
    if (p->n1d) return "1D plans";
    if (is_half(p->prec)) return "16-bit plans";
    if (p->weighted) return "weighted plans";
    if (is_r2r(p->g.transform)) return "DCT / DST plans";
    if (!all_axes(p)) return "plans with a kept axis";
    if (p->g.padded()) return "padded plans";
    if (p->g.pruned()) return "pruned plans";
    if (p->comps > 1) return "interleaved plans";
    if (p->boxed()) return "box plans";
    if (p->embedded()) return "plans with strides";
    return nullptr;
}

// Whether the schedules may take another form than the sequential one: the overlapped schedules build their passes for
// power-of-two lengths.
static bool alt_schedules(const dfft_plan_s* p) { return pow2_axes(p) && !sequential_only(p); }

// Row pitch, in elements (complex units; reals for DCT / DST plans), of the z-contiguous side of the caller's buffers that
// holds Nz points per row: the input of forward passes, the output of inverse ones.  Real rows of R2C / C2R plans are Nz reals (Nz/2 units) apart, or, in
// place, Nzc units apart (the padded layout of FFTW and cuFFT: the last one or two reals of a row are never touched).
// Pruned plans hold Mz points per row (R2C / C2R: Mz reals, Mz/2 units).
static long long z_row_pitch(const dfft_plan_s* p) {
    const Geometry& g = p->g;
    return (long long)(p->inplace ? g.nzc : g.transform != DFFT_R2C ? g.mz : g.mz / 2);
}

// Whether the z and y passes run as one fused launch (fft_zy_fused_kernel): one-rank slab C2C plans of the full 3D
// transform with Ny == Nz of an instantiated length (zy_fused_length) whose array is larger than the L2 — below that the
// three passes are L2-resident already and gain nothing.
static bool zy_fused(const dfft_plan_s* p, int inverse, int d) {
    const Geometry& g = p->g;
    if (p->P != 1 || g.decomp != DFFT_SLAB_ZY_THEN_X || g.transform != DFFT_C2C || d != 3 || sequential_only(p)) return false;
    if (g.ny != g.nz || !zy_fused_length(ilog2_exact(g.ny))) return false;
    // the fused stage reads and writes the blocked hand-over layout of the x pass
    if (p->blocked_ch <= 0 || g.nz % size_t(p->blocked_ch) || (inverse && !p->blocked_inv)) return false;
    return g.ny * g.nz * p->esize * g.nx > p->l2_bytes;
}

// one launch of z and y: zs = the z pass, ys = the y pass (of the same direction), phase = timer section
static int fuse_zy(dfft_plan_s* p, Step zs, const Step& ys, const char* label, const char* phase, Step& out) {
    if (zs.log2n != ys.log2n) return fail(DFFT_ERR_STATE, "internal: fused z + y stage needs Ny == Nz");
    out = zs;
    out.kernel = KERNEL_ZY_FUSED;
    out.label = label;
    out.phase = phase;
    out.prm_y = ys.prm;
    out.zyf = ZyFused{};
    // Groups of one plane; phase A runs L planes ahead of phase B: L + 1 planes of intermediate in flight, a third of the
    // L2 (512^2 complex-double: L = 3; L = 2, L = 5 and groups of two planes were slower, DESIGN.md section 3.4).
    out.zyf.order.nx = int(p->g.nx);
    out.zyf.order.gpp = 1;
    {
        const long long ahead = (long long)(p->l2_bytes / (3 * p->g.ny * p->g.nz * p->esize)) - 1;
        out.zyf.order.ahead = int(ahead < 1 ? 1 : ahead);
        if (const char* e = getenv("DFFT_ZY_AHEAD")) out.zyf.order.ahead = std::max(1, atoi(e));  // look-ahead sweeps
    }
    out.zyf.err = p->err_d;
    out.zyf.timeout_cycles = p->rendezvous_timeout_cycles;
    if (!p->tabs.dry) {
        // [0] ticket counter, [1 + g] per-group counters; zeroed once, then only ever incremented (epoch targets)
        const size_t bytes = sizeof(unsigned long long) * (1 + size_t(out.zyf.order.groups()));
        void* c = nullptr;
        if (cudaMalloc(&c, bytes) != cudaSuccess) return fail(DFFT_ERR_CUDA, "fused z + y stage: counter allocation failed");
        p->tabs.bytes.push_back(c);  // freed with the schedules
        if (cudaMemset(c, 0, bytes) != cudaSuccess) return fail(DFFT_ERR_CUDA, "fused z + y stage: counter initialisation failed");
        out.zyf.ctr = reinterpret_cast<unsigned long long*>(c);
#ifdef DFFT_ZY_TRACE
        // trace build: ZY_TRACE_SLOTS stamps per work item (4096 points each, both phases), rewritten by every launch
        const size_t tbytes = sizeof(unsigned long long) * ZY_TRACE_SLOTS * 2 * size_t(p->g.nx) * (p->g.ny * p->g.nz / 4096);
        void* t = nullptr;
        if (cudaMalloc(&t, tbytes) != cudaSuccess) return fail(DFFT_ERR_CUDA, "fused z + y stage: trace allocation failed");
        p->tabs.bytes.push_back(t);
        if (cudaMemset(t, 0, tbytes) != cudaSuccess) return fail(DFFT_ERR_CUDA, "fused z + y stage: trace initialisation failed");
        out.zyf.trace = reinterpret_cast<unsigned long long*>(t);
#endif
    }
    return DFFT_SUCCESS;
}

// Whether a batched exec runs as one launch of fft_batch_small_kernel: one-rank slab C2C plans of the full 3D transform
// of cubic fields of an instantiated length (batch_small_length), from BATCH_SMALL_MIN fields on.  Decided from the
// length, the precision and the batch only; every other batched plan runs its per-field schedule once per field.
constexpr size_t BATCH_SMALL_MIN = 2;
static bool batch_small(const dfft_plan_s* p, int d) {
    const Geometry& g = p->g;
    if (p->P != 1 || g.decomp != DFFT_SLAB_ZY_THEN_X || g.transform != DFFT_C2C || d != 3 || sequential_only(p)) return false;
    if (g.nx != g.ny || g.ny != g.nz || !batch_small_length(ilog2_exact(g.nx))) return false;
    return p->batch >= BATCH_SMALL_MIN && p->batch * g.nx <= 0x7fffffff;
}

static int build_batch_small(dfft_plan_s* p, int inverse, Schedule& sc) {
    const size_t N = p->g.nx;
    sc.whole_batch = true;
    Step s;
    s.type = STEP_PASS;
    s.kernel = KERNEL_BATCH_SMALL;
    s.label = "batched pass";
    s.phase = inverse ? "2D FFT Y-Z-Direction" : "1D FFT X-Direction";  // the exec's last section
    s.kind = PASS_C2C_CONTIG;
    s.log2n = ilog2_exact(N);
    s.prm.inverse = inverse;
    void* tw = nullptr;
    if (p->tabs.get_tw(s.log2n, &tw) != cudaSuccess) return fail(DFFT_ERR_CUDA, "twiddle table allocation failed");
    s.prm.tw = tw;
    s.prm.in = single_view(nullptr, 0, 0, 1);
    s.prm.out = single_view(nullptr, 0, 0, 1);
    s.in_user = 1;
    s.out_user = 2;
    s.bsf.tw = tw;
    s.bsf.err = p->err_d;
    s.bsf.timeout_cycles = p->rendezvous_timeout_cycles;
    // look-ahead in fields: phase A runs L fields ahead of phase B, L + 1 fields of intermediate in flight, a third of the
    // L2 (the rule of the fused z + y stage, with a field in place of a plane)
    const long long ahead = (long long)(p->l2_bytes / (3 * N * N * N * p->esize)) - 1;
    s.bsf.order.ahead = int(ahead < 1 ? 1 : ahead);
    if (!p->tabs.dry) {
        const size_t bytes = sizeof(unsigned long long) * (1 + p->batch);
        void* c = nullptr;
        if (cudaMalloc(&c, bytes) != cudaSuccess) return fail(DFFT_ERR_CUDA, "batched stage: counter allocation failed");
        p->tabs.bytes.push_back(c);  // freed with the schedules
        if (cudaMemset(c, 0, bytes) != cudaSuccess) return fail(DFFT_ERR_CUDA, "batched stage: counter initialisation failed");
        s.bsf.ctr = reinterpret_cast<unsigned long long*>(c);
    }
    sc.steps.push_back(s);
    return DFFT_SUCCESS;
}

// One pass step of n-point lines along `axis` (0 x, 1 y, 2 z), with the tables of its length (pass_tables), recording the
// timer section `phase`; the builders set its views and dims.  DCT / DST plans run the C2C builders over reals: their C2C
// kinds become R2R ones, of the axis's kind.
static int new_pass(dfft_plan_s* p, int inverse, PassKind kind, size_t n, int axis, const char* phase, Step& s) {
    const Geometry& g = p->g;
    s = Step();
    s.type = STEP_PASS;
    s.label = (kind == PASS_C2C_TILED) ? "strided pass" : (kind == PASS_R2C ? "z pass (R2C)" : (kind == PASS_C2R ? "z pass (C2R)" : "z pass"));
    s.axis = axis;
    s.phase = phase;
    s.n = n;
    s.prm.A0 = 1; s.prm.A1 = 1; s.prm.B = 1;
    s.prm.inverse = inverse;
    if (!p->taxes[axis]) {
        // a kept axis: this pass's views, moved by the copy kernel without tables (labels: name_copies)
        s.kind = kind == PASS_C2C_TILED ? PASS_COPY_TILED : PASS_COPY_CONTIG;
        return DFFT_SUCCESS;
    }
    if (is_r2r(g.transform)) {
        kind = kind == PASS_C2C_TILED ? PASS_R2R_TILED : PASS_R2R_CONTIG;
        s.r2r = p->kinds[axis];
    }
    s.kind = kind;
    // Bluestein lengths: the view mapping stays the kind's; the exec launches the Bluestein kernel.  Type-I R2R passes:
    // log2 N of their N +- 1 reals per line
    s.log2n = pass_log2(kind, n, s.r2r);
    {   // padded plans: the spectral extent of the axis; pruned plans: its data extent
        const size_t k = axis == 0 ? g.kx : axis == 1 ? g.ky : g.kzc, full = axis == 0 ? g.nx : axis == 1 ? g.ny : g.nzc;
        if (k != full) s.keep = k;
        const size_t m = axis == 0 ? g.mx : axis == 1 ? g.my : g.mz, phys = axis == 0 ? g.nx : axis == 1 ? g.ny : g.nz;
        if (m != phys) s.data = m;
    }
    if (s.log2n < 1 || s.log2n > MAX_LOG2N)
        return fail(DFFT_ERR_UNSUPPORTED, "axis length " + std::to_string(n) + " is not a supported power of two (2..8192)");
    void *tw = nullptr, *tw2 = nullptr, *blu = nullptr;
    const int rc = pass_tables(p->tabs, kind, n, s.r2r, &tw, &tw2, &blu);
    s.prm.tw = tw;
    s.prm.tw2 = tw2;
    s.blu = blu;
    return rc;
}

// A rendezvous of `group` (0 all ranks, 1 first transposition group, 2 second) on plan stream `stream`
static Step new_rendezvous(int group, int phase_id, const char* phase, int stream) {
    Step s;
    s.type = STEP_RENDEZVOUS;
    s.label = group == 0 ? "entry rendezvous" : (group == 1 ? "rendezvous 1" : "rendezvous 2");
    s.group = group;
    s.phase_id = phase_id;
    s.phase = phase;
    s.stream = stream;
    return s;
}

// The blocked hand-over of the second transposition: the scattering pass (forward the y pass, inverse the x pass) stores
// into the slots of its G2 members, the gathering pass (forward x, inverse y) reads its own.  A receiver's nz columns of z
// are laid out as
//   forward  [nzm/CH][mx][ny_q][CH] + tail [mx][ny_q][rem]      (ny_q: the receiver's y rows; mx: the data's x planes)
//   inverse  [nzm/CH][ky][nx_q][CH] + tail [nx_q][ky][rem]      (nx_q: the receiver's x planes)
// with rem = nz % CH leftover columns and nzm = nz - rem, so the rows a tile of the scattering pass sends to one receiver
// are adjacent (one contiguous run per receiver: what NVLink stores need), and the gathering pass reads rows CH apart.
// The tail is the plain layout of the leftover columns, run by one extra launch of each pass.  The other side of both
// passes is plain, z innermost.  One rank, forward (x_inner): [ky][nzm/CH][nx][CH], so that every x-pass tile is one
// contiguous block.  A pass covers planes [a, +npl) of its a0 axis and the z columns [z0, +zc), whole blocks.
struct HandOver {
    size_t CH = 0, rem = 0, nzm = 0;
    bool any_rem = false;  // some rank of the grid has leftover columns: every rank runs the tail steps (B = 0 on the others)
    bool fwd = true, x_inner = false;
    int me = 0;
    size_t es = 0, nz = 0;
    size_t L = 0;            // extent of the scattering pass's a0 axis at the receivers (forward nx, inverse ky)
    size_t M_me = 0;         // this rank's extent of its n axis (forward its y rows, inverse its x planes)
    const Split* recv = nullptr;  // the receivers' extents along it (forward oy, inverse sx)
    const std::vector<int>* G = nullptr;
    const unsigned char* tab = nullptr;  // segment table of recv (scattering views over more than one receiver)
    std::vector<void*> slot;             // the hand-over slot (D2) of every rank

    // blocked: both transpositions are peer stores and both passes run (d = 3); sequential: the schedule of build_schedule,
    // the only one that takes the x-innermost layout of one rank
    HandOver(const dfft_plan_s* p, int inverse, bool blocked, bool sequential, const unsigned char* tab_) {
        const Geometry& g = p->g;
        me = p->rank;
        fwd = !inverse;
        es = p->esize * p->comps;
        nz = g.sz.size[g.pj(me)];
        L = fwd ? g.mx : g.ky;
        recv = fwd ? &g.oy : &g.sx;
        M_me = recv->size[g.pi(me)];
        G = &p->grp[2];
        tab = tab_;
        CH = blocked && (fwd || p->blocked_inv) ? size_t(p->blocked_ch) : 0;
        if (!CH) return;
        for (int r = 0; r < p->P; ++r) slot.push_back(p->slot(p->slots.D2, r));
        rem = nz % CH;
        nzm = nz - rem;
        for (size_t v : g.sz.size) any_rem = any_rem || v % CH != 0;
        x_inner = fwd && sequential && G->size() == 1 && p->single_rank_layout;
    }
    // The z chunks of the overlapped passes: ns ranges, of whole blocks when blocked (at most nzm / CH of them; the
    // leftover columns go with the last one)
    Split chunks(size_t ns) const {
        Split c;
        if (!CH) { c.make(nz, ns); return c; }
        c.make(nzm / CH, std::min(ns, nzm / CH));
        for (size_t k = 0; k < c.size.size(); ++k) { c.size[k] *= CH; c.start[k] *= CH; }
        return c;
    }
    // The scattering pass: input `plain` (the whole z extent from its base), stores into every receiver
    void scatter(Step& s, View plain, size_t a, size_t npl, size_t z0, size_t zc) const {
        dims(s, npl, zc);
        s.prm.in = columns(plain, z0, CH);
        seg_view(s.prm.out, tab, *G, [&](int q, int r) { return blocks(slot[r], recv->size[q], a, z0, true, recv->start[q]); });
    }
    Step scatter_tail(const Step& s, View plain, size_t a) const {
        Step t = tail(s);
        t.prm.in = columns(plain, nzm, 0);
        seg_view(t.prm.out, tab, *G, [&](int q, int r) { return leftover(slot[r], recv->size[q], a, true, recv->start[q]); });
        return t;
    }
    // The gathering pass: reads its own slot, stores into `plain`
    void gather(Step& s, View plain, size_t a, size_t npl, size_t z0, size_t zc) const {
        dims(s, npl, zc);
        s.prm.in = own(blocks(slot[me], M_me, a, z0, false, 0));
        s.prm.out = columns(plain, z0, CH);
    }
    Step gather_tail(const Step& s, View plain, size_t a) const {
        Step t = tail(s);
        t.prm.in = own(leftover(slot[me], M_me, a, false, 0));
        t.prm.out = columns(plain, nzm, 0);
        return t;
    }

  private:
    void dims(Step& s, size_t npl, size_t zc) const {
        s.prm.A0 = int(npl); s.prm.A1 = int(zc / CH); s.prm.B = int(CH);
    }
    // the pass of the leftover columns: a copy of s, on the same stream, that waits for nothing and records nothing
    Step tail(const Step& s) const {
        Step t = s;
        t.label = s.axis == 1 ? "y pass (tail)" : "x pass (tail)";
        t.phase = nullptr;
        t.prm.bulk_out = 0;
        t.waits.clear();
        t.record = -1;
        t.prm.A1 = 1; t.prm.B = int(rem);
        return t;
    }
    // the plain side from column z0 on: rows CH apart within a pass of blocks (sA1 = CH), one row per line in the tail
    View columns(View v, size_t z0, size_t sA1) const {
        for (int i = 0; i < v.nseg; ++i) {
            v.seg[i].base = eptr(v.seg[i].base, z0, es);
            v.seg[i].sA1 = (long long)sA1;
        }
        return v;
    }
    static View own(const SegN& sn) { return single_view(sn.s.base, sn.s.sA0, sn.s.sA1, sn.sN); }
    // the blocked part in the slot `base` of a receiver holding m along the scattering pass's n axis: writer, a0 runs over
    // L (from a) and n over m; reader, a0 runs over m (from a) and n over L
    SegN blocks(void* base, size_t m, size_t a, size_t z0, bool writer, size_t n0) const {
        const size_t sl = x_inner ? CH : m * CH, sm = x_inner ? nzm * L : CH, blk = x_inner ? L * CH : L * m * CH;
        const size_t sa = writer ? sl : sm, sn = writer ? sm : sl;
        return mkseg(eptr(base, (z0 / CH) * blk + a * sa, es), (long long)sa, (long long)blk, (long long)sn, n0);
    }
    // the tail behind it: x outermost (forward [L][m][rem], inverse [m][L][rem])
    SegN leftover(void* base, size_t m, size_t a, bool writer, size_t n0) const {
        const size_t sl = fwd ? m * rem : rem, sm = fwd ? rem : L * rem;
        const size_t sa = writer ? sl : sm, sn = writer ? sm : sl;
        return mkseg(eptr(base, L * m * nzm + a * sa, es), (long long)sa, 0, (long long)sn, n0);
    }
};

// The axes of a rank's box of data (x outermost, z innermost), and no axis
enum BoxAxis { AX = 0, AY = 1, AZ = 2, NO_AXIS = -1 };
// The box axes a pass's batch indices a0, a1 and its line index n run over (NO_AXIS: stride 0)
struct Roles {
    int a0, a1, n;
};
using Origin = std::array<size_t, 3>;

// A plain transposition over group 1 or 2: the sending pass transforms axis s and scatters it over the members by `ss`,
// and the receiving pass gathers axis t, which the senders hold split by `st`, to its whole extent.  The third axis keeps
// this rank's extent `u`.
//   direct (peer stores into slot D1 / D2): receiver q's array is the box with ss.size[q] along s and the whole t; each
//     sender writes its sub-box at st.start of its position along t
//   all-to-all: the same box with the sender's own extent along t, packed at soff[q] of slot SS, scount[q] elements;
//     the receive side mirrors it at roff[q] of slot SR — one view when t is x, where the senders' blocks stack
// The receiving pass transforms t (forward Z_Then_YX: y, with t = x outermost), so its input segments lie along its n axis.
// `at` moves a view to a sub-box (the plane groups and z chunks of the overlapped schedules).  slot: the slot a direct
// transposition stores into, when not the group's own (D1 for group 1, D2 for group 2).
struct Transposition {
    const dfft_plan_s* p;
    int group, s, t;
    const Split *ss, *st;
    size_t u, whole;
    const unsigned char *tab_s, *tab_t;  // segment tables of ss and st (views over more than one member)
    const std::vector<int>* G;
    int pos = 0;  // this rank's position in G
    bool direct;
    int D;        // the slot of a direct transposition
    Step a2a;     // the all-to-all step of one that is not

    Transposition(const dfft_plan_s* p_, int group_, int s_, int t_, const Split& ss_, const Split& st_, size_t u_,
                  const unsigned char* tab_s_, const unsigned char* tab_t_, int slot = -1)
        : p(p_), group(group_), s(s_), t(t_), ss(&ss_), st(&st_), u(u_), whole(st_.start.back() + st_.size.back()), tab_s(tab_s_),
          tab_t(tab_t_), G(&p_->grp[group_]) {
        while ((*G)[pos] != p->rank) ++pos;
        D = group == 1 ? p->slots.D1 : p->slots.D2;
        if (D >= 0 && slot >= 0) D = slot;
        direct = D >= 0;
        if (direct) return;
        a2a.type = STEP_A2A;
        a2a.label = "nccl all-to-all";
        a2a.group = group;
        a2a.send_slot = p->slots.SS;
        a2a.recv_slot = p->slots.SR;
        size_t so = 0, ro = 0;
        for (size_t q = 0; q < G->size(); ++q) {
            a2a.scount.push_back(ss->size[q] * st->size[pos] * u);
            a2a.rcount.push_back(ss->size[pos] * st->size[q] * u);
            a2a.soff.push_back(so);
            a2a.roff.push_back(ro);
            so += a2a.scount[q];
            ro += a2a.rcount[q];
        }
    }
    // the sending pass's output: its sub-box of every receiver's array (direct) or of every block of my send slot
    View send(Roles r, Origin at = {}) const {
        View v{};
        if (direct) at[t] += st->start[pos];
        seg_view(v, tab_s, *G, [&](int q, int rk) {
            if (direct) return box(p->slot(D, rk), 0, r, ss->size[q], whole, at, ss->start[q]);
            return box(p->slot(p->slots.SS, p->rank), a2a.soff[q], r, ss->size[q], st->size[pos], at, ss->start[q]);
        });
        return v;
    }
    // the receiving pass's input: my array in slot D (direct) or the blocks of my receive slot
    View recv(Roles r, Origin at = {}) const {
        void* base = p->slot(direct ? D : p->slots.SR, p->rank);
        if (direct || t == AX) {
            const SegN b = box(base, 0, r, ss->size[pos], whole, at, 0);
            return single_view(b.s.base, b.s.sA0, b.s.sA1, b.sN);
        }
        View v{};
        seg_view(v, tab_t, *G, [&](int q, int) { return box(base, a2a.roff[q], r, ss->size[pos], st->size[q], at, st->start[q]); });
        return v;
    }
    // after the sending pass: the all-to-all, or the rendezvous after which every member's stores have landed
    void finish(Schedule& sc) const {
        static const char* const names[3][2] = {{"Transpose (Finished Receive)", "Transpose (Finished All2All)"},
                                                {"First Transpose (Finished Receive)", "First Transpose (Finished All2All)"},
                                                {"Second Transpose (Finished Receive)", "Second Transpose (Finished All2All)"}};
        const char* const* name = names[p->g.decomp == DFFT_PENCIL ? group : 0];
        if (!direct) {
            sc.steps.push_back(a2a);
            sc.steps.back().phase = name[1];
        } else if (G->size() > 1) {
            sc.steps.push_back(new_rendezvous(group, group, name[0], 0));
        }
    }

  private:
    // the box with extents es_ along s and et along t, from `base` + off elements, at sub-box `at`
    SegN box(void* base, size_t off, Roles r, size_t es_, size_t et, const Origin& at, size_t n0) const {
        size_t e[3];
        e[s] = es_;
        e[t] = et;
        e[3 - s - t] = u;
        const long long stride[3] = {(long long)(e[1] * e[2]), (long long)e[2], 1};
        auto sr = [&](int axis) { return axis == NO_AXIS ? 0LL : stride[axis]; };
        return mkseg(eptr(base, off + at[0] * e[1] * e[2] + at[1] * e[2] + at[2], p->esize * p->comps), sr(r.a0), sr(r.a1), sr(r.n), n0);
    }
};

static int build_schedule(dfft_plan_s* p, int inverse, int d, Schedule& sc) {
    const Geometry& g = p->g;
    const int me = p->rank, P = p->P;
    const int pi = g.pi(me), pj = g.pj(me);
    // DCT / DST plans run the C2C builders over reals; new_pass turns their C2C kinds into R2R ones.  The views count
    // points; interleaved plans widen them to values afterwards (widen_views).
    const bool c2c = g.transform != DFFT_R2C;
    Tables& T = p->tabs;

    // groups: transposition 1 / 2 member lists (positions along the split axis)
    const std::vector<int>& G1 = p->grp[1];
    const std::vector<int>& G2 = p->grp[2];

    if (p->any_direct) sc.steps.push_back(new_rendezvous(0, 0, nullptr, 0));  // everyone has left the previous exec: slots are free

    // spectral extents (padded plans: K; the pass lengths stay the physical N) and data extents (pruned plans: M, the
    // physical side of the axes not yet transformed).  Z_Then_YX: rows of the y-pass planes in its slots (zyx_rows).
    const size_t kzc = g.kzc, ky = g.ky, kx = g.kx, mx = g.mx, my = g.my;
    const bool zyx = g.decomp == DFFT_SLAB_Z_THEN_YX;
    const bool zy = zy_fused(p, inverse, d);  // one fused launch for the z and y passes
    int rc;

    // sizes of this rank
    const size_t nx_i = g.sx.size[pi], x0_i = g.sx.start[pi];
    const size_t ny_j = zyx ? my : g.sy.size[pj];
    const size_t nz_j = zyx ? g.sz.size[me] : g.sz.size[pj];
    const size_t oy_i = zyx ? ky : g.oy.size[pi], oy0_i = zyx ? 0 : g.oy.start[pi];

    const unsigned char *tab_z = nullptr, *tab_y_in = nullptr, *tab_y_out = nullptr, *tab_x = nullptr;
    if (G1.size() > 1) {
        if (T.seg_table(g.sz, &tab_z) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
        if (!zyx && T.seg_table(g.sy, &tab_y_in) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
    }
    if (G2.size() > 1 || (zyx && G1.size() > 1)) {
        if (!zyx && T.seg_table(g.oy, &tab_y_out) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
        if (T.seg_table(g.sx, &tab_x) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
    }

    if (!inverse) {
        // ------------------------------------------------------------------ forward
        // pass 1: z (contiguous), lines (x in nx_i, y in ny_j)
        Step s1;
        rc = new_pass(p, inverse, c2c ? PASS_C2C_CONTIG : PASS_R2C, c2c ? g.nz : g.nz / 2, 2, zyx || g.decomp == DFFT_PENCIL ? "1D FFT Z-Direction" : nullptr, s1);
        if (rc) return rc;
        s1.prm.A0 = int(nx_i); s1.prm.A1 = int(ny_j);
        {   // input: caller's buffer; real lines of nz reals = nz/2 complex (in place: padded rows)
            const long long pitch = z_row_pitch(p);
            s1.prm.in = single_view(nullptr, pitch * (long long)ny_j, pitch, 1);
            s1.in_user = 1;
        }
        if (d == 1) {
            s1.prm.out = single_view(nullptr, (long long)(ny_j * kzc), (long long)kzc, 1);
            s1.out_user = 2;
            sc.steps.push_back(s1);
            return DFFT_SUCCESS;
        }
        // transposition 1: scatter along z over G1; dest q holds [nx][ny][nz_q] (Z_Then_YX: x split -> z split) or, a pencil
        // row, [nx_i][ny][nz_q]
        const Transposition t1 = zyx ? Transposition(p, 1, AZ, AX, g.sz, g.sx, g.zyx_rows(), tab_z, tab_x)
                                     : Transposition(p, 1, AZ, AY, g.sz, g.sy, nx_i, tab_z, tab_y_in);
        s1.prm.out = t1.send({AX, AY, AZ});
        if (g.decomp == DFFT_SLAB_ZY_THEN_X) s1.phase = nullptr;
        if (!zy) sc.steps.push_back(s1);
        t1.finish(sc);

        // pass 2: y (tiled): a0 = x, n = y, b = z in nz_j
        Step s2;
        const size_t nx2 = zyx ? mx : nx_i;  // x extent held after transposition 1
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.ny, 1, g.decomp == DFFT_SLAB_ZY_THEN_X ? "2D FFT Y-Z-Direction" : (zyx ? nullptr : "1D FFT Y-Direction"), s2);
        if (rc) return rc;
        s2.label = "y pass";
        s2.prm.A0 = int(nx2); s2.prm.A1 = 1; s2.prm.B = int(nz_j);
        s2.prm.in = t1.recv({AX, NO_AXIS, AY});
        if (d == 2 || zyx) {
            if (d == 2) {
                s2.prm.out = single_view(nullptr, (long long)(ky * nz_j), 0, (long long)nz_j);
                s2.out_user = 2;
                sc.steps.push_back(s2);
                return DFFT_SUCCESS;
            }
            // z_then_yx: y pass in place (padded: its Ky output rows keep the input's strides, the first Ky * nz_j elements of
            // every x plane; pruned: My input rows, Ky output rows, planes of zyx_rows), then x pass into the caller's out
            s2.prm.out = s2.prm.in;
            if (s2.prm.in.nseg != 1) return fail(DFFT_ERR_STATE, "internal: z_then_yx gather view");
            sc.steps.push_back(s2);
            Step s3;
            rc = new_pass(p, inverse, PASS_C2C_TILED, g.nx, 0, "2D FFT Y-X-Direction", s3);
            if (rc) return rc;
            s3.label = "x pass";
            s3.prm.A0 = 1; s3.prm.A1 = 1; s3.prm.B = int(ky * nz_j);
            s3.prm.in = single_view(s2.prm.in.seg[0].base, 0, 0, (long long)(g.zyx_rows() * nz_j));
            s3.prm.out = single_view(nullptr, 0, 0, (long long)(ky * nz_j));
            s3.out_user = 2;
            sc.steps.push_back(s3);
            return DFFT_SUCCESS;
        }
        // transposition 2: scatter along y over G2 (column of the grid, or all ranks for the slab); dest q holds
        // [nx][oy_q][nz_j]
        const Transposition t2(p, 2, AY, AX, g.oy, g.sx, nz_j, tab_y_out, tab_x);
        const HandOver ho(p, inverse, t1.direct && t2.direct, true, tab_y_out);
        Step s2t;
        if (ho.CH) {
            // rows are only adjacent when the tile is CH wide: with remote peers take the wide tile (TB = CH = 8 for
            // the 1024-point f64 pass: 128-byte instead of 64-byte rows per NVLink write), locally the faster narrow one
            s2.prm.tile_pref = G2.size() > 1 ? p->xchg_tile_pref : 1;
            s2.prm.bulk_out = G2.size() > 1 ? p->bulk_store : 0;
            const View in = s2.prm.in;
            ho.scatter(s2, in, x0_i, nx_i, 0, ho.nzm);
            if (ho.any_rem) s2t = ho.scatter_tail(s2, in, x0_i);
        } else {
            if (t2.direct && G2.size() > 1) s2.prm.tile_pref = p->xchg_tile_pref;
            s2.prm.out = t2.send({AX, NO_AXIS, AY});
        }
        if (zy) {
            if (ho.any_rem || !t1.direct || !t2.direct || G1.size() > 1 || G2.size() > 1) return fail(DFFT_ERR_STATE, "internal: fused z + y stage");
            Step f;
            rc = fuse_zy(p, s1, s2, "zy pass", s2.phase, f);
            if (rc) return rc;
            sc.steps.push_back(f);
        } else if (ho.any_rem) { const char* ph = s2.phase; s2.phase = nullptr; sc.steps.push_back(s2); s2t.phase = ph; sc.steps.push_back(s2t); }
        else sc.steps.push_back(s2);
        t2.finish(sc);

        // pass 3: x (tiled): n = x, b = (y in oy_i, z in nz_j); received blocks are x-major => contiguous
        Step s3;
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.nx, 0, "1D FFT X-Direction", s3);
        if (rc) return rc;
        s3.label = "x pass";
        if (ho.CH) {
            // a0 = y_loc, a1 = z block, n = x
            const View out = single_view(nullptr, (long long)nz_j, 0, (long long)(oy_i * nz_j));
            ho.gather(s3, out, 0, oy_i, 0, ho.nzm);
            s3.prm.tile_swz = p->x_swz;
            if (ho.any_rem) {
                Step s3t = ho.gather_tail(s3, out, 0);
                s3t.out_user = 2;
                sc.steps.push_back(s3t);
            }
        } else {
            s3.prm.A0 = 1; s3.prm.A1 = 1; s3.prm.B = int(oy_i * nz_j);
            s3.prm.in = t2.recv({NO_AXIS, NO_AXIS, AX});
            s3.prm.out = single_view(nullptr, 0, 0, (long long)(oy_i * nz_j));
        }
        s3.out_user = 2;
        sc.steps.push_back(s3);
        return DFFT_SUCCESS;
    }

    // ---------------------------------------------------------------------- inverse
    // Reverse order: x, transposition 2', y, transposition 1', z.  Partial d: only the last d of them.
    const PassKind zkind = c2c ? PASS_C2C_CONTIG : PASS_C2R;
    const size_t zlen = c2c ? g.nz : g.nz / 2;
    const long long zpitch_out = z_row_pitch(p);  // output line pitch in complex units

    if (d == 1) {
        Step s;
        rc = new_pass(p, inverse, zkind, zlen, 2, "1D FFT Z-Direction", s);
        if (rc) return rc;
        s.prm.A0 = int(nx_i); s.prm.A1 = int(ny_j);
        s.prm.in = single_view(nullptr, (long long)(ny_j * kzc), (long long)kzc, 1);
        s.in_user = 1;
        s.prm.out = single_view(nullptr, zpitch_out * (long long)ny_j, zpitch_out, 1);
        s.out_user = 2;
        sc.steps.push_back(s);
        return DFFT_SUCCESS;
    }

    if (zyx) {
        // input [nx][ny][nz_me]: y pass (to a slot), x pass scattering along x to the owners of x (dest q holds
        // [nx_q][ny][kzc]), then z inverse on [nx_me][ny][kzc].
        const Transposition t1(p, 1, AX, AZ, g.sx, g.sz, my, tab_x, tab_z);
        Step sy_;
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.ny, 1, nullptr, sy_);
        if (rc) return rc;
        sy_.label = "y pass";
        const int W = t1.direct ? p->slots.D2 : p->slots.SR;  // a local scratch slot that is not the transposition target
        // one rank with x kept: the y pass leaves [nx][ny][kzc] in D1, where the z pass reads it, and no x copy runs (the
        // other decompositions run their d = 2 steps instead, get_schedule)
        const bool no_x = P == 1 && !p->taxes[0];
        sy_.prm.A0 = int(kx); sy_.prm.B = int(nz_j);
        sy_.prm.in = single_view(nullptr, (long long)(ky * nz_j), 0, (long long)nz_j);
        sy_.in_user = 1;
        sy_.prm.out = single_view(p->slot(no_x ? p->slots.D1 : W, me), (long long)(my * nz_j), 0, (long long)nz_j);
        sc.steps.push_back(sy_);
        Step sx_;
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.nx, 0, "2D FFT Y-X-Direction", sx_);
        if (rc) return rc;
        sx_.label = "x pass";
        sx_.prm.A0 = 1; sx_.prm.A1 = int(my); sx_.prm.B = int(nz_j);
        sx_.prm.in = single_view(p->slot(W, me), 0, (long long)nz_j, (long long)(my * nz_j));
        sx_.prm.out = t1.send({NO_AXIS, AY, AX});
        if (!no_x) sc.steps.push_back(sx_);
        t1.finish(sc);
        Step sz_;
        rc = new_pass(p, inverse, zkind, zlen, 2, "1D FFT Z-Direction", sz_);
        if (rc) return rc;
        sz_.prm.A0 = int(nx_i); sz_.prm.A1 = int(my);
        sz_.prm.in = t1.recv({AX, AY, AZ});
        sz_.prm.out = single_view(nullptr, zpitch_out * (long long)my, zpitch_out, 1);
        sz_.out_user = 2;
        sc.steps.push_back(sz_);
        return DFFT_SUCCESS;
    }

    // pencil / slab zy_x inverse: the x pass scatters x over G2 (dest (q, j) holds [nx_q][ky][nz_j]), the y pass scatters y
    // over G1 (dest (i, q) holds [nx_i][ny_q][kzc])
    const bool slab = g.decomp == DFFT_SLAB_ZY_THEN_X;
    const Transposition t2(p, 2, AX, AY, g.sx, g.oy, nz_j, tab_x, tab_y_out);
    const Transposition t1(p, 1, AY, AZ, g.sy, g.sz, nx_i, tab_y_in, tab_z);
    // Blocked hand-over for the inverse as well (HandOver; DFFT_BLOCKED_INV=0 keeps the plain layout): the y pass reads rows
    // nx_i*CH apart instead of one row per (y, z) plane
    const HandOver ho(p, inverse, d == 3 && t2.direct && t1.direct, true, tab_x);
    if (ho.CH) {
        // x pass: in = caller's [nx][oy_i][nz_j]; tile = (y_loc, z block); n = x
        Step s3;
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.nx, 0, "1D FFT X-Direction", s3);
        if (rc) return rc;
        s3.label = "x pass";
        s3.in_user = 1;
        s3.prm.tile_pref = G2.size() > 1 ? p->xchg_tile_pref : 1;
        s3.prm.bulk_out = G2.size() > 1 ? p->bulk_store : 0;
        const View in = single_view(nullptr, (long long)nz_j, 0, (long long)(oy_i * nz_j));
        ho.scatter(s3, in, oy0_i, oy_i, 0, ho.nzm);
        if (ho.any_rem) {
            Step s3t = ho.scatter_tail(s3, in, oy0_i);
            std::swap(s3.phase, s3t.phase);
            sc.steps.push_back(s3);
            sc.steps.push_back(s3t);
        } else {
            sc.steps.push_back(s3);
        }
        t2.finish(sc);
        // y pass: tile = (x_loc, z block); n = y
        Step s2;
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.ny, 1, slab ? nullptr : "1D FFT Y-Direction", s2);
        if (rc) return rc;
        s2.label = "y pass";
        s2.prm.tile_pref = G1.size() > 1 ? p->xchg_tile_pref : 1;
        const View out = t1.send({AX, NO_AXIS, AY});
        ho.gather(s2, out, 0, nx_i, 0, ho.nzm);
        if (ho.any_rem) {
            Step s2t = ho.gather_tail(s2, out, 0);
            std::swap(s2.phase, s2t.phase);
            sc.steps.push_back(s2);
            sc.steps.push_back(s2t);
        } else if (!zy) {
            sc.steps.push_back(s2);
        }
        t1.finish(sc);
        Step s1;
        rc = new_pass(p, inverse, zkind, zlen, 2, slab ? "2D FFT Y-Z-Direction" : "1D FFT Z-Direction", s1);
        if (rc) return rc;
        s1.prm.A0 = int(nx_i); s1.prm.A1 = int(ny_j);
        s1.prm.in = t1.recv({AX, AY, AZ});
        s1.prm.out = single_view(nullptr, zpitch_out * (long long)ny_j, zpitch_out, 1);
        s1.out_user = 2;
        if (zy) {
            if (ho.any_rem || G1.size() > 1 || G2.size() > 1) return fail(DFFT_ERR_STATE, "internal: fused z + y stage");
            Step f;
            rc = fuse_zy(p, s1, s2, "yz pass", s1.phase, f);
            if (rc) return rc;
            sc.steps.push_back(f);
        } else {
            sc.steps.push_back(s1);
        }
        return DFFT_SUCCESS;
    }
    if (d == 3) {
        Step s3;
        rc = new_pass(p, inverse, PASS_C2C_TILED, g.nx, 0, "1D FFT X-Direction", s3);
        if (rc) return rc;
        s3.label = "x pass";
        s3.prm.A0 = 1; s3.prm.A1 = 1; s3.prm.B = int(oy_i * nz_j);
        s3.prm.in = single_view(nullptr, 0, 0, (long long)(oy_i * nz_j));
        s3.in_user = 1;
        if (t2.direct && G2.size() > 1) s3.prm.tile_pref = p->xchg_tile_pref;
        s3.prm.out = t2.send({NO_AXIS, NO_AXIS, AX});
        sc.steps.push_back(s3);
        t2.finish(sc);
    }
    // y pass on [nx_i][ky][nz_j]: from the x pass (d = 3) or the caller's buffer (d = 2)
    Step s2;
    rc = new_pass(p, inverse, PASS_C2C_TILED, g.ny, 1, slab ? nullptr : "1D FFT Y-Direction", s2);
    if (rc) return rc;
    s2.label = "y pass";
    s2.prm.A0 = int(nx_i); s2.prm.A1 = 1; s2.prm.B = int(nz_j);
    if (d == 3) {
        s2.prm.in = t2.recv({AX, NO_AXIS, AY});
    } else {
        s2.prm.in = single_view(nullptr, (long long)(ky * nz_j), 0, (long long)nz_j);
        s2.in_user = 1;
    }
    if (t1.direct && G1.size() > 1) s2.prm.tile_pref = p->xchg_tile_pref;
    s2.prm.out = t1.send({AX, NO_AXIS, AY});
    sc.steps.push_back(s2);
    t1.finish(sc);
    // z pass on [nx_i][ny_j][kzc]
    Step s1;
    rc = new_pass(p, inverse, zkind, zlen, 2, slab ? "2D FFT Y-Z-Direction" : "1D FFT Z-Direction", s1);
    if (rc) return rc;
    s1.prm.A0 = int(nx_i); s1.prm.A1 = int(ny_j);
    s1.prm.in = t1.recv({AX, AY, AZ});
    s1.prm.out = single_view(nullptr, zpitch_out * (long long)ny_j, zpitch_out, 1);
    s1.out_user = 2;
    sc.steps.push_back(s1);
    return DFFT_SUCCESS;
}

// 1D plans (dfft_plan_create_1d, DESIGN.md section 3.22): the N-point signal as the slab grid [N1][N2][N3], each rank
// holding an x-slab [nx_i][N2][N3] of it on both sides.  Forward:
//   transpose  copy pass along y: my x-slab into every rank's y-slab [N1][oy_q][N3] (slot D1, or the all-to-all slots)
//   x pass     gathers x, scatters it back to x-slabs (slot D2 or the all-to-all slots): the 3D inverse's x pass
//   y pass     each point n2 of line (k1, n3) loaded times W_(N1 N2)^(n2 k1) = W_N^(n2 k1 N3), into slot D1
//   z pass     each point n3 of line (k1, k2) loaded times W_N^(n3 (k1 + N1 k2)), into the caller's out
// out[k1][k2][k3] = X[k1 + N1 k2 + N1 N2 k3], FFTW-MPI's scrambled order.  The inverse is the adjoint: the z and y passes
// store times the conjugate twiddles, then the 3D forward's y -> x transposition and x pass, and the copy back to x-slabs.
// On one rank the copy passes are not needed: the x pass reads the caller's in (forward) or writes its out (inverse).
// Every slot is free when a peer stores into it: D1 (forward) was last read by the z pass of the previous exec, before
// the entry rendezvous, and D2 by nobody; inverse, D1 was read by the y pass before the rendezvous of the y -> x
// transposition.
// Natural-order plans (dfft_plan_create_1d_natural, DESIGN.md section 3.23) hold their spectrum as [N3][N2][N1], each rank
// the chunk [oz_i][N2][N1] of the N3 split p->oz.  Their z pass runs TILED in its transposing form (Twiddle1d::sB): it reads
// the rows [k1][k2][:] of my x-slab and scatters k3 to the owners' chunks, at column x0_i.  On one rank it stores into the
// caller's out (forward) or reads its in (inverse).  On more ranks:
//   forward  ... y pass | rendezvous | z pass into every rank's D2 | rendezvous | landing copy: D2 -> the caller's out
//   inverse  scatter copy: the caller's in -> every rank's D2 [N3][N2][nx_q] | rendezvous | z pass: D2 -> D1 | rendezvous
//            | the y pass, x pass and copy of the scrambled inverse
// The landing slot is D2: forward its last reader is my y pass, inverse the next writer into it is a peer's y pass, so a
// rendezvous between the y and z passes frees it without a slot more.  All-to-all plans exchange through SS / SR
// instead, in stream order, and need no such rendezvous.
static int build_1d(dfft_plan_s* p, int inverse, Schedule& sc) {
    const Geometry& g = p->g;
    const int me = p->rank, P = p->P;
    const size_t nx_i = g.sx.size[me], x0_i = g.sx.start[me], oy_i = g.oy.size[me], ny = g.ny, nz = g.nz;
    Tables& T = p->tabs;
    int rc;
    const unsigned char *tab_y = nullptr, *tab_x = nullptr;
    if (P > 1 && (T.seg_table(g.oy, &tab_y) != cudaSuccess || T.seg_table(g.sx, &tab_x) != cudaSuccess)) return fail(DFFT_ERR_CUDA, "segment table");
    if (p->any_direct) sc.steps.push_back(new_rendezvous(0, 0, nullptr, 0));
    // x-slabs -> y-slabs (the 3D forward's y -> x transposition) into slot D1, and back (the 3D inverse's x -> y one)
    const Transposition to_y(p, 2, AY, AX, g.oy, g.sx, nz, tab_y, tab_x, inverse ? -1 : p->slots.D1);
    const Transposition to_x(p, 2, AX, AY, g.sx, g.oy, nz, tab_x, tab_y, inverse ? p->slots.D1 : -1);
    void* d1 = p->slot(p->slots.D1, me);
    const bool natural = !p->oz.size.empty();
    const unsigned char* tab_z = nullptr;
    if (natural && P > 1 && T.seg_table(p->oz, &tab_z) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
    void* tw = nullptr;
    if (T.get_tw1d(ilog2_exact(p->n1d), &tw) != cudaSuccess) return fail(DFFT_ERR_CUDA, "twiddle table allocation failed");
    // the y and z passes over my x-slab [nx_i][N2][N3] in slot D1 and the caller's buffer, twiddled
    auto twiddled = [&](int axis, Step& s) -> int {
        rc = axis == 1 ? new_pass(p, inverse, PASS_C2C_TILED, ny, 1, nullptr, s) : new_pass(p, inverse, PASS_C2C_CONTIG, nz, 2, nullptr, s);
        if (rc) return rc;
        s.twiddle = axis == 1 ? "y" : "z";
        s.tw = Twiddle1d{tw, (long long)x0_i, axis == 1 ? 0 : (long long)g.nx, axis == 1 ? (long long)nz : 1, ilog2_exact(p->n1d)};
        if (axis == 1) {
            s.label = "y pass";
            s.prm.A0 = int(nx_i); s.prm.A1 = 1; s.prm.B = int(nz);
            s.prm.in = s.prm.out = single_view(d1, (long long)(ny * nz), 0, (long long)nz);
        } else {  // forward from slot D1 into the caller's out, inverse from the caller's in into slot D1
            s.prm.A0 = int(nx_i); s.prm.A1 = int(ny);
            s.prm.in = single_view(inverse ? nullptr : d1, (long long)(ny * nz), (long long)nz, 1);
            s.prm.out = single_view(inverse ? d1 : nullptr, (long long)(ny * nz), (long long)nz, 1);
            if (inverse) s.in_user = 1;
            else s.out_user = 2;
        }
        return DFFT_SUCCESS;
    };
    // the copy pass between my x-slab on the caller's side and the y-slabs (one line per (x, z), n = y)
    auto transpose = [&](const View& in, const View& out, Step& s) {
        s = Step();
        s.label = "transpose";
        s.kind = PASS_COPY_TILED;
        s.n = ny;
        s.axis = 1;
        s.prm.A0 = int(nx_i); s.prm.A1 = 1; s.prm.B = int(nz);
        s.prm.inverse = inverse;
        s.prm.in = in;
        s.prm.out = out;
    };
    const View slab = single_view(nullptr, (long long)(ny * nz), 0, (long long)nz);
    Step x, y, z, c;
    rc = new_pass(p, inverse, PASS_C2C_TILED, g.nx, 0, "1D FFT X-Direction", x);
    if (rc) return rc;
    x.label = "x pass";
    x.prm.A0 = 1; x.prm.A1 = 1; x.prm.B = int(oy_i * nz);
    if ((rc = twiddled(1, y)) || (rc = twiddled(2, z))) return rc;
    // the z pass and, natural order on more ranks, its exchange and copy
    auto push_z = [&]() {
        z.phase = inverse ? nullptr : "2D FFT Y-Z-Direction";
        if (!natural) { sc.steps.push_back(z); return; }
        // the transposing z pass: tiles of TB consecutive k1 of one k2 (a0 = k2, b = k1 - x0_i), its row side my x-slab in
        // slot D1, lines N2 N3 apart; the other side [k3][k2][k1] with k1 contiguous
        z.kind = PASS_C2C_TILED;
        z.prm.A0 = int(ny); z.prm.A1 = 1; z.prm.B = int(nx_i);
        z.tw.sB = (long long)(ny * nz);
        const View rows = single_view(d1, (long long)nz, 0, 1);
        const View chunk = single_view(nullptr, (long long)g.nx, 0, (long long)(ny * g.nx));  // [N3][N2][N1] (one rank)
        z.in_user = z.out_user = 0;
        if (inverse) { z.prm.in = chunk; z.in_user = 1; z.prm.out = rows; }
        else { z.prm.in = rows; z.prm.out = chunk; z.out_user = 2; }
        if (P == 1) { sc.steps.push_back(z); return; }
        // the output chunks [oz_q][N2][N1] as boxes with k3, k2, k1 for x, y, z: the forward z pass sends k3 to its owners at
        // column x0_i, the inverse scatter copy k1 to the x-slabs [N3][N2][nx_q] at row z0_i
        const Transposition to_n(p, 2, AX, AZ, p->oz, g.sx, ny, tab_z, tab_x), from_n(p, 2, AZ, AX, g.sx, p->oz, ny, tab_x, tab_z);
        // the copy between the caller's chunk and the landing slot, one line per (k3, k2), n = k1
        auto natural_copy = [&](const char* label, const View& in, const View& out, Step& s) {
            s = Step();
            s.label = label;
            s.kind = PASS_COPY_CONTIG;
            s.n = g.nx;
            s.axis = 2;
            s.prm.A0 = int(p->oz.size[me]); s.prm.A1 = int(ny); s.prm.B = 1;
            s.prm.inverse = inverse;
            s.prm.in = in;
            s.prm.out = out;
        };
        const View mine = single_view(nullptr, (long long)(ny * g.nx), (long long)g.nx, 1);
        z.prm.tile_pref = p->xchg_tile_pref;
        if (!inverse) {
            z.out_user = 0;
            z.prm.out = to_n.send({AY, NO_AXIS, AX});
            if (to_n.direct) sc.steps.push_back(new_rendezvous(2, 2, nullptr, 0));  // my y pass has read D2
            sc.steps.push_back(z);
            to_n.finish(sc);
            natural_copy("landing copy", to_n.recv({AX, AY, AZ}), mine, c);
            c.out_user = 2;
            sc.steps.push_back(c);
            return;
        }
        natural_copy("scatter copy", mine, from_n.send({AX, AY, AZ}), c);
        c.in_user = 1;
        sc.steps.push_back(c);
        from_n.finish(sc);
        z.in_user = 0;
        z.prm.in = from_n.recv({AY, NO_AXIS, AX});
        sc.steps.push_back(z);
        if (from_n.direct) sc.steps.push_back(new_rendezvous(2, 2, nullptr, 0));  // every z pass has read D2
    };
    if (!inverse) {
        if (P > 1) {
            transpose(slab, to_y.send({AX, NO_AXIS, AY}), c);
            c.in_user = 1;
            sc.steps.push_back(c);
            to_y.finish(sc);
            x.prm.in = to_y.recv({NO_AXIS, NO_AXIS, AX});
        } else {
            x.prm.in = single_view(nullptr, 0, 0, (long long)(ny * nz));
            x.in_user = 1;
        }
        x.prm.out = to_x.send({NO_AXIS, NO_AXIS, AX});
        sc.steps.push_back(x);
        to_x.finish(sc);
        y.prm.in = to_x.recv({AX, NO_AXIS, AY});
        sc.steps.push_back(y);
        push_z();
        return DFFT_SUCCESS;
    }
    push_z();
    y.prm.out = to_y.send({AX, NO_AXIS, AY});
    y.phase = "2D FFT Y-Z-Direction";
    sc.steps.push_back(y);
    to_y.finish(sc);
    x.prm.in = to_y.recv({NO_AXIS, NO_AXIS, AX});
    if (P > 1) {
        x.prm.out = to_x.send({NO_AXIS, NO_AXIS, AX});
        sc.steps.push_back(x);
        to_x.finish(sc);
        transpose(to_x.recv({AX, NO_AXIS, AY}), slab, c);
        c.out_user = 2;
        sc.steps.push_back(c);
    } else {
        x.prm.out = single_view(nullptr, 0, 0, (long long)(ny * nz));
        x.out_user = 2;
        sc.steps.push_back(x);
    }
    return DFFT_SUCCESS;
}

}  // namespace dfft

namespace dfft {

// Overlapped schedules, Peer2Peer on every transposition (send_method Streams): slab ZY_Then_X and pencil.
//
// The reference's Streams variant overlaps pack(q+1) with send(q) (mpicufft_slab.cpp:398-415).  Here the exchanges are
// FFT passes that store straight into the peers' slots, so the overlap is between whole FFT passes.  Forward, one builder
// for both: a slab is the pencil grid with one-member row groups (G1 = {me}), whose z pass stores into my own slot A and
// whose y pass waits for it without a rendezvous:
//   stream 0: z pass per plane group, scattering along z into the row peers' slot A             (HBM / NVLink-bound)
//   stream 1: per plane group: meet the row peers; then the y pass per (plane group, z chunk), persistent on
//             `xchg_ctas` CTAs, scattering along y into the column peers' slot B                 (NVLink-bound)
//   stream 2: per z chunk: meet the column peers, x pass of that chunk                           (HBM-bound)
// The y pass of chunk c+1 runs while the x pass consumes chunk c, and while later plane groups are still in the z pass.
// On a pencil grid only the x pass can hide behind an exchange (both scatters share the NVLink ports).
// Slab inverse: x pass per z chunk scatters (stream 1), y pass per chunk follows (stream 2), the z pass runs last on the
// caller's stream.  Pencil inverse: it mirrors the forward one — again only the local pass, now the z pass, can hide:
//   stream 0: x pass, scattering along x into the column peers' slot B; meet the column peers   (NVLink-bound)
//   stream 1: y pass per plane group on a capped grid, scattering along y into the row peers' slot A  (NVLink-bound)
//   stream 2: per plane group: meet the row peers, z pass of that group into the caller's buffer  (HBM-bound)
static int exchange_ctas(const dfft_plan_s* p, int inverse) {
    const int t = p->tuned_ctas[inverse ? 1 : 0];
    return t != -2 ? t : p->xchg_ctas;
}

// Plane groups of the overlapped z / y passes and z chunks of their y / x passes: every rank must build the same number
// of steps, so both derive from global minima
static size_t plane_groups(const dfft_plan_s* p, int inverse) {
    size_t min_nx = p->g.nx;
    for (size_t v : p->g.sx.size) min_nx = std::min(min_nx, v);
    return std::min<size_t>(size_t(inverse && p->tuned_groups_inv > 0 ? p->tuned_groups_inv : p->ovl_groups), min_nx);
}
static size_t z_chunk_count(const dfft_plan_s* p, int inverse) {
    size_t min_nz = p->g.nzc;
    for (size_t v : p->g.sz.size) min_nz = std::min(min_nz, v);
    const int t = p->tuned_chunks[inverse ? 1 : 0];
    const size_t want = size_t(t > 0 ? t : p->ovl_chunks);
    return min_nz >= 32 * want ? want : (min_nz >= 32 ? 2 : 1);
}

static int build_overlapped_forward(dfft_plan_s* p, Schedule& sc) {
    const Geometry& g = p->g;
    const int me = p->rank;
    const int pi = g.pi(me), pj = g.pj(me);
    const size_t es = p->esize;
    const bool c2c = g.transform == DFFT_C2C;
    Tables& T = p->tabs;
    sc.overlapped = true;
    const size_t ny = g.ny;
    const size_t nx_i = g.sx.size[pi], x0_i = g.sx.start[pi];
    const size_t ny_j = g.sy.size[pj];
    const size_t nz_j = g.sz.size[pj];
    const size_t oy_i = g.oy.size[pi];
    const std::vector<int>& G2 = p->grp[2];
    int nev = 0;

    const size_t NG = plane_groups(p, 0), NS = z_chunk_count(p, 0);
    Split groups;
    groups.make(nx_i, NG);
    // a slab has no first transposition: its z pass stores into my own slot A
    const bool pencil = g.decomp == DFFT_PENCIL;
    const unsigned char *tab_z = nullptr, *tab_y = nullptr;
    if ((pencil && T.seg_table(g.sz, &tab_z) != cudaSuccess) || T.seg_table(g.oy, &tab_y) != cudaSuccess)
        return fail(DFFT_ERR_CUDA, "segment table");
    const Transposition t1(p, 1, AZ, AY, g.sz, g.sy, nx_i, tab_z, nullptr), t2(p, 2, AY, AX, g.oy, g.sx, nz_j, tab_y, nullptr);
    const HandOver ho(p, 0, true, false, tab_y);
    const Split chunks = ho.chunks(NS);
    // the ranks of a pencil grid hold different z extents: a chunk count clamped to one rank's blocks could differ
    // between them
    if (pencil && chunks.size.size() != NS) return fail(DFFT_ERR_STATE, "internal: blocked z chunks");
    const size_t NSc = chunks.size.size();

    sc.steps.push_back(new_rendezvous(0, 0, nullptr, 0));  // everyone has left the previous exec
    // the auxiliary streams fork from the caller's stream at the start of run_schedule, i.e. BEFORE the
    // entry rendezvous: make them wait for it explicitly
    const int ev_entry = nev++;
    sc.steps.back().record = ev_entry;
    int rc;
    std::vector<int> ev_z(NG), ev_y(NSc);
    for (size_t gi = 0; gi < NG; ++gi) {
        Step s;
        rc = new_pass(p, 0, c2c ? PASS_C2C_CONTIG : PASS_R2C, c2c ? g.nz : g.nz / 2, 2, nullptr, s);
        if (rc) return rc;
        const size_t pl0 = groups.start[gi], npl = groups.size[gi];
        const long long pitch = z_row_pitch(p);
        s.prm.A0 = int(npl); s.prm.A1 = int(ny_j);
        s.prm.in = single_view((void*)(size_t)(pl0 * ny_j * pitch * es), pitch * (long long)ny_j, pitch, 1);
        s.in_user = 1;
        s.prm.out = t1.send({AX, AY, AZ}, {pl0, 0, 0});
        s.record = ev_z[gi] = nev++;
        sc.steps.push_back(s);
    }
    for (size_t c = 0; c < NSc; ++c) {
        const size_t z0 = chunks.start[c], zc = chunks.size[c];
        for (size_t gi = 0; gi < NG; ++gi) {
            const size_t pl0 = groups.start[gi], npl = groups.size[gi];
            Step s;
            rc = new_pass(p, 0, PASS_C2C_TILED, ny, 1, nullptr, s);
            if (rc) return rc;
            s.label = "y pass";
            if (c == 0) {
                // plane group gi has arrived: at a rendezvous with the row peers, or (slab) straight from my own z pass
                std::vector<int> w{ev_z[gi]};
                if (gi == 0) w.push_back(ev_entry);
                if (pencil) {
                    Step r = new_rendezvous(1, 1, nullptr, 1);
                    r.waits = w;
                    sc.steps.push_back(r);
                } else {
                    s.waits = w;
                }
            }
            const View in = t1.recv({AX, NO_AXIS, AY}, {pl0, 0, 0});
            if (ho.CH) {
                s.prm.bulk_out = G2.size() > 1 ? p->bulk_store : 0;
                ho.scatter(s, in, x0_i + pl0, npl, z0, zc);
            } else {
                s.prm.A0 = int(npl); s.prm.A1 = 1; s.prm.B = int(zc);
                s.prm.in = t1.recv({AX, NO_AXIS, AY}, {pl0, 0, z0});
                s.prm.out = t2.send({AX, NO_AXIS, AY}, {pl0, 0, z0});
            }
            s.prm.max_ctas = exchange_ctas(p, 0);
            s.prm.tile_pref = G2.size() > 1 ? p->xchg_tile_pref : 0;
            s.stream = 1;
            const bool tail_here = ho.any_rem && c + 1 == NSc;
            if (gi + 1 == NG && !tail_here) s.record = ev_y[c] = nev++;
            sc.steps.push_back(s);
            if (tail_here) {
                Step t = ho.scatter_tail(s, in, x0_i + pl0);
                if (gi + 1 == NG) t.record = ev_y[c] = nev++;
                sc.steps.push_back(t);
            }
        }
    }
    const View out = single_view(nullptr, (long long)nz_j, 0, (long long)(oy_i * nz_j));
    for (size_t c = 0; c < NSc; ++c) {
        const size_t z0 = chunks.start[c], zc = chunks.size[c];
        Step r = new_rendezvous(2, 2, nullptr, 2);
        r.waits.push_back(ev_y[c]);
        sc.steps.push_back(r);
        Step s;
        rc = new_pass(p, 0, PASS_C2C_TILED, g.nx, 0, nullptr, s);
        if (rc) return rc;
        s.label = "x pass";
        if (ho.CH) {
            ho.gather(s, out, 0, oy_i, z0, zc);
            s.prm.tile_swz = p->x_swz;
        } else {
            s.prm.A0 = 1; s.prm.A1 = int(oy_i); s.prm.B = int(zc);
            s.prm.in = t2.recv({NO_AXIS, AY, AX}, {0, 0, z0});
            s.prm.out = single_view((void*)(size_t)(z0 * es), 0, (long long)nz_j, (long long)(oy_i * nz_j));
        }
        s.out_user = 2;
        s.stream = 2;
        sc.steps.push_back(s);
        if (ho.any_rem && c + 1 == NSc) sc.steps.push_back(ho.gather_tail(s, out, 0));
    }
    sc.nevents = nev;
    return DFFT_SUCCESS;
}

static int build_overlapped_slab_inverse(dfft_plan_s* p, Schedule& sc) {
    const Geometry& g = p->g;
    const int me = p->rank;
    const size_t es = p->esize;
    const bool c2c = g.transform == DFFT_C2C;
    Tables& T = p->tabs;
    sc.overlapped = true;
    const size_t nzc = g.nzc, ny = g.ny;
    const size_t nx_p = g.sx.size[me];
    const size_t oy_me = g.oy.size[me], oy0_me = g.oy.start[me];
    int nev = 0;

    const unsigned char* tab_x = nullptr;
    if (T.seg_table(g.sx, &tab_x) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
    // dest q holds [nx_q][ny][nzc]
    const Transposition t2(p, 2, AX, AY, g.sx, g.oy, nzc, tab_x, nullptr);
    const HandOver ho(p, 1, true, false, tab_x);
    const Split chunks = ho.chunks(z_chunk_count(p, 1));
    const size_t NSc = chunks.size.size();

    sc.steps.push_back(new_rendezvous(0, 0, nullptr, 0));  // everyone has left the previous exec
    const int ev_entry = nev++;  // which the auxiliary streams wait for (build_overlapped_forward)
    sc.steps.back().record = ev_entry;
    int rc;
    std::vector<int> ev_x(NSc), ev_yi(NSc);
    const View in = single_view(nullptr, (long long)nzc, 0, (long long)(oy_me * nzc));
    for (size_t c = 0; c < NSc; ++c) {
        const size_t z0 = chunks.start[c], zc = chunks.size[c];
        Step s;
        rc = new_pass(p, 1, PASS_C2C_TILED, g.nx, 0, nullptr, s);
        if (rc) return rc;
        s.label = "x pass";
        s.in_user = 1;
        if (ho.CH) {
            s.prm.bulk_out = p->bulk_store;
            ho.scatter(s, in, oy0_me, oy_me, z0, zc);
        } else {
            s.prm.A0 = 1; s.prm.A1 = int(oy_me); s.prm.B = int(zc);
            s.prm.in = single_view((void*)(size_t)(z0 * es), 0, (long long)nzc, (long long)(oy_me * nzc));
            s.prm.out = t2.send({NO_AXIS, AY, AX}, {0, 0, z0});
        }
        s.prm.max_ctas = exchange_ctas(p, 1);
        s.prm.tile_pref = p->xchg_tile_pref;
        s.stream = 1;
        if (c == 0) s.waits.push_back(ev_entry);
        const bool tail_here = ho.any_rem && c + 1 == NSc;
        if (!tail_here) s.record = ev_x[c] = nev++;
        sc.steps.push_back(s);
        if (tail_here) {
            Step t = ho.scatter_tail(s, in, oy0_me);
            t.record = ev_x[c] = nev++;
            sc.steps.push_back(t);
        }
    }
    const View out = single_view(p->slot(p->slots.D1, me), (long long)(ny * nzc), 0, (long long)nzc);
    for (size_t c = 0; c < NSc; ++c) {
        const size_t z0 = chunks.start[c], zc = chunks.size[c];
        Step r = new_rendezvous(2, 2, nullptr, 2);
        r.waits.push_back(ev_x[c]);
        sc.steps.push_back(r);
        Step s;
        rc = new_pass(p, 1, PASS_C2C_TILED, ny, 1, nullptr, s);
        if (rc) return rc;
        s.label = "y pass";
        s.stream = 2;
        if (ho.CH) {
            s.prm.tile_pref = 1;
            ho.gather(s, out, 0, nx_p, z0, zc);
            const bool tail_here = ho.any_rem && c + 1 == NSc;
            if (!tail_here) s.record = ev_yi[c] = nev++;
            sc.steps.push_back(s);
            if (tail_here) {
                Step t = ho.gather_tail(s, out, 0);
                t.record = ev_yi[c] = nev++;
                sc.steps.push_back(t);
            }
        } else {
            s.prm.A0 = int(nx_p); s.prm.A1 = 1; s.prm.B = int(zc);
            s.prm.in = t2.recv({AX, NO_AXIS, AY}, {0, 0, z0});
            s.prm.out = s.prm.in;  // in place
            s.record = ev_yi[c] = nev++;
            sc.steps.push_back(s);
        }
    }
    Step s;
    const long long zpitch = z_row_pitch(p);
    rc = new_pass(p, 1, c2c ? PASS_C2C_CONTIG : PASS_C2R, c2c ? g.nz : g.nz / 2, 2, nullptr, s);
    if (rc) return rc;
    s.prm.A0 = int(nx_p); s.prm.A1 = int(ny);
    s.prm.in = single_view(p->slot(ho.CH ? p->slots.D1 : p->slots.D2, me), (long long)(ny * nzc), (long long)nzc, 1);
    s.prm.out = single_view(nullptr, zpitch * (long long)ny, zpitch, 1);
    s.out_user = 2;
    for (size_t c = 0; c < NSc; ++c) s.waits.push_back(ev_yi[c]);
    sc.steps.push_back(s);
    sc.nevents = nev;
    return DFFT_SUCCESS;
}

}  // namespace dfft

namespace dfft {

// DFFT_PENCIL_OVERLAP: 1 (default) = Streams plans on a grid with two real transpositions run the forward overlapped
// schedule, and dfft_plan_tune may select an overlapped schedule for any grid and direction after measuring it;
// 0 = sequential schedules only; 2 = overlapped schedules wherever they can be built, untuned (tests, experiments).
static int pencil_overlap_mode() {
    const char* e = getenv("DFFT_PENCIL_OVERLAP");
    return e ? atoi(e) : 1;
}
static bool pencil_overlap_enabled() { return pencil_overlap_mode() != 0; }

static int build_overlapped_pencil_inverse(dfft_plan_s* p, Schedule& sc) {
    const Geometry& g = p->g;
    const int me = p->rank;
    const int pi = g.pi(me), pj = g.pj(me);
    const size_t es = p->esize;
    const bool c2c = g.transform == DFFT_C2C;
    Tables& T = p->tabs;
    sc.overlapped = true;
    const size_t ny = g.ny, nx = g.nx;
    const size_t nx_i = g.sx.size[pi];
    const size_t ny_j = g.sy.size[pj];
    const size_t nz_j = g.sz.size[pj];
    const size_t oy_i = g.oy.size[pi], oy0_i = g.oy.start[pi];
    const std::vector<int>& G1 = p->grp[1];
    const std::vector<int>& G2 = p->grp[2];
    int nev = 0;
    const size_t NG = plane_groups(p, 1);
    Split groups;
    groups.make(nx_i, NG);
    const unsigned char *tab_x = nullptr, *tab_y_in = nullptr;
    if (T.seg_table(g.sx, &tab_x) != cudaSuccess || T.seg_table(g.sy, &tab_y_in) != cudaSuccess) return fail(DFFT_ERR_CUDA, "segment table");
    // dest (q, j) holds [nx_q][ny][nz_j], dest (i, q) [nx_i][ny_q][nzc]
    const Transposition t2(p, 2, AX, AY, g.sx, g.oy, nz_j, tab_x, nullptr), t1(p, 1, AY, AZ, g.sy, g.sz, nx_i, tab_y_in, nullptr);
    const HandOver ho(p, 1, true, false, tab_x);
    int rc;

    sc.steps.push_back(new_rendezvous(0, 0, nullptr, 0));  // everyone has left the previous exec
    // x pass on the caller's [nx][oy_i][nz_j], whole, uncapped: nothing local can run beside it yet
    {
        Step s;
        rc = new_pass(p, 1, PASS_C2C_TILED, nx, 0, nullptr, s);
        if (rc) return rc;
        s.label = "x pass";
        s.in_user = 1;
        s.prm.tile_pref = G2.size() > 1 ? p->xchg_tile_pref : 1;
        if (ho.CH) {
            s.prm.bulk_out = G2.size() > 1 ? p->bulk_store : 0;
            const View in = single_view(nullptr, (long long)nz_j, 0, (long long)(oy_i * nz_j));
            ho.scatter(s, in, oy0_i, oy_i, 0, ho.nzm);
            sc.steps.push_back(s);
            if (ho.any_rem) sc.steps.push_back(ho.scatter_tail(s, in, oy0_i));
        } else {
            s.prm.A0 = 1; s.prm.A1 = 1; s.prm.B = int(oy_i * nz_j);
            s.prm.in = single_view(nullptr, 0, 0, (long long)(oy_i * nz_j));
            s.prm.out = t2.send({NO_AXIS, NO_AXIS, AX});
            sc.steps.push_back(s);
        }
    }
    sc.steps.push_back(new_rendezvous(2, 2, nullptr, 0));  // all column peers have delivered their rows
    const int ev_x = nev++;
    sc.steps.back().record = ev_x;
    std::vector<int> ev_y(NG);
    for (size_t gi = 0; gi < NG; ++gi) {
        const size_t pl0 = groups.start[gi], npl = groups.size[gi];
        Step s;
        rc = new_pass(p, 1, PASS_C2C_TILED, ny, 1, nullptr, s);
        if (rc) return rc;
        s.label = "y pass";
        s.stream = 1;
        if (gi == 0) s.waits.push_back(ev_x);
        s.prm.max_ctas = exchange_ctas(p, 1);
        s.prm.tile_pref = G1.size() > 1 ? p->xchg_tile_pref : 1;
        const View out = t1.send({AX, NO_AXIS, AY}, {pl0, 0, 0});
        if (ho.CH) {
            ho.gather(s, out, pl0, npl, 0, ho.nzm);
            if (!ho.any_rem) s.record = ev_y[gi] = nev++;
            sc.steps.push_back(s);
            if (ho.any_rem) {
                Step t = ho.gather_tail(s, out, pl0);
                t.record = ev_y[gi] = nev++;
                sc.steps.push_back(t);
            }
        } else {
            s.prm.A0 = int(npl); s.prm.A1 = 1; s.prm.B = int(nz_j);
            s.prm.in = t2.recv({AX, NO_AXIS, AY}, {pl0, 0, 0});
            s.prm.out = out;
            s.record = ev_y[gi] = nev++;
            sc.steps.push_back(s);
        }
    }
    const PassKind zkind = c2c ? PASS_C2C_CONTIG : PASS_C2R;
    const long long zpitch = z_row_pitch(p);  // output line pitch in complex units
    for (size_t gi = 0; gi < NG; ++gi) {
        const size_t pl0 = groups.start[gi], npl = groups.size[gi];
        Step r = new_rendezvous(1, 1, nullptr, 2);  // all row peers have delivered plane group gi
        r.waits.push_back(ev_y[gi]);
        sc.steps.push_back(r);
        Step s;
        rc = new_pass(p, 1, zkind, c2c ? g.nz : g.nz / 2, 2, nullptr, s);
        if (rc) return rc;
        s.prm.A0 = int(npl); s.prm.A1 = int(ny_j);
        s.prm.in = t1.recv({AX, AY, AZ}, {pl0, 0, 0});
        s.prm.out = single_view((void*)(size_t)(pl0 * ny_j * size_t(zpitch) * es), zpitch * (long long)ny_j, zpitch, 1);
        s.out_user = 2;
        s.stream = 2;
        sc.steps.push_back(s);
    }
    sc.nevents = nev;
    return DFFT_SUCCESS;
}

}  // namespace dfft

// =====================================================================================================
// memory / peer mapping
// =====================================================================================================
static int nccl_allgather_bytes(dfft_plan_s* p, const void* mine, size_t bytes, std::vector<char>& all) {
    const int P = p->P;
    all.assign(bytes * P, 0);
    if (P == 1) {
        memcpy(all.data(), mine, bytes);
        return DFFT_SUCCESS;
    }
    char* d = nullptr;
    CK_CUDA(cudaMalloc(&d, bytes * (P + 1)));
    CK_CUDA(cudaMemcpy(d + bytes * P, mine, bytes, cudaMemcpyHostToDevice));
    CK_NCCL(ncclAllGather(d + bytes * P, d, bytes, ncclChar, p->comm->nccl, p->own_stream));
    CK_CUDA(cudaStreamSynchronize(p->own_stream));
    CK_CUDA(cudaMemcpy(all.data(), d, bytes * P, cudaMemcpyDeviceToHost));
    CK_CUDA(cudaFree(d));
    return DFFT_SUCCESS;
}

// Base address and size of the allocation that contains `ptr` (driver API cuMemGetAddressRange, resolved at run time
// through the runtime so that libdfft.so does not link libcuda).
static bool alloc_range(const void* ptr, unsigned long long* base, size_t* span) {
    typedef int (*fn_t)(unsigned long long*, size_t*, unsigned long long);
    static fn_t fn = nullptr;
    if (!fn) {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) != cudaSuccess || !f) {
            cudaGetLastError();
            return false;
        }
        fn = (fn_t)f;
    }
    return fn(base, span, (unsigned long long)ptr) == 0;
}

static void plan_release_memory(dfft_plan_s* p) {
    for (void* q : p->opened) cudaIpcCloseMemHandle(q);
    p->opened.clear();
    if (p->work && p->work_owned) cudaFree(p->work);
    p->work = nullptr;
    p->work_owned = false;
    p->slot_ptr.clear();
    for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 3; ++b) p->sched[a][b] = Schedule();
    p->tabs.release_seg_tables();
}

static int plan_setup_memory(dfft_plan_s* p, void* user_device) {
    plan_release_memory(p);
    const int P = p->P, me = p->rank;
    if (user_device) {
        p->work = user_device;
        p->work_owned = false;
    } else {
        CK_CUDA(cudaMalloc(&p->work, p->work_bytes));
        p->work_owned = true;
    }
    p->slot_ptr.assign(p->nslots, std::vector<void*>(P, nullptr));
    for (int s = 0; s < p->nslots; ++s) p->slot_ptr[s][me] = (char*)p->work + size_t(s) * p->slot_bytes;
    if (p->any_direct) {
        // A caller-supplied work area may sit INSIDE a larger allocation (a tensor of a caching allocator): the IPC
        // handle then names the whole allocation and cudaIpcOpenMemHandle returns its base on the peer, so the byte
        // offset of the work area inside its allocation travels with the handle.
        cudaIpcMemHandle_t h;
        cudaError_t e = cudaIpcGetMemHandle(&h, p->work);
        int ok = (e == cudaSuccess) ? 1 : 0;
        if (!ok) cudaGetLastError();
        unsigned long long offset = 0;
        if (ok) {
            unsigned long long base = 0;
            size_t span = 0;
            if (!alloc_range(p->work, &base, &span)) ok = 0;
            else {
                offset = (unsigned long long)p->work - base;
                if (offset + p->work_bytes > span) ok = 0;  // the area does not fit its allocation
            }
        }
        struct Rec { cudaIpcMemHandle_t h; int ok; int pad; unsigned long long offset; } rec{};
        rec.h = h; rec.ok = ok; rec.offset = offset;
        std::vector<char> all;
        int rc = nccl_allgather_bytes(p, &rec, sizeof(rec), all);
        if (rc) return rc;
        for (int r = 0; r < P; ++r) {
            const Rec* rr = reinterpret_cast<const Rec*>(all.data()) + r;
            if (!rr->ok) return fail(DFFT_ERR_PEER, "rank " + std::to_string(r) + ": work area is not exportable with cudaIpcGetMemHandle "
                                                    "(it must lie inside one cudaMalloc allocation that holds getWorkSizeDevice() bytes from "
                                                    "the given pointer); use comm_method All2All");
        }
        for (int r = 0; r < P; ++r) {
            if (r == me) continue;
            const Rec* rr = reinterpret_cast<const Rec*>(all.data()) + r;
            void* mapped = nullptr;
            e = cudaIpcOpenMemHandle(&mapped, rr->h, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                cudaGetLastError();
                return fail(DFFT_ERR_PEER, std::string("cudaIpcOpenMemHandle failed: ") + cudaGetErrorString(e));
            }
            p->opened.push_back(mapped);
            for (int s = 0; s < p->nslots; ++s) p->slot_ptr[s][r] = (char*)mapped + rr->offset + size_t(s) * p->slot_bytes;
        }
    }
    return DFFT_SUCCESS;
}

static int plan_setup_flags(dfft_plan_s* p) {
    const int P = p->P, me = p->rank;
    CK_CUDA(cudaMalloc(&p->flags, sizeof(unsigned long long) * NPHASE * P));
    CK_CUDA(cudaMemset(p->flags, 0, sizeof(unsigned long long) * NPHASE * P));
    CK_CUDA(cudaMalloc(&p->err_d, sizeof(int)));
    CK_CUDA(cudaMemset(p->err_d, 0, sizeof(int)));
    std::vector<unsigned long long*> pf(P, nullptr);
    pf[me] = p->flags;
    if (p->any_direct) {
        cudaIpcMemHandle_t h;
        CK_CUDA(cudaIpcGetMemHandle(&h, p->flags));
        std::vector<char> all;
        int rc = nccl_allgather_bytes(p, &h, sizeof(h), all);
        if (rc) return rc;
        for (int r = 0; r < P; ++r) {
            if (r == me) continue;
            void* mapped = nullptr;
            cudaError_t e = cudaIpcOpenMemHandle(&mapped, reinterpret_cast<const cudaIpcMemHandle_t*>(all.data())[r], cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                cudaGetLastError();
                return fail(DFFT_ERR_PEER, std::string("cudaIpcOpenMemHandle(flags) failed: ") + cudaGetErrorString(e));
            }
            p->opened_flags.push_back(mapped);
            pf[r] = (unsigned long long*)mapped;
        }
    }
    CK_CUDA(cudaMalloc(&p->peer_flags_d, sizeof(void*) * P));
    CK_CUDA(cudaMemcpy(p->peer_flags_d, pf.data(), sizeof(void*) * P, cudaMemcpyHostToDevice));
    std::vector<int> gl(3 * P, 0);
    for (int k = 0; k < 3; ++k)
        for (size_t q = 0; q < p->grp[k].size(); ++q) gl[k * P + q] = p->grp[k][q];
    CK_CUDA(cudaMalloc(&p->groups_d, sizeof(int) * 3 * P));
    CK_CUDA(cudaMemcpy(p->groups_d, gl.data(), sizeof(int) * 3 * P, cudaMemcpyHostToDevice));
    return DFFT_SUCCESS;
}

// =====================================================================================================
// execution
// =====================================================================================================
// Views on the caller's buffers store a byte offset in seg[0].base; field f of a batched plan starts f field sizes further.
// which: the step's in_user / out_user (1: `in`, 2: `out` — in_user 2 is a view that reads `out`, in-place plans).
static void user_view(View& v, int which, const Schedule& sc, size_t f, void* out, const void* in) {
    if (which == 1) v.seg[0].base = (char*)const_cast<void*>(in) + f * sc.field_in + (size_t)v.seg[0].base;
    if (which == 2) v.seg[0].base = (char*)out + f * sc.field_out + (size_t)v.seg[0].base;
}

// 16-bit plans: the factor f_a the FFT pass step s multiplies its stores by, float(|s|^(log2 n_a / L)) of the direction's
// scale s, negative on the passes of the exec's last FFT axis when s is; 1 for copy passes and for s = 1
static double step_factor(const dfft_plan_s* p, const Schedule& sc, const Step& s) {
    const double sc_ = p->scale[sc.inverse];
    if (s.share_den == 0 || sc_ == 1.0) return 1.0;
    // exact for powers of two: log2 |s| * num / den of s = 1/N is -log2 n_a
    const double m = sc_ == 0.0 ? 0.0 : std::exp2(std::log2(std::fabs(sc_)) * s.share_num / s.share_den);
    return double(float(s.sign && sc_ < 0 ? -m : m));
}

// 16-bit plans: the output scale split over the exec's FFT passes (step_factor), so that an FP16 intermediate grows no more
// than the scaled result does.  L sums log2 n_a over the axes the schedule transforms (log2 Nz for the R2C z axis); the
// steps of its last FFT axis carry the sign.
static void split_scale(const dfft_plan_s* p, Schedule& sc) {
    const size_t n[3] = {p->g.nx, p->g.ny, p->g.nz};
    bool on[3] = {false, false, false};
    int last = -1, L = 0;
    for (const Step& s : sc.steps)
        if (s.type == STEP_PASS && !is_copy(s.kind)) { on[s.axis] = true; last = s.axis; }
    for (int a = 0; a < 3; ++a) L += on[a] ? ilog2_exact(n[a]) : 0;
    for (Step& s : sc.steps) {
        if (s.type != STEP_PASS || is_copy(s.kind)) continue;
        s.share_num = ilog2_exact(n[s.axis]);
        s.share_den = L;
        s.sign = s.axis == last;
    }
}

// Enqueues PASS step s of sc for field f on ss: the copy, FFT, fused or batched kernel over its views, its stores scaled by
// the direction's output scale when they are final values.  An in-place copy onto itself with nothing to scale is not
// launched (*launched = false).
static cudaError_t run_pass_step(const dfft_plan_s* p, const Schedule& sc, const Step& s, size_t f, void* out, const void* in, cudaStream_t ss,
                                 bool* launched) {
    *launched = false;
    const bool half = is_half(p->prec);
    if (s.identity && (half || p->scale[sc.inverse] == 1.0)) return cudaSuccess;  // 16-bit plans never scale a copy
    const double scale = half ? step_factor(p, sc, s) : s.final_store ? p->scale[sc.inverse] : 1.0;
    FftParams prm = s.prm, prm_y = s.prm_y;
    user_view(prm.in, s.in_user, sc, f, out, in);
    user_view(prm.out, s.out_user, sc, f, out, in);
    user_view(prm_y.in, s.y_in_user, sc, f, out, in);
    user_view(prm_y.out, s.y_out_user, sc, f, out, in);
    cudaError_t e = cudaErrorInvalidValue;
    switch (s.kernel) {
        case KERNEL_PASS:
            if (is_copy(s.kind)) {
                e = launch_copy_pass(p->prec, is_r2r(p->g.transform), s.kind, s.n, prm, scale, ss);
            } else {
                const size_t n = s.n ? s.n : size_t(1) << s.log2n;
                int hole[4];
                pass_hole(s.kind, n, s.keep, s.data, hole);
                const void* w = s.weighted ? p->weights[s.axis] : nullptr;  // null: the unweighted kernel
                e = launch_fft_pass(p->prec, s.kind, n, prm, s.blu, scale, ss, s.r2r, s.keep || s.data || w || s.twiddle ? hole : nullptr, w,
                                    s.twiddle ? &s.tw : nullptr);
            }
            break;
        case KERNEL_ZY_FUSED: e = launch_zy_fused(p->prec, s.log2n, prm, prm_y, s.zyf, scale, ss); break;
        case KERNEL_BATCH_SMALL:
            e = launch_batch_small(p->prec, s.log2n, prm.in.seg[0].base, prm.out.seg[0].base, (long long)p->batch, s.prm.inverse, s.bsf, scale, ss);
            break;
    }
    *launched = e == cudaSuccess;
    return e;
}

// capture: `st` is capturing into a CUDA graph (one-rank plans only, see exec_common).  Then only the kernels are
// enqueued: no timer or timeline events, and the plan's record of its last exec (launch count, stream, timer) stays
// what the last eager exec left.
// nfields: fields of a batched plan to transform (0 = all of them; dfft_plan_tune measures field 0 only).
static int run_schedule(dfft_plan_s* p, Schedule& sc, void* out, const void* in, cudaStream_t st, bool capture = false, size_t nfields = 0) {
    const int P = p->P, me = p->rank;
    const size_t es = p->esize;
    if (!capture) {
        p->epoch++;
        p->last_stream = st;
    }
    int launches = 0;
    int ev = 0;
    const bool timing = p->timing && !capture;
    cudaStream_t const ax0 = p->aux[0], ax1 = p->aux[1];
    cudaStream_t streams[3] = {st, ax0, ax1};
    auto mark = [&](const char* name, int is_fft, const char* label = "") -> cudaError_t {
        if (!timing || (sc.overlapped && is_fft != -1)) return cudaSuccess;  // overlapped: only start / end are meaningful
        if (ev >= int(p->events.size())) {
            cudaEvent_t e;
            cudaError_t r = cudaEventCreate(&e);
            if (r != cudaSuccess) return r;
            p->events.push_back(e);
            p->ev_names.push_back(name);
            p->ev_is_fft.push_back(is_fft);
            p->ev_labels.push_back(label);
        }
        p->ev_names[ev] = name;
        p->ev_is_fft[ev] = is_fft;
        p->ev_labels[ev] = label;
        return cudaEventRecord(p->events[ev++], st);
    };
    // overlapped schedules: the auxiliary streams fork from the caller's stream before a field and join it after
    auto fork = [&]() -> cudaError_t {
        cudaError_t e = cudaEventRecord(p->fork_ev, st);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ax0, p->fork_ev, 0);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ax1, p->fork_ev, 0);
        return e;
    };
    auto join = [&]() -> cudaError_t {
        cudaError_t e = cudaSuccess;
        for (int a = 0; a < 2 && e == cudaSuccess; ++a) {
            e = cudaEventRecord(p->join_ev[a], a == 0 ? ax0 : ax1);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(st, p->join_ev[a], 0);
        }
        return e;
    };
    if (sc.overlapped) {
        while (int(p->sync_events.size()) < sc.nevents) {
            cudaEvent_t e;
            CK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            p->sync_events.push_back(e);
        }
        CK_CUDA(fork());
    }
    CK_CUDA(mark("start", -1));
    int tl = 0;
    auto tl_mark = [&](cudaStream_t ss_, const char* label, int stream_id) -> cudaError_t {
        if (!timing) return cudaSuccess;
        if (tl >= int(p->tl_events.size())) {
            cudaEvent_t e;
            cudaError_t r = cudaEventCreate(&e);
            if (r != cudaSuccess) return r;
            p->tl_events.push_back(e);
            p->tl_labels.push_back(label);
            p->tl_streams.push_back(stream_id);
        }
        p->tl_labels[tl] = label;
        p->tl_streams[tl] = stream_id;
        return cudaEventRecord(p->tl_events[tl++], ss_);
    };
    const size_t fields = sc.whole_batch ? 1 : (nfields ? nfields : p->batch);
    for (size_t f = 0; f < fields; ++f) {
        // batched plans: the phase times mark the section ends of the last field; the step list covers every field
        const bool last = f + 1 == fields;
        if (f > 0 && sc.overlapped) {
            CK_CUDA(join());
            CK_CUDA(fork());
        }
        for (Step& s : sc.steps) {
            cudaStream_t ss = streams[s.stream];
            for (int w : s.waits) CK_CUDA(cudaStreamWaitEvent(ss, p->sync_events[w], 0));
            CK_CUDA(tl_mark(ss, s.label, s.stream));
            const char* phase = last ? s.phase : nullptr;
            if (s.type == STEP_PASS) {
                bool launched = false;
                const cudaError_t e = run_pass_step(p, sc, s, f, out, in, ss, &launched);
                if (e != cudaSuccess) return fail(DFFT_ERR_CUDA, std::string("FFT pass launch failed: ") + cudaGetErrorString(e));
                if (launched) ++launches;
                CK_CUDA(mark(phase, 1, s.label));
            } else if (s.type == STEP_RENDEZVOUS) {
                const std::vector<int>& G = p->grp[s.group];
                if (G.size() > 1) {
                    const unsigned long long ticket = ++p->ticket[s.phase_id];
                    rendezvous_kernel<<<1, 32 * int((G.size() + 31) / 32), 0, ss>>>(p->peer_flags_d, p->flags, p->groups_d + s.group * P, int(G.size()), me, P,
                                                                                  s.phase_id, ticket, p->err_d, p->rendezvous_timeout_cycles);
                    CK_CUDA(cudaGetLastError());
                    ++launches;
                }
                CK_CUDA(mark(phase, 0, s.label));
            } else {
                const std::vector<int>& G = p->grp[s.group];
                char* sb = (char*)p->slot(s.send_slot, me);
                char* rb = (char*)p->slot(s.recv_slot, me);
                CK_NCCL(ncclGroupStart());
                for (size_t q = 0; q < G.size(); ++q) {
                    if (G[q] == me) continue;
                    if (s.scount[q]) CK_NCCL(ncclSend(sb + s.soff[q] * es, s.scount[q] * es, ncclChar, G[q], p->comm->nccl, ss));
                    if (s.rcount[q]) CK_NCCL(ncclRecv(rb + s.roff[q] * es, s.rcount[q] * es, ncclChar, G[q], p->comm->nccl, ss));
                }
                CK_NCCL(ncclGroupEnd());
                for (size_t q = 0; q < G.size(); ++q)
                    if (G[q] == me && s.scount[q])
                        CK_CUDA(cudaMemcpyAsync(rb + s.roff[q] * es, sb + s.soff[q] * es, s.scount[q] * es, cudaMemcpyDeviceToDevice, ss));
                CK_CUDA(mark(phase, 0, s.label));
            }
            CK_CUDA(tl_mark(ss, s.label, s.stream));
            if (s.record >= 0) CK_CUDA(cudaEventRecord(p->sync_events[s.record], ss));
        }
    }
    if (timing) p->tl_used = tl;
    if (sc.overlapped) CK_CUDA(join());
    CK_CUDA(mark("Run complete", -1));
    if (capture) return DFFT_SUCCESS;
    if (timing) p->n_events_used = ev;
    p->last_launches = launches;
    p->execs++;
    sc.executed = true;
    return DFFT_SUCCESS;
}

// Bytes of one field in the caller's `in` and `out` of an exec (direction, d): the product of that buffer's layout, in
// reals for the real side of R2C / C2R and for DCT / DST plans (whose elements are reals).  No schedule touches a caller buffer beyond it (tests/test_batch.py checks every
// step's accesses), so fields sit back to back at this distance.
// In-place plans: one buffer, so one distance, dfft_get_domain_size(), which covers every layout (Geometry::domain_elems).
static void field_bytes(const dfft_plan_s* p, int inverse, int d, size_t* in_b, size_t* out_b) {
    if (p->inplace) {
        *in_b = *out_b = p->domain_bytes;
        return;
    }
    size_t s0[3], sd[3], o[3];
    p->g.layout(p->rank, 0, s0, o);
    p->g.layout(p->rank, d, sd, o);
    const size_t es = p->esize * p->comps;  // bytes per point
    const size_t real_es = p->g.transform == DFFT_R2C ? es / 2 : es;
    size_t b0 = s0[0] * s0[1] * s0[2] * real_es, bd = sd[0] * sd[1] * sd[2] * es;
    // box plans: the caller's array on a boxed side is its box (out_boxes: the output of d = 3 only)
    if (!p->in_boxes.empty()) b0 = p->in_boxes[p->rank].volume() * real_es;
    if (d == 3 && !p->out_boxes.empty()) bd = p->out_boxes[p->rank].volume() * es;
    // embedded sides: the caller's field stride
    if (p->in_embedded) b0 = size_t(p->in_strides[0]) * real_es;
    if (d == 3 && p->out_embedded) bd = size_t(p->out_strides[0]) * es;
    *in_b = inverse ? bd : b0;
    *out_b = inverse ? b0 : bd;
}

// In-place plans of one rank: build_schedule gave the views on slot D1 byte offsets from a null base; they address the
// caller's buffer, like the views on `out` (in_user / out_user 2, the same pointer as `in`).  Every other view without
// a user flag lies in the plan's one allocated slot.
static void relocate_buffer_views(const dfft_plan_s* p, Schedule& sc) {
    const char* slot = static_cast<const char*>(p->slot_ptr[0][p->rank]);
    auto relocate = [&](const View& v, int& user) {
        const char* b = static_cast<const char*>(v.seg[0].base);
        if (user == 0 && !(b >= slot && b < slot + p->slot_bytes)) user = 2;
    };
    for (Step& s : sc.steps) {
        if (s.type != STEP_PASS) continue;
        relocate(s.prm.in, s.in_user);
        relocate(s.prm.out, s.out_user);
        if (s.kernel == KERNEL_ZY_FUSED) {
            relocate(s.prm_y.in, s.y_in_user);
            relocate(s.prm_y.out, s.y_out_user);
        }
    }
}

// ---- kept axes (DESIGN.md section 3.12) ------------------------------------------------------------------------------
// The builders label passes by their role ("y pass", "x pass (tail)"); copy passes are named after their axis instead.
static void name_copies(Schedule& sc) {
    static const char* const names[3][2] = {{"x copy", "x copy (tail)"}, {"y copy", "y copy (tail)"}, {"z copy", "z copy (tail)"}};
    for (Step& s : sc.steps)
        if (s.type == STEP_PASS && is_copy(s.kind)) s.label = names[s.axis][std::strstr(s.label, "(tail)") ? 1 : 0];
}

// A kept z whose copy is local and keeps element order — both views one segment with the same strides, the input the
// caller's `in` (forward) or the output the caller's `out` (inverse), the other side a slot of this rank — is dropped
// whenever another pass follows it (forward) or precedes it (inverse).  Forward: the passes that read the slot region it
// fills read the caller's `in` at the same offsets instead, up to the first pass that writes into that region.  Inverse:
// the passes that fill the region it reads write the caller's `out` instead (out_user 2, so the output scale lands on
// them).  This holds for slab ZY_Then_X on any rank count and for every decomposition on one rank; elsewhere the z pass
// scatters across ranks.  A single z copy (d = 1) stays: it is the exec.
static void drop_z_copy(const dfft_plan_s* p, Schedule& sc, int inverse) {
    if (p->taxes[2]) return;
    std::vector<size_t> passes;
    for (size_t k = 0; k < sc.steps.size(); ++k)
        if (sc.steps[k].type == STEP_PASS) passes.push_back(k);
    if (passes.size() < 2) return;
    const size_t iz = inverse ? passes.back() : passes.front();
    const Step z = sc.steps[iz];
    if (!is_copy(z.kind) || z.axis != 2 || z.prm.in.nseg != 1 || z.prm.out.nseg != 1) return;
    const Seg &a = z.prm.in.seg[0], &b = z.prm.out.seg[0];
    if (a.sA0 != b.sA0 || a.sA1 != b.sA1 || z.prm.in.sN != z.prm.out.sN) return;
    if (inverse ? (z.in_user != 0 || z.out_user != 2) : (z.in_user != 1 || z.out_user != 0)) return;
    // the slot region the copy fills (forward) or drains (inverse), and the shift that takes it to the caller's buffer
    const View& sv = inverse ? z.prm.in : z.prm.out;
    const long long A0 = std::max(z.prm.A0, 1), A1 = std::max(z.prm.A1, 1);
    const long long last = (A0 - 1) * sv.seg[0].sA0 + (A1 - 1) * sv.seg[0].sA1 + (long long)(z.n - 1) * sv.sN;
    const char* lo = static_cast<const char*>(sv.seg[0].base);
    const char* hi = lo + size_t(last + 1) * p->esize;
    const long long shift = static_cast<const char*>(inverse ? b.base : a.base) - lo;
    auto inside = [&](const View& v, int user) {
        const char* base = static_cast<const char*>(v.seg[0].base);
        return user == 0 && v.nseg == 1 && base >= lo && base < hi;
    };
    auto move = [&](View& v) { v.seg[0].base = const_cast<char*>(static_cast<const char*>(v.seg[0].base)) + shift; };
    // local: the pass next to it (no rendezvous or all-to-all between them) reads (forward) or fills (inverse) the region —
    // with a rendezvous between them, peers deliver into the region (the Z_Then_YX inverse) and it must stay
    const Step& nb = sc.steps[inverse ? iz - 1 : iz + 1];
    if (nb.type != STEP_PASS || !(inverse ? inside(nb.prm.out, nb.out_user) : inside(nb.prm.in, nb.in_user))) return;
    if (!inverse) {
        for (size_t k = iz + 1; k < sc.steps.size(); ++k) {
            Step& s = sc.steps[k];
            if (s.type != STEP_PASS) continue;
            const bool overwrites = inside(s.prm.out, s.out_user);
            if (inside(s.prm.in, s.in_user)) { move(s.prm.in); s.in_user = 1; }
            if (overwrites) break;
        }
    } else {
        for (size_t k = iz; k-- > 0;) {
            Step& s = sc.steps[k];
            if (s.type != STEP_PASS) continue;
            if (inside(s.prm.in, s.in_user)) break;
            if (inside(s.prm.out, s.out_user)) { move(s.prm.out); s.out_user = 2; }
        }
    }
    sc.steps.erase(sc.steps.begin() + long(iz));
    // the inverse's last timer section moves to the pass that now ends the exec
    if (inverse && z.phase && !sc.steps[iz - 1].phase) sc.steps[iz - 1].phase = z.phase;
}

// the same elements of the same buffer (in place, the caller's `in` and `out` are one buffer)
static bool same_view(const View& a, int ua, const View& b, int ub, bool inplace) {
    auto buf = [&](int u) { return u == 0 ? 0 : inplace ? 1 : u; };
    if (buf(ua) != buf(ub) || a.nseg != b.nseg || a.sN != b.sN || (a.nseg > 1 && a.seg_of_n != b.seg_of_n)) return false;
    for (int i = 0; i < a.nseg; ++i)
        if (a.seg[i].base != b.seg[i].base || a.seg[i].sA0 != b.seg[i].sA0 || a.seg[i].sA1 != b.seg[i].sA1 || a.seg[i].n0 != b.seg[i].n0)
            return false;
    return true;
}

// A copy whose input and output views are identical moves nothing (the in-place y pass of Z_Then_YX, the in-place z
// pass of one rank) and is not emitted — unless it stores final values, where the output scale still has to be applied
// (in-place execs that end in a kept axis on the caller's buffer, e.g. d = 1 with z kept).
static void drop_identity_copies(const dfft_plan_s* p, Schedule& sc) {
    for (size_t k = 0; k < sc.steps.size();) {
        Step& s = sc.steps[k];
        if (s.type == STEP_PASS && is_copy(s.kind) && same_view(s.prm.in, s.in_user, s.prm.out, s.out_user, p->inplace)) {
            // the scale may change after the schedule is built: a final store stays in the list and run_schedule skips it
            // while the scale is 1
            if (s.final_store) {
                s.identity = true;
            } else {
                if (s.phase && k > 0 && !sc.steps[k - 1].phase) sc.steps[k - 1].phase = s.phase;
                sc.steps.erase(sc.steps.begin() + long(k));
                continue;
            }
        }
        ++k;
    }
}

// Interleaved plans: build_schedule lays out points of C values (its byte offsets count C * esize); the kernels address
// single values.  So every stride scales by C, a pass whose contiguous dimension is z sees C columns per z point, the z
// pass runs lines C apart with b the component (PASS_C2C_ILV: B = C, sN = C), and all-to-all counts are in values.  The
// R2C / C2R z pass becomes the pass of Nz-point lines, one per component (PASS_R2C_ILV / PASS_C2R_ILV), with the Nz-point
// twiddle table;
// its real side, built in complex units of Nz / 2 per row, is counted in reals (element (a0, a1, n, c) at
// base + a0 sA0 + a1 sA1 + n C + c).
static int widen_views(dfft_plan_s* p, Schedule& sc) {
    const long long C = (long long)p->comps;
    if (C == 1) return DFFT_SUCCESS;
    auto widen = [&](View& v, long long f) {
        v.sN *= C;
        for (int i = 0; i < v.nseg; ++i) { v.seg[i].sA0 *= C * f; v.seg[i].sA1 *= C * f; }
    };
    for (Step& s : sc.steps) {
        if (s.type == STEP_A2A)
            for (std::vector<size_t>* v : {&s.scount, &s.soff, &s.rcount, &s.roff})
                for (size_t& x : *v) x *= size_t(C);
        if (s.type != STEP_PASS) continue;
        const bool r2c = s.kind == PASS_R2C, c2r = s.kind == PASS_C2R;
        widen(s.prm.in, r2c ? 2 : 1);
        widen(s.prm.out, c2r ? 2 : 1);
        s.prm.B = s.kind == PASS_C2C_TILED ? s.prm.B * int(C) : int(C);
        if (s.kind == PASS_C2C_CONTIG) s.kind = PASS_C2C_ILV;
        if (r2c || c2r) {
            s.kind = r2c ? PASS_R2C_ILV : PASS_C2R_ILV;
            s.n = 2 * (s.n ? s.n : size_t(1) << s.log2n);
            s.log2n = ilog2_exact(s.n);
            void *tw = nullptr, *tw2 = nullptr, *blu = nullptr;
            const int rc = pass_tables(p->tabs, s.kind, s.n, 0, &tw, &tw2, &blu);
            if (rc) return rc;
            s.prm.tw = tw;
            s.prm.tw2 = nullptr;
        }
    }
    return DFFT_SUCCESS;
}

// This rank's block of layout `which` (0 input, 1 and 2 after z and y, 3 output) as the caller holds it: its box on a boxed
// side of a box plan (the physical side of every d, the output of d = 3), the plan's own layout otherwise.  1D plans hold
// the x-slab of the input layout on both sides, natural-order ones their chunk [oz_r][N2][N1] of the output grid
// [N3][N2][N1] on the output side.
static void caller_block(const dfft_plan_s* p, int which, size_t s[3], size_t o[3]) {
    p->g.layout(p->rank, p->n1d ? 0 : which, s, o);
    if (which == 3 && !p->oz.size.empty()) {
        s[0] = p->oz.size[size_t(p->rank)]; s[1] = p->g.ny; s[2] = p->g.nx;
        o[0] = p->oz.start[size_t(p->rank)]; o[1] = o[2] = 0;
    }
    const std::vector<Box>& boxes = which == 0 ? p->in_boxes : p->out_boxes;
    if ((which == 0 || which == 3) && !boxes.empty())
        for (int k = 0; k < 3; ++k) { s[k] = boxes[size_t(p->rank)].extent(k); o[k] = boxes[size_t(p->rank)].lo[k]; }
}

// ---- box-distributed plans (DESIGN.md section 3.17) ------------------------------------------------------------------
// One side of an exec whose caller arrays are boxes: per rank the caller's box and the natural block of layout `which` (0
// the physical side, 3 the output) that the wrapped schedule reads or writes, in the elements of the schedule's views.  The
// real side of R2C / C2R plans is counted in complex pairs there, so its z bounds are halved (dfft_plan_create_boxes keeps
// them even).
struct BoxSide {
    std::vector<Box> box, nat;
};
static BoxSide box_side(const dfft_plan_s* p, const std::vector<Box>& boxes, int which) {
    BoxSide b;
    const bool pairs = which == 0 && p->g.transform == DFFT_R2C;
    for (int r = 0; r < p->P; ++r) {
        size_t s[3], o[3];
        p->g.layout(r, which, s, o);
        Box n = Box::of(s, o), c = boxes[size_t(r)];
        if (pairs) { n.lo[2] /= 2; n.hi[2] /= 2; c.lo[2] /= 2; c.hi[2] /= 2; }
        b.nat.push_back(n);
        b.box.push_back(c);
    }
    return b;
}

// One reshape copy: the grid points of `pc` from the dense array of box `src` at `sb` to the dense array of box `dst` at
// `db` (both contain pc), lines along z.  An empty piece is a copy of no lines, so that every rank lists the same steps.
static Step piece_copy(const dfft_plan_s* p, int inverse, const char* label, const Box& pc, void* sb, const Box& src, void* db, const Box& dst) {
    Step s;
    s.type = STEP_PASS;
    s.kind = PASS_COPY_CONTIG;
    s.label = label;
    s.axis = 2;
    const bool empty = pc.volume() == 0;
    s.n = empty ? 0 : pc.extent(2);
    s.prm.A0 = empty ? 0 : int(pc.extent(0));
    s.prm.A1 = empty ? 0 : int(pc.extent(1));
    s.prm.B = 1;
    s.prm.inverse = inverse;
    auto view = [&](void* base, const Box& b) {
        return single_view(eptr(base, empty ? 0 : b.offset(pc.lo), p->esize), (long long)(b.extent(1) * b.extent(2)), (long long)b.extent(2), 1);
    };
    s.prm.in = view(sb, src);
    s.prm.out = view(db, dst);
    return s;
}

// The reshape of one boxed side: `pre` — before the first pass, from the caller's boxes (in_user 1) into the natural block
// in slot BX; otherwise after the last pass, from the natural blocks in BX into the caller's boxes (out_user 2).
//   Peer2Peer, pre: each rank pushes the piece of its box that every rank q owns into q's BX, then a rendezvous of all ranks.
//     The caller's buffers are not mapped on the peers, so the owner of the data has to store it.
//   Peer2Peer, post: a rendezvous, then each rank gathers the pieces of its box from every rank's BX (remote reads).
//   All2All: the pieces are packed into SS at the all-to-all's send offsets, exchanged, and unpacked from SR.
static void reshape_steps(const dfft_plan_s* p, int inverse, const BoxSide& S, bool pre, std::vector<Step>& out) {
    const int me = p->rank, P = p->P;
    const char* label = pre ? "reshape in" : "reshape out";
    void* const user = nullptr;  // views on the caller's buffers hold byte offsets (user_view)
    void* const bx = p->slot(p->slots.BX, me);
    auto rendezvous = [&]() {
        Step r = new_rendezvous(0, 0, nullptr, 0);
        r.label = "reshape rendezvous";
        out.push_back(r);
    };
    if (p->box_direct) {
        if (!pre) rendezvous();
        for (int q = 0; q < P; ++q) {
            Step s = pre ? piece_copy(p, inverse, label, S.box[me] & S.nat[q], user, S.box[me], p->slot(p->slots.BX, q), S.nat[q])
                         : piece_copy(p, inverse, label, S.nat[q] & S.box[me], p->slot(p->slots.BX, q), S.nat[q], user, S.box[me]);
            (pre ? s.in_user : s.out_user) = pre ? 1 : 2;
            out.push_back(s);
        }
        if (pre) rendezvous();
        return;
    }
    // all-to-all: what I send to q is my part of q's box (pre: my box's part of q's natural block), what I receive q's
    Step a;
    a.type = STEP_A2A;
    a.label = "nccl all-to-all";
    a.group = 0;
    a.send_slot = p->slots.SS;
    a.recv_slot = p->slots.SR;
    std::vector<Box> send(static_cast<size_t>(P)), recv(static_cast<size_t>(P));
    size_t so = 0, ro = 0;
    for (int q = 0; q < P; ++q) {
        send[q] = pre ? S.box[me] & S.nat[q] : S.nat[me] & S.box[q];
        recv[q] = pre ? S.box[q] & S.nat[me] : S.nat[q] & S.box[me];
        a.scount.push_back(send[q].volume());
        a.rcount.push_back(recv[q].volume());
        a.soff.push_back(so);
        a.roff.push_back(ro);
        so += send[q].volume();
        ro += recv[q].volume();
    }
    void* const ss = p->slot(p->slots.SS, me);
    void* const sr = p->slot(p->slots.SR, me);
    for (int q = 0; q < P; ++q) {
        Step s = pre ? piece_copy(p, inverse, label, send[q], user, S.box[me], eptr(ss, a.soff[q], p->esize), send[q])
                     : piece_copy(p, inverse, label, send[q], bx, S.nat[me], eptr(ss, a.soff[q], p->esize), send[q]);
        if (pre) s.in_user = 1;
        out.push_back(s);
    }
    out.push_back(a);
    for (int q = 0; q < P; ++q) {
        Step s = pre ? piece_copy(p, inverse, label, recv[q], eptr(sr, a.roff[q], p->esize), recv[q], bx, S.nat[me])
                     : piece_copy(p, inverse, label, recv[q], eptr(sr, a.roff[q], p->esize), recv[q], user, S.box[me]);
        if (!pre) s.out_user = 2;
        out.push_back(s);
    }
}

// Box plans: the schedule of the natural layouts, its views on a boxed side's caller buffer moved to the same offsets in
// slot BX, with the reshape of that side before it (after its entry rendezvous: the peers have left the previous exec) or
// after it.  Forward: the physical side is `in`, the output `out`; inverse the other way round.  out_boxes apply to d = 3
// only: the spectral side of a partial exec keeps its natural layout.  BX holds the natural array of a side only between
// its reshape and the pass that reads it (pre), or the pass that writes it and its reshape (post); the wrapped schedule
// reads the pre side's data before it writes the post side's (one slot serves both).
static int wrap_boxes(dfft_plan_s* p, int inverse, int d, Schedule& sc) {
    const bool phys = !p->in_boxes.empty(), spec = d == 3 && !p->out_boxes.empty();
    const bool pre = inverse ? spec : phys, post = inverse ? phys : spec;
    if (!pre && !post) return DFFT_SUCCESS;
    if (p->slots.BX < 0) return fail(DFFT_ERR_STATE, "internal: box plan without a staging slot");
    char* const bx = static_cast<char*>(p->slot(p->slots.BX, p->rank));
    for (Step& s : sc.steps) {
        if (s.type != STEP_PASS) continue;
        if (s.kernel != KERNEL_PASS) return fail(DFFT_ERR_STATE, "internal: box plans run single passes");
        if (pre && s.in_user == 1) { s.prm.in.seg[0].base = bx + (size_t)s.prm.in.seg[0].base; s.in_user = 0; }
        if (post && s.out_user == 2) { s.prm.out.seg[0].base = bx + (size_t)s.prm.out.seg[0].base; s.out_user = 0; }
    }
    std::vector<Step> head, tail;
    if (pre) reshape_steps(p, inverse, box_side(p, inverse ? p->out_boxes : p->in_boxes, inverse ? 3 : 0), true, head);
    if (post) reshape_steps(p, inverse, box_side(p, inverse ? p->in_boxes : p->out_boxes, inverse ? 0 : 3), false, tail);
    const bool entry = !sc.steps.empty() && sc.steps[0].type == STEP_RENDEZVOUS && sc.steps[0].group == 0;
    sc.steps.insert(sc.steps.begin() + (entry ? 1 : 0), head.begin(), head.end());
    sc.steps.insert(sc.steps.end(), tail.begin(), tail.end());
    return DFFT_SUCCESS;
}

// ---- embedded layouts (DESIGN.md section 3.18) -----------------------------------------------------------------------
// One side of an exec on caller arrays with their own strides (dfft_plan_set_strides): the dense block e[x][y][z] that the
// schedule's views on that buffer address, and the caller's x and y strides, both in the views' elements (complex pairs on
// the real side of R2C / C2R, whose strides are even).
struct EmbedSide {
    bool on = false;
    size_t e[3] = {0, 0, 0};
    long long sx = 0, sy = 0;
};
static EmbedSide embed_side(const dfft_plan_s* p, bool physical) {
    EmbedSide E;
    E.on = physical ? p->in_embedded : p->out_embedded;
    if (!E.on) return E;
    size_t o[3];
    caller_block(p, physical ? 0 : 3, E.e, o);
    const long long* s = physical ? p->in_strides : p->out_strides;
    const long long pairs = physical && p->g.transform == DFFT_R2C ? 2 : 1;
    E.e[2] /= size_t(pairs);
    E.sx = s[1] / pairs;
    E.sy = s[2] / pairs;
    return E;
}

// The views of one pass (or one phase of the fused stage) on embedded sides: a view on the dense block maps base offset
// i Ny Nz + j Nz + k to i X + j Y + k, and each of its dimensions (a0, a1, n and the contiguous b) to the caller's stride of
// the one axis it runs along.  That is exact when no dimension carries into the next axis: per axis, the base's index plus
// the reach of every dimension along it stays inside the block, which is checked.  The one dimension that may span two
// axes is b of a TILED pass whose rows are whole y-z planes (x passes without the blocked hand-over, B = y rows x z
// columns): it is split into a1 = the y rows and b = z first, for both views, which needs a1 unused.  es: bytes per element;
// in_len / out_len: points along n of each view.
static int embed_pass(FftParams& prm, int in_user, int out_user, const EmbedSide& Ein, const EmbedSide& Eout, size_t es, size_t in_len,
                      size_t out_len) {
    auto split_needed = [&](const View& v, const EmbedSide& E) {
        const long long off = (long long)(size_t)v.seg[0].base / (long long)es;
        return E.on && E.e[2] > 0 && prm.B > 0 && off % (long long)E.e[2] + prm.B > (long long)E.e[2];
    };
    for (int w = 0; w < 2; ++w) {
        const View& v = w ? prm.out : prm.in;
        const EmbedSide& E = w ? Eout : Ein;
        if (!(w ? out_user : in_user) || !split_needed(v, E)) continue;
        const long long nz = (long long)E.e[2], off = (long long)(size_t)v.seg[0].base / (long long)es;
        if (prm.A1 != 1 || off % nz != 0 || prm.B % nz != 0) return fail(DFFT_ERR_STATE, "internal: an embedded view's rows span more than y and z");
        prm.A1 = int(prm.B / nz);
        prm.B = int(nz);
        for (View* u : {&prm.in, &prm.out})
            for (int i = 0; i < u->nseg; ++i) u->seg[i].sA1 = nz;
    }
    auto map = [&](View& v, const EmbedSide& E, size_t len) -> int {
        if (v.nseg != 1) return fail(DFFT_ERR_STATE, "internal: an embedded view has segments");
        const size_t bytes = (size_t)v.seg[0].base;
        const long long ext[4] = {prm.A0, prm.A1, (long long)len, prm.B};
        long long* const stride[3] = {&v.seg[0].sA0, &v.seg[0].sA1, &v.sN};
        const long long plane = (long long)(E.e[1] * E.e[2]), row = (long long)E.e[2];
        if (ext[0] <= 0 || ext[1] <= 0 || ext[2] <= 0 || ext[3] <= 0) {  // no element: nothing to address
            v.seg[0].base = nullptr;
            return DFFT_SUCCESS;
        }
        if (plane == 0) return fail(DFFT_ERR_STATE, "internal: an embedded view on an empty block");
        if (bytes % es) return fail(DFFT_ERR_STATE, "internal: an embedded view's offset is not whole elements");
        // (x, y, z) of an offset in the dense block; S: the caller's stride of each axis
        auto split = [&](long long o, long long c[3]) { c[0] = o / plane; c[1] = o % plane / row; c[2] = o % row; };
        const long long S[3] = {E.sx, E.sy, 1};
        long long reach[3];
        split((long long)(bytes / es), reach);
        long long base = reach[0] * S[0] + reach[1] * S[1] + reach[2] * S[2];
        for (int k = 0; k < 4; ++k) {
            const long long s = k < 3 ? *stride[k] : 1;
            long long c[3];
            if (s < 0) return fail(DFFT_ERR_STATE, "internal: an embedded view runs backwards");
            split(s, c);
            const int axes = (c[0] != 0) + (c[1] != 0) + (c[2] != 0);
            if (ext[k] > 1 && axes > 1) return fail(DFFT_ERR_STATE, "internal: an embedded view's dimension spans two axes");
            for (int a = 0; a < 3; ++a) reach[a] += (ext[k] - 1) * c[a];
            if (k < 3) *stride[k] = ext[k] > 1 ? c[0] * S[0] + c[1] * S[1] + c[2] * S[2] : 0;
        }
        for (int a = 0; a < 3; ++a)
            if (reach[a] >= (long long)E.e[a]) return fail(DFFT_ERR_STATE, "internal: an embedded view leaves its block");
        v.seg[0].base = reinterpret_cast<void*>(size_t(base) * es);
        return DFFT_SUCCESS;
    };
    int rc = DFFT_SUCCESS;
    if (in_user && Ein.on) rc = map(prm.in, Ein, in_len);
    if (!rc && out_user && Eout.on) rc = map(prm.out, Eout, out_len);
    return rc;
}

// Embedded plans: every view on a caller buffer with its own strides, mapped by embed_pass.  Forward: `in` is the physical
// side, `out` the output; inverse the other way round.  out_strides apply to d = 3 only: the spectral side of a partial exec
// stays dense.  The builders, the box reshapes and the kept-axis copies have laid these views out on the dense blocks.
static int embed_views(dfft_plan_s* p, int inverse, int d, Schedule& sc) {
    if (!p->embedded()) return DFFT_SUCCESS;
    const EmbedSide phys = embed_side(p, true);
    const EmbedSide spec = d == 3 ? embed_side(p, false) : EmbedSide();
    const EmbedSide& Ein = inverse ? spec : phys;
    const EmbedSide& Eout = inverse ? phys : spec;
    for (Step& s : sc.steps) {
        if (s.type != STEP_PASS) continue;
        if (s.kernel != KERNEL_PASS) return fail(DFFT_ERR_STATE, "internal: embedded plans run single passes");
        // points along n of each view, as dfft_debug_run_step counts them
        size_t in_len = 0, out_len = 0;
        s.view_lens(&in_len, &out_len);
        const int rc = embed_pass(s.prm, s.in_user, s.out_user, Ein, Eout, p->esize, in_len, out_len);
        if (rc) return rc;
    }
    return DFFT_SUCCESS;
}

// The one place that decides which schedule a (direction, d) pair runs — used by exec and by dfft_plan_describe, so
// the CPU schedule emulation always validates exactly what executes.
static int get_schedule(dfft_plan_s* p, int inverse, int d, Schedule** out) {
    if (p->n1d && d != 3) return fail(DFFT_ERR_UNSUPPORTED, "1D plans run the whole transform (d = 3)");
    Schedule& sc = p->sched[inverse ? 1 : 0][d - 1];
    p->axes_fixed = true;
    if (!sc.built) {
        sc = Schedule();  // a build that failed may have left steps and flags
        g_view_error = false;
        const bool streams = p->cfg.send_method == DFFT_SEND_STREAMS || (p->g.decomp == DFFT_PENCIL && p->cfg.send_method2 == DFFT_SEND_STREAMS);
        const bool seq_won = p->tuned_seq[inverse ? 1 : 0] != 0;
        const bool want_overlap = streams && d == 3 && p->P > 1 && p->g.decomp == DFFT_SLAB_ZY_THEN_X && p->direct2 && p->xchg_ctas >= 0 && !seq_won &&
                                  alt_schedules(p);
        // pencil: forward on a grid with two real transpositions by default; every other
        // combination (inverse, p1 or p2 == 1) only once dfft_plan_tune has measured it faster than the sequential schedule
        const bool both_multi = p->grp[1].size() > 1 && p->grp[2].size() > 1;
        const bool tuned = p->tuned_ctas[inverse ? 1 : 0] != -2;
        const bool want_pencil_overlap = streams && d == 3 && p->g.decomp == DFFT_PENCIL && p->direct1 && p->direct2 && p->P > 1 && p->xchg_ctas >= 0 &&
                                         pencil_overlap_enabled() && !seq_won && ((both_multi && !inverse) || tuned || pencil_overlap_mode() == 2) &&
                                         alt_schedules(p);
        // one rank with x kept: the layout after d = 2 is the output layout, so d = 3 runs the d = 2 steps (no x copy)
        const int db = p->P == 1 && !p->taxes[0] && d == 3 ? 2 : d;
        int rc;
        if (p->n1d) rc = build_1d(p, inverse ? 1 : 0, sc);
        else if (batch_small(p, d)) rc = build_batch_small(p, inverse ? 1 : 0, sc);
        // the overlapped slab and pencil schedules share their forward builder; their inverses run different pipelines
        else if ((want_overlap || want_pencil_overlap) && !inverse) rc = build_overlapped_forward(p, sc);
        else if (want_overlap) rc = build_overlapped_slab_inverse(p, sc);
        else if (want_pencil_overlap) rc = build_overlapped_pencil_inverse(p, sc);
        else rc = build_schedule(p, inverse ? 1 : 0, db, sc);
        if (rc) return rc;
        rc = widen_views(p, sc);
        if (rc) return rc;
        if (!all_axes(p)) {
            name_copies(sc);
            drop_z_copy(p, sc, inverse ? 1 : 0);
        }
        rc = wrap_boxes(p, inverse ? 1 : 0, d, sc);
        if (rc) return rc;
        rc = embed_views(p, inverse ? 1 : 0, d, sc);
        if (rc) return rc;
        // No step reads the caller's `out` (views on it are only ever stored to), so every store into it is an output
        // value of the exec: the steps that write `out` are exactly the ones that store final values.  This covers the tail
        // launches of blocked hand-over layouts, every z chunk of overlapped x passes, the last pass of partial transforms
        // and the fused and batched stages (whose earlier phase writes only the work area, or `out` inside the same launch).
        // tests/test_scale.py replays every such schedule and checks that each output value is scaled exactly once.
        for (Step& s : sc.steps) s.final_store = s.type == STEP_PASS && s.out_user == 2;
        for (Step& s : sc.steps) s.weighted = p->weighted && s.type == STEP_PASS && s.kernel == KERNEL_PASS && !is_copy(s.kind);
        if (is_half(p->prec)) split_scale(p, sc);
        // In place the buffer also holds intermediates: its views from slot D1 are marked after the final stores.
        // tests/test_inplace.py replays these schedules on one address range.
        if (p->buf_slot) relocate_buffer_views(p, sc);
        if (!all_axes(p)) drop_identity_copies(p, sc);
        sc.inverse = inverse ? 1 : 0;
        field_bytes(p, inverse, d, &sc.field_in, &sc.field_out);
        if (g_view_error) return fail(DFFT_ERR_STATE, "internal: segments of one view disagree on the axis stride");
        sc.built = true;  // only a schedule that every step above accepted is reused
    }
    *out = &sc;
    return DFFT_SUCCESS;
}

static int timer_gather(dfft_plan_s* p);
static const char* transform_name(int t) {
    return t == DFFT_C2C ? "C2C" : t == DFFT_DCT ? "DCT" : t == DFFT_DST ? "DST" : t == DFFT_R2HC ? "per-axis R2R" : "R2C/C2R";
}
// need_transform: DFFT_R2C, DFFT_C2C, or EXEC_R2R for the execs of real-to-real plans
constexpr int EXEC_R2R = -1;
static int exec_common(dfft_plan_t p, void* out, const void* in, int inverse, int d, int need_transform, void* stream, bool sync) {
    // sync == true: the plain calls run on the plan's own stream; _async calls use exactly the stream given
    // (NULL = the CUDA default stream)
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (p->comm->dry) return fail(DFFT_ERR_STATE, "geometry-only plan (dfft_comm_create_dry) cannot execute");
    if (!p->work) return fail(DFFT_ERR_STATE, "plan has no work area (call dfft_set_work_area)");
    if (need_transform == EXEC_R2R ? !is_r2r(p->g.transform) : p->g.transform != need_transform)
        return fail(DFFT_ERR_INVALID, std::string("plan was created for ") + transform_name(p->g.transform));
    if (d < 1 || d > 3) return fail(DFFT_ERR_INVALID, "d must be 1, 2 or 3");
    if (!out || !in) return fail(DFFT_ERR_INVALID, "null buffer");
    if (p->inplace && out != in) return fail(DFFT_ERR_INVALID, "in-place plan: out must equal in");
    {   // embedded sides: the views address whole elements from the caller's pointer (a pair of reals on the real side of
        // R2C / C2R, which is esize bytes like a complex element)
        const bool phys = p->in_embedded, spec = d == 3 && p->out_embedded;
        const bool in_emb = inverse ? spec : phys, out_emb = inverse ? phys : spec;
        if ((in_emb && (uintptr_t)in % p->esize) || (out_emb && (uintptr_t)out % p->esize))
            return fail(DFFT_ERR_INVALID, "a buffer with strides (dfft_plan_set_strides) must be aligned to " + std::to_string(p->esize) + " bytes");
    }
    CK_CUDA(cudaSetDevice(p->comm->device));
    cudaStream_t st = sync ? p->own_stream : (cudaStream_t)stream;
    // A stream capture records the kernels into a graph without running them, so nothing may be set up on the way
    // (allocations, table uploads, kernel attributes): the schedule must have run eagerly before.  Multi-rank plans take
    // their rendezvous epochs from the host, which a replay would repeat.
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (!sync) CK_CUDA(cudaStreamIsCapturing(st, &cap));
    const bool capture = cap != cudaStreamCaptureStatusNone;
    if (capture && p->P > 1) return fail(DFFT_ERR_UNSUPPORTED, "capture of multi-rank plans is not supported yet");
    if (capture && !p->sched[inverse ? 1 : 0][d - 1].executed)
        return fail(DFFT_ERR_STATE, "run one exec of this direction before capturing it into a CUDA graph");
    Schedule* scp = nullptr;
    {
        int rc = get_schedule(p, inverse, d, &scp);
        if (rc) return rc;
    }
    Schedule& sc = *scp;
    if (sync) {
        // explicit edge from the legacy default stream (belt and braces on top of the blocking-stream semantics; it
        // also covers callers whose own streams are blocking streams, which the legacy stream itself waits for)
        CK_CUDA(cudaEventRecord(p->entry_ev, cudaStreamLegacy));
        CK_CUDA(cudaStreamWaitEvent(st, p->entry_ev, 0));
    }
    int rc = run_schedule(p, sc, out, in, st, capture);
    if (rc) return rc;
    if (!sync) return DFFT_SUCCESS;
    rc = dfft_plan_wait(p);
    if (rc) return rc;
    CK_CUDA(cudaDeviceSynchronize());  // the reference's execs end like this (mpicufft_slab.cpp:807, 870)
    // the reference gathers and appends the section times after every non-warm-up exec
    // (mpicufft_slab.cpp:817-821)
    if (!p->csv_path.empty() && p->timing && d == 3) {
        if (p->csv_warmup_left > 0) p->csv_warmup_left--;
        else return timer_gather(p);
    }
    return DFFT_SUCCESS;
}

// =====================================================================================================
// phase-timer CSV in the reference's on-disk schema (/root/reference/src/timer.cpp:58-101; file names
// mpicufft_slab.cpp:99-103, mpicufft_slab_z_then_yx.cpp:76-80, mpicufft_pencil.cpp:67-72)
// =====================================================================================================
static const char* const SECTIONS_SLAB[] = {"init", "2D FFT (Sync)", "2D FFT Y-Z-Direction", "Transpose (First Send)", "Transpose (Packing)",
    "Transpose (Start Local Transpose)", "Transpose (Start Receive)", "Transpose (First Receive)", "Transpose (Finished Receive)",
    "Transpose (Start All2All)", "Transpose (Finished All2All)", "Transpose (Unpacking)", "1D FFT X-Direction", "Run complete"};
static const char* const SECTIONS_ZYX[] = {"init", "1D FFT Z-Direction", "Transpose (First Send)", "Transpose (Packing)",
    "Transpose (Start Local Transpose)", "Transpose (Start Receive)", "Transpose (First Receive)", "Transpose (Finished Receive)",
    "Transpose (Start All2All)", "Transpose (Finished All2All)", "Transpose (Unpacking)", "2D FFT Y-X-Direction", "Run complete"};
static const char* const SECTIONS_PENCIL[] = {"init", "1D FFT Z-Direction", "First Transpose (First Send)", "First Transpose (Packing)",
    "First Transpose (Start Local Transpose)", "First Transpose (Start Receive)", "First Transpose (First Receive)",
    "First Transpose (Finished Receive)", "First Transpose (Start All2All)", "First Transpose (Finished All2All)",
    "First Transpose (Unpacking)", "First Transpose (Send Complete)", "1D FFT Y-Direction", "Second Transpose (First Send)",
    "Second Transpose (Packing)", "Second Transpose (Start Local Transpose)", "Second Transpose (Start Receive)",
    "Second Transpose (First Receive)", "Second Transpose (Finished Receive)", "Second Transpose (Start All2All)",
    "Second Transpose (Finished All2All)", "Second Transpose (Unpacking)", "1D FFT X-Direction", "Run complete"};

static void plan_sections(const dfft_plan_s* p, const char* const** list, int* n) {
    if (p->g.decomp == DFFT_PENCIL) { *list = SECTIONS_PENCIL; *n = int(sizeof(SECTIONS_PENCIL) / sizeof(char*)); }
    else if (p->g.decomp == DFFT_SLAB_Z_THEN_YX) { *list = SECTIONS_ZYX; *n = int(sizeof(SECTIONS_ZYX) / sizeof(char*)); }
    else { *list = SECTIONS_SLAB; *n = int(sizeof(SECTIONS_SLAB) / sizeof(char*)); }
}

static int timer_gather(dfft_plan_s* p) {
    if (p->n_events_used < 2) return fail(DFFT_ERR_STATE, "no timed exec to gather");
    const char* const* names = nullptr;
    int ns = 0;
    plan_sections(p, &names, &ns);
    std::vector<double> dur(ns, 0.0);
    dur[0] = p->init_ms;
    CK_CUDA(cudaEventSynchronize(p->events[p->n_events_used - 1]));
    double last = 0;
    for (int k = 1; k < p->n_events_used; ++k) {
        float f = 0;
        CK_CUDA(cudaEventElapsedTime(&f, p->events[0], p->events[k]));
        last = f;
        if (!p->ev_names[k]) continue;
        for (int i = 0; i < ns; ++i)
            if (!strcmp(names[i], p->ev_names[k])) dur[i] = f;
    }
    dur[ns - 1] = last;  // "Run complete"
    if (p->n_events_used == 2 && p->tl_used >= 2) {
        // overlapped schedule: the steps ran on several streams and only start / end were marked on the caller's.  The
        // reference's sections are cumulative times, so a section gets the time at which the LAST step of its kind ended
        // (step timeline, dfft_get_timeline).
        const bool pencil = p->g.decomp == DFFT_PENCIL;
        auto section_of = [&](const char* label) -> const char* {
            if (!strncmp(label, "z pass", 6)) return p->g.decomp == DFFT_SLAB_ZY_THEN_X ? nullptr : "1D FFT Z-Direction";
            if (!strncmp(label, "y pass", 6)) return pencil ? "1D FFT Y-Direction" : "2D FFT Y-Z-Direction";
            if (!strncmp(label, "x pass", 6)) return "1D FFT X-Direction";
            if (!strcmp(label, "rendezvous 1")) return "First Transpose (Finished Receive)";
            if (!strcmp(label, "rendezvous 2")) return pencil ? "Second Transpose (Finished Receive)" : "Transpose (Finished Receive)";
            return nullptr;
        };
        for (int i = 0; i + 1 < p->tl_used; i += 2) {
            const char* sec = section_of(p->tl_labels[i]);
            if (!sec) continue;
            float f = 0;
            CK_CUDA(cudaEventSynchronize(p->tl_events[i + 1]));
            CK_CUDA(cudaEventElapsedTime(&f, p->events[0], p->tl_events[i + 1]));
            for (int k = 0; k < ns; ++k)
                if (!strcmp(names[k], sec) && f > dur[k]) dur[k] = f;
        }
    }
    std::vector<char> all;
    int rc = nccl_allgather_bytes(p, dur.data(), sizeof(double) * ns, all);
    if (rc) return rc;
    if (p->rank != 0 || p->csv_path.empty()) return DFFT_SUCCESS;
    const double* o = reinterpret_cast<const double*>(all.data());
    struct stat sb;
    std::ofstream f;
    if (stat(p->csv_path.c_str(), &sb) != 0) {
        f.open(p->csv_path);
        f << ",";
        for (int i = 0; i < p->P; ++i) f << i << ",";
    } else {
        f.open(p->csv_path, std::ios_base::app);
    }
    if (!f) return fail(DFFT_ERR_INVALID, "cannot open " + p->csv_path);
    f << "\n";
    for (int i = 0; i < ns; ++i) {
        f << names[i] << ",";
        for (int r = 0; r < p->P; ++r) f << o[size_t(r) * ns + i] << ",";
        f << "\n";
    }
    return DFFT_SUCCESS;
}

// =====================================================================================================
// C ABI
// =====================================================================================================
extern "C" {

const char* dfft_last_error_string(void) { return g_err.c_str(); }
int dfft_version(void) { return DFFT_VERSION; }

int dfft_get_unique_id(void* id) {
    if (!id) return fail(DFFT_ERR_INVALID, "null id");
    static_assert(sizeof(ncclUniqueId) <= DFFT_UNIQUE_ID_BYTES, "unique id size");
    ncclUniqueId u;
    CK_NCCL(ncclGetUniqueId(&u));
    memset(id, 0, DFFT_UNIQUE_ID_BYTES);
    memcpy(id, &u, sizeof(u));
    return DFFT_SUCCESS;
}

int dfft_comm_create(int rank, int nranks, const void* id, int device, dfft_comm_t* comm) {
    if (!comm || nranks < 1 || rank < 0 || rank >= nranks) return fail(DFFT_ERR_INVALID, "bad rank / nranks");
    if (nranks > MAXSEG) return fail(DFFT_ERR_UNSUPPORTED, "at most " + std::to_string(MAXSEG) + " ranks");
    CK_CUDA(cudaSetDevice(device));
    dfft_comm_s* c = new dfft_comm_s();
    c->rank = rank; c->nranks = nranks; c->device = device;
    if (nranks > 1) {
        if (!id) { delete c; return fail(DFFT_ERR_INVALID, "unique id required for nranks > 1"); }
        ncclUniqueId u;
        memcpy(&u, id, sizeof(u));
        ncclResult_t r = ncclCommInitRank(&c->nccl, nranks, u, rank);
        if (r != ncclSuccess) { delete c; return fail(DFFT_ERR_NCCL, std::string("ncclCommInitRank: ") + ncclGetErrorString(r)); }
    }
    *comm = c;
    return DFFT_SUCCESS;
}
int dfft_comm_create_dry(int rank, int nranks, dfft_comm_t* comm) {
    if (!comm || nranks < 1 || rank < 0 || rank >= nranks) return fail(DFFT_ERR_INVALID, "bad rank / nranks");
    if (nranks > MAXSEG) return fail(DFFT_ERR_UNSUPPORTED, "at most " + std::to_string(MAXSEG) + " ranks");
    dfft_comm_s* c = new dfft_comm_s();
    c->rank = rank; c->nranks = nranks; c->device = -1; c->dry = true;
    *comm = c;
    return DFFT_SUCCESS;
}
int dfft_comm_destroy(dfft_comm_t c) {
    if (!c) return DFFT_SUCCESS;
    if (c->nccl) ncclCommDestroy(c->nccl);
    delete c;
    return DFFT_SUCCESS;
}
int dfft_comm_rank(dfft_comm_t c) { return c ? c->rank : -1; }
int dfft_comm_size(dfft_comm_t c) { return c ? c->nranks : -1; }

int dfft_partition(size_t n, size_t parts, size_t* sizes, size_t* starts) {
    if (!parts || !sizes || !starts) return fail(DFFT_ERR_INVALID, "bad partition request");
    Split s;
    s.make(n, parts);
    for (size_t p = 0; p < parts; ++p) { sizes[p] = s.size[p]; starts[p] = s.start[p]; }
    return DFFT_SUCCESS;
}

int dfft_layout(int decomp, int transform, size_t nx, size_t ny, size_t nz, size_t p1, size_t p2, int rank, int which,
                size_t size[3], size_t start[3]) {
    Geometry g;
    int nranks = decomp == DFFT_PENCIL ? int(p1 * p2) : int(p1);
    if (!g.init(decomp, transform, nx, ny, nz, p1, p2, nranks)) return fail(DFFT_ERR_INVALID, "invalid partition");
    if (rank < 0 || rank >= nranks || which < 0 || which > 3) return fail(DFFT_ERR_INVALID, "bad rank / which");
    g.layout(rank, which, size, start);
    return DFFT_SUCCESS;
}

int dfft_plan_create(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny,
                     size_t nz, size_t p1, size_t p2, int allocate, dfft_plan_t* plan) {
    return dfft_plan_create_batched(comm, config, decomp, precision, transform, nx, ny, nz, p1, p2, 1, allocate, plan);
}

}  // extern "C"

// Plan features, as bits: what a plan description or a plan has, and what a creator or a setter adds.  A description
// has the feature of the creator that made it (F_BOXES, F_PADDED, F_PRUNED, F_INTERLEAVED or F_KINDS) whatever its
// arguments; a plan has F_PADDED, F_PRUNED and F_INTERLEAVED when its K, M or C says so.
enum Feature : unsigned {
    F_HALF = 1u << 0,         // 16-bit storage (DFFT_F16 / DFFT_BF16)
    F_R2R = 1u << 1,          // a DCT / DST transform or per-axis kinds
    F_INPLACE = 1u << 2,      // dfft_plan_create_inplace, or in place by dfft_plan_create_r2r
    F_BOXES = 1u << 3,        // dfft_plan_create_boxes
    F_PADDED = 1u << 4,       // dfft_plan_create_padded; a plan with K < N
    F_PRUNED = 1u << 5,       // dfft_plan_create_pruned; a plan with M < N
    F_INTERLEAVED = 1u << 6,  // dfft_plan_create_interleaved; a plan of more than one component
    F_KINDS = 1u << 7,        // dfft_plan_create_r2r
    F_KEPT_AXES = 1u << 8,    // dfft_plan_set_transform_axes with an axis kept
    F_STRIDES = 1u << 9,      // dfft_plan_set_strides
    F_WEIGHTS = 1u << 10,     // dfft_plan_set_weights
    F_1D = 1u << 11,          // dfft_plan_create_1d
};

// The features that do not combine, in the order they are refused: adding `adds` to a description or a plan that has
// `with` returns DFFT_ERR_UNSUPPORTED.  A row with F_HALF names what has no 16-bit storage.
struct Refusal { unsigned adds, with; const char* what; };
static const Refusal refusals[] = {
    {F_BOXES, F_HALF, "box plans"},
    {F_PADDED, F_HALF, "padded plans"},
    {F_PRUNED, F_HALF, "pruned plans"},
    {F_INTERLEAVED, F_HALF, "interleaved plans"},
    {F_KINDS, F_HALF, "real-to-real plans"},
    {F_HALF, F_R2R, "DCT / DST plans"},
    {F_KEPT_AXES, F_PADDED, "padded plans transform every axis"},
    {F_KEPT_AXES, F_PRUNED, "pruned plans transform every axis"},
    {F_KEPT_AXES, F_INTERLEAVED, "interleaved plans transform every axis"},
    {F_STRIDES, F_HALF, "plans with strides"},
    {F_STRIDES, F_INPLACE, "in-place plans keep the padded layout of FFTW and cuFFT: strides are for out-of-place plans"},
    {F_STRIDES, F_INTERLEAVED, "interleaved plans keep their [x][y][z][C] layout: strides are for plans of one component"},
    {F_STRIDES, F_PRUNED, "pruned plans read and write dense data blocks: strides are for plans without a data size"},
    {F_WEIGHTS, F_INTERLEAVED, "interleaved plans of more than one component have no spectral weights"},
    {F_WEIGHTS, F_R2R, "real-to-real plans (DCT / DST and per-axis kinds) have no spectral weights"},
    {F_WEIGHTS, F_HALF, "spectral weights"},
    {F_1D, F_HALF, "1D plans"},
    {F_KEPT_AXES, F_1D, "1D plans transform every axis of their grid"},
    {F_STRIDES, F_1D, "1D plans read and write dense chunks of the signal: strides are for 3D plans"},
    {F_WEIGHTS, F_1D, "1D plans have no spectral weights"},
};
// The first refusal of adding `adds` to a description or a plan with the features `has`, or DFFT_SUCCESS
static int refuse(unsigned has, unsigned adds) {
    for (const Refusal& r : refusals)
        if ((r.adds & adds) && (r.with & has))
            return (r.adds | r.with) & F_HALF ? refuse_half(r.what) : fail(DFFT_ERR_UNSUPPORTED, r.what);
    return DFFT_SUCCESS;
}
static unsigned features(const dfft_plan_s* p) {
    return (is_half(p->prec) ? F_HALF : 0) | (is_r2r(p->g.transform) ? F_R2R : 0) | (p->inplace ? F_INPLACE : 0) | (p->g.padded() ? F_PADDED : 0) |
           (p->g.pruned() ? F_PRUNED : 0) | (p->comps > 1 ? F_INTERLEAVED : 0) | (p->n1d ? F_1D : 0);
}

// bytes of one element: complex, or real for DCT / DST plans
static size_t elem_bytes(int precision, int transform) {
    return (precision == DFFT_F64 ? 16 : is_half(precision) ? 4 : 8) / (is_r2r(transform) ? 2 : 1);
}

// The description of a plan: what one dfft_plan_create* entry point asks for.  Each creator sets the fields of its feature.
struct PlanSpec {
    unsigned made_by;  // F_BOXES, F_PADDED, F_PRUNED, F_INTERLEAVED, F_KINDS or F_1D; 0 for dfft_plan_create_batched / _inplace
    int decomp, precision, transform;
    size_t n[3], p1, p2, batch;
    bool inplace = false;
    const int* kinds = nullptr;                 // dfft_plan_create_r2r: the kinds of the x, y and z axis
    size_t comps = 1;                           // values per grid point
    size_t k[3] = {0, 0, 0}, m[3] = {0, 0, 0};  // the spectral and data sizes; 0: the grid
    std::vector<Box> boxes[2];                  // the in and out box of every rank; empty: that side has its natural layout
    size_t signal = 0;                          // dfft_plan_create_1d: N, with n the factors N1, N2, N3 (0 where none was found)
    bool natural = false;                       // dfft_plan_create_1d_natural: the output in natural order
    PlanSpec(unsigned made_by_, int decomp_, int precision_, int transform_, size_t nx, size_t ny, size_t nz, size_t p1_, size_t p2_, size_t batch_)
        : made_by(made_by_), decomp(decomp_), precision(precision_), transform(transform_), n{nx, ny, nz}, p1(p1_), p2(p2_), batch(batch_) {}
    unsigned features() const { return made_by | (is_half(precision) ? F_HALF : 0) | (is_r2r(transform) ? F_R2R : 0) | (inplace ? F_INPLACE : 0); }
};

// The spectral (padded, pruned) or data (pruned) sizes of a plan
static int check_sub_grid(const size_t n[3], const size_t sizes[3], const char* what) {
    for (int a = 0; a < 3; ++a) {
        if (sizes[a] == 0 || sizes[a] > n[a])
            return fail(DFFT_ERR_INVALID, std::string(what) + " size " + std::to_string(sizes[a]) + " of axis " + "xyz"[a] + " must be in [1, " +
                                              std::to_string(n[a]) + "]");
        if (sizes[a] < n[a] && ilog2_exact(n[a]) < 0)
            return fail(DFFT_ERR_UNSUPPORTED, std::string("axis ") + "xyz"[a] + " of length " + std::to_string(n[a]) + " is not a power of two: its " +
                                                  what + " size must be its length");
    }
    return DFFT_SUCCESS;
}

// C values per point: the C = 1 plan with every element widened to C consecutive values (DESIGN.md section 3.14).  The
// z pass of C > 1 runs interleaved lines (PASS_C2C_ILV) or R2C / C2R lines of Nz points, one per component (PASS_R2C_ILV /
// PASS_C2R_ILV), which exist for a power-of-two Nz (R2C: up to 8192).
constexpr size_t MAX_COMPONENTS = 64;

// Every rule a plan description must meet, checked before anything is allocated: first the rules of the creator that
// made it, then those of every plan.  The order decides which error an input with several faults gets.  g: the plan's
// geometry.
static int check_spec(dfft_comm_t comm, const dfft_plan_t* plan, const PlanSpec& s, Geometry& g) {
    const unsigned has = s.features();
    const size_t* n = s.n;
    if (s.made_by == F_BOXES && (!comm || !plan)) return fail(DFFT_ERR_INVALID, "null comm / plan");
    if (int rc = refuse(has, s.made_by)) return rc;
    if (s.made_by == F_BOXES) {  // DESIGN.md section 3.17
        if (s.transform != DFFT_C2C && s.transform != DFFT_R2C && s.transform != DFFT_DCT && s.transform != DFFT_DST)
            return fail(DFFT_ERR_INVALID, "box plans are C2C, R2C / C2R, DCT or DST");
        const size_t grid[2][3] = {{n[0], n[1], n[2]}, {n[0], n[1], s.transform == DFFT_R2C ? n[2] / 2 + 1 : n[2]}};
        for (int side = 0; side < 2; ++side)
            if (!s.boxes[side].empty() && !tiles(s.boxes[side], grid[side]))
                return fail(DFFT_ERR_INVALID, std::string(side ? "out_boxes" : "in_boxes") +
                                                  " must tile the grid: every box non-empty and inside it, no two overlapping, together all of it");
        // the real side of R2C / C2R plans moves as pairs of reals (the z pass's complex units)
        if (s.transform == DFFT_R2C)
            for (const Box& b : s.boxes[0])
                if (b.lo[2] % 2 || b.hi[2] % 2) return fail(DFFT_ERR_UNSUPPORTED, "R2C / C2R box plans need even z bounds in in_boxes");
    } else if (s.made_by == F_PADDED || s.made_by == F_PRUNED) {
        if (s.transform == DFFT_DCT || s.transform == DFFT_DST)
            return fail(DFFT_ERR_UNSUPPORTED, s.made_by == F_PADDED ? "padded plans are C2C or R2C / C2R" : "pruned plans are C2C or R2C / C2R");
        if (s.transform != DFFT_C2C && s.transform != DFFT_R2C) return fail(DFFT_ERR_INVALID, "bad transform");
        if (s.made_by == F_PRUNED)
            if (int rc = check_sub_grid(n, s.m, "data")) return rc;
        if (int rc = check_sub_grid(n, s.k, "spectral")) return rc;
        // the real side of R2C / C2R moves as pairs of reals (the z pass's complex units)
        if (s.made_by == F_PRUNED && s.transform == DFFT_R2C && s.m[2] % 2)
            return fail(DFFT_ERR_UNSUPPORTED, "R2C / C2R pruned plans need an even data size along z");
    } else if (s.made_by == F_INTERLEAVED) {
        if (s.comps == 0) return fail(DFFT_ERR_INVALID, "components must be at least 1");
        if (s.comps > MAX_COMPONENTS) return fail(DFFT_ERR_UNSUPPORTED, "at most " + std::to_string(MAX_COMPONENTS) + " components per point");
        if (s.comps > 1) {
            if (s.transform != DFFT_C2C && s.transform != DFFT_R2C && !is_r2r(s.transform)) return fail(DFFT_ERR_INVALID, "bad transform");
            if (is_r2r(s.transform)) return fail(DFFT_ERR_UNSUPPORTED, "interleaved plans with more than one component are C2C or R2C / C2R");
            if (ilog2_exact(n[2]) < 1) return fail(DFFT_ERR_UNSUPPORTED, "interleaved plans need a power-of-two Nz (x and y may have any C2C length)");
            // the interleaved R2C / C2R z pass runs Nz-point complex lines
            if (s.transform == DFFT_R2C && ilog2_exact(n[2]) > MAX_LOG2N)
                return fail(DFFT_ERR_UNSUPPORTED, "interleaved R2C / C2R plans need Nz <= " + std::to_string(1 << MAX_LOG2N));
        }
    } else if (s.made_by == F_1D) {  // DESIGN.md section 3.22
        if (!comm || !plan) return fail(DFFT_ERR_INVALID, "null comm / plan");
        const int l = ilog2_exact(s.signal);
        if (l < 3 || l > 3 * MAX_LOG2N)
            return fail(DFFT_ERR_UNSUPPORTED, "1D plans take n a power of two in [8, 2^" + std::to_string(3 * MAX_LOG2N) + "]");
        if (n[0] == 0)
            return fail(DFFT_ERR_UNSUPPORTED, "n = " + std::to_string(s.signal) + " has no split into three powers of two in [2, 8192] with " +
                                                  (s.natural ? "N1, N2 and N3" : "N1 and N2") + " at least the rank count");
        if (!pow2_length(n[0]) || !pow2_length(n[1]) || !pow2_length(n[2]))
            return fail(DFFT_ERR_UNSUPPORTED, "the factors of a 1D plan must be powers of two in [2, 8192]");
        if (n[0] * n[1] * n[2] != s.signal) return fail(DFFT_ERR_INVALID, "the factors of a 1D plan must multiply to n");
        if (n[0] < size_t(comm->nranks) || n[1] < size_t(comm->nranks))
            return fail(DFFT_ERR_INVALID, "the factors N1 and N2 of a 1D plan must be at least the rank count, so that every rank holds data");
        if (s.natural && n[2] < size_t(comm->nranks))
            return fail(DFFT_ERR_INVALID, "the factor N3 of a natural-order 1D plan must be at least the rank count, so that every rank holds "
                                          "output");
    } else if (s.made_by == F_KINDS) {
        if (!s.kinds) return fail(DFFT_ERR_INVALID, "null kinds");
        for (int a = 0; a < 3; ++a)
            if (!is_r2r_kind(s.kinds[a]))
                return fail(DFFT_ERR_INVALID, "kinds must be DFFT_DCT, DFFT_DST, DFFT_R2HC, DFFT_DCT1, DFFT_DST1, DFFT_DCT4 or DFFT_DST4");
    }

    if (!comm || !plan) return fail(DFFT_ERR_INVALID, "null comm / plan");
    if (s.batch == 0) return fail(DFFT_ERR_INVALID, "batch must be at least 1");
    if (s.precision < DFFT_F32 || s.precision > DFFT_BF16) return fail(DFFT_ERR_INVALID, "bad precision");
    if (s.transform != DFFT_R2C && s.transform != DFFT_C2C && !is_r2r(s.transform)) return fail(DFFT_ERR_INVALID, "bad transform");
    if (s.transform == DFFT_R2HC && !s.kinds) return fail(DFFT_ERR_INVALID, "bad transform (per-axis kinds: dfft_plan_create_r2r)");
    if (int rc = refuse(has, has & F_HALF)) return rc;
    if (is_half(s.precision) && s.transform == DFFT_C2C && !(pow2_length(n[0]) && pow2_length(n[1]) && pow2_length(n[2])))
        return fail(DFFT_ERR_UNSUPPORTED, "16-bit storage (DFFT_F16 / DFFT_BF16) takes power-of-two lengths in [2, 8192] only (no Bluestein pass)");
    if (!g.init(s.decomp, s.transform, n[0], n[1], n[2], s.p1, s.p2, comm->nranks, s.k[0], s.k[1], s.k[2], s.m[0], s.m[1], s.m[2]))
        return fail(DFFT_ERR_INVALID, "invalid partition: P1*P2 must equal the communicator size");
    if (s.transform == DFFT_C2C) {
        if (!c2c_length(n[0]) || !c2c_length(n[1]) || !c2c_length(n[2]))
            return fail(DFFT_ERR_UNSUPPORTED, "Nx, Ny, Nz of C2C plans must be powers of two in [2, 8192] or any length in [3, 4096]");
    } else if (is_r2r(s.transform)) {
        for (int a = 0; a < 3; ++a) {
            const int kind = s.kinds ? s.kinds[a] : s.transform;
            if (!r2r_kind_length(kind, n[a]))
                return fail(DFFT_ERR_UNSUPPORTED, kind == DFFT_DCT1   ? "DCT-I axes must have 2^k + 1 points in [3, 8193]"
                                                  : kind == DFFT_DST1 ? "DST-I axes must have 2^k - 1 points in [3, 8191]"
                                                  : is_type4(kind)    ? "DCT-IV / DST-IV axes must have 2^k points in [4, 8192]"
                                                                      : "Nx, Ny, Nz of DCT / DST plans must be powers of two in [2, 8192]");
        }
    } else if (ilog2_exact(n[0]) < 1 || ilog2_exact(n[1]) < 1 || ilog2_exact(n[2]) < 1 || ilog2_exact(n[0]) > MAX_LOG2N ||
               ilog2_exact(n[1]) > MAX_LOG2N || ilog2_exact(n[2]) > MAX_LOG2N + 1 || n[2] < 4) {
        return fail(DFFT_ERR_UNSUPPORTED, "Nx, Ny, Nz must be powers of two in [2, 8192] (Nz >= 4 for R2C)");
    }
    // every rank needs a non-empty share along each split axis
    if (g.sx.size.back() == 0 || g.sy.size.back() == 0 || g.sz.size.back() == 0 || g.oy.size.back() == 0)
        return fail(DFFT_ERR_INVALID, "partition leaves a rank without data");
    // the whole batch of every caller buffer (any direction, any partial d: field_bytes) must be addressable
    const int r = comm->rank;
    const size_t es = elem_bytes(s.precision, s.transform) * s.comps, real_es = s.transform == DFFT_R2C ? es / 2 : es;
    auto points = [&](int which) {  // of this rank's caller array of layout `which`: its box, if that side has boxes
        const std::vector<Box>* b = which == 0 ? &s.boxes[0] : which == 3 ? &s.boxes[1] : nullptr;
        if (b && !b->empty()) return (*b)[size_t(r)].volume();
        size_t sz[3], o[3];
        g.layout(r, which, sz, o);
        return sz[0] * sz[1] * sz[2];
    };
    size_t widest = s.inplace ? g.domain_elems(r) * es : points(0) * real_es;
    for (int d = 1; d <= 3 && !s.inplace; ++d) widest = std::max(widest, points(d) * es);
    if (s.batch > SIZE_MAX / widest)
        return fail(DFFT_ERR_INVALID, "batch of " + std::to_string(s.batch) + " fields of " + std::to_string(widest) +
                                          " bytes overflows the address range (size_t)");
    return DFFT_SUCCESS;
}

static int plan_create(dfft_comm_t comm, const dfft_config* config, const PlanSpec& s, int allocate, dfft_plan_t* plan) {
    Geometry geom;
    if (int rc = check_spec(comm, plan, s, geom)) return rc;
    const int decomp = s.decomp, precision = s.precision, transform = s.transform;
    const size_t nx = s.n[0], ny = s.n[1], nz = s.n[2], comps = s.comps;
    const bool dry = comm->dry, inplace = s.inplace;
    if (!dry) CK_CUDA(cudaSetDevice(comm->device));
    const auto t_init0 = std::chrono::steady_clock::now();
    dfft_plan_s* p = new dfft_plan_s();
    p->comm = comm;
    if (config) {
        p->cfg = *config;
        if (config->benchmark_dir) p->bench_dir = config->benchmark_dir;
        p->cfg.benchmark_dir = nullptr;
    } else {
        p->cfg.comm_method = DFFT_PEER2PEER; p->cfg.comm_method2 = DFFT_PEER2PEER;
    }
    p->rank = comm->rank; p->P = comm->nranks;
    p->prec = precision;
    for (int a = 0; a < 3; ++a) p->kinds[a] = s.kinds ? s.kinds[a] : is_r2r(transform) ? transform : 0;
    p->esize = elem_bytes(precision, transform);
    p->comps = comps;
    p->tabs.prec = precision;
    p->tabs.dry = dry;
    p->g = geom;
    const Geometry& g = p->g;
    p->inplace = inplace;
    p->batch = s.batch;
    p->n1d = s.signal;
    if (s.natural) p->oz.make(nz, size_t(comm->nranks));
    // box plans: a side whose boxes are all natural keeps no boxes, so that it makes exactly the plan of
    // dfft_plan_create_batched
    auto keep_boxes = [&](const std::vector<Box>& b, int which, std::vector<Box>& dst) {
        for (int r = 0; r < int(b.size()); ++r) {
            size_t s_[3], o_[3];
            g.layout(r, which, s_, o_);
            if (!(b[size_t(r)] == Box::of(s_, o_))) { dst = b; return; }
        }
    };
    keep_boxes(s.boxes[0], 0, p->in_boxes);
    keep_boxes(s.boxes[1], 3, p->out_boxes);
    // elements (of the schedule's views) of rank r's box arrays: the real side of R2C / C2R in complex pairs
    auto box_elems = [&](int r) {
        size_t m = 0;
        if (!p->in_boxes.empty()) m = p->in_boxes[size_t(r)].volume() / (transform == DFFT_R2C ? 2 : 1);
        if (!p->out_boxes.empty()) m = std::max(m, p->out_boxes[size_t(r)].volume());
        return m;
    };
    // the largest stage array of this rank; it also covers the padded real input of in-place R2C plans, which has the
    // extent of the layout after d = 1
    // natural-order 1D plans: and the output chunk [oz_r][N2][N1], which the landing slot holds too
    auto chunk_elems = [&](int r) { return p->oz.size.empty() ? 0 : p->oz.size[size_t(r)] * ny * nx; };
    p->domain_bytes = std::max({g.domain_elems(p->rank), box_elems(p->rank), chunk_elems(p->rank)}) * p->esize * comps;
    // groups
    const int me = p->rank, P = p->P;
    p->grp[0].clear();
    for (int r = 0; r < P; ++r) p->grp[0].push_back(r);
    if (decomp == DFFT_PENCIL) {
        const int i = g.pi(me), j = g.pj(me);
        for (int q = 0; q < g.P2; ++q) p->grp[1].push_back(i * g.P2 + q);
        for (int q = 0; q < g.P1; ++q) p->grp[2].push_back(q * g.P2 + j);
    } else if (decomp == DFFT_SLAB_ZY_THEN_X) {
        p->grp[1].push_back(me);
        p->grp[2] = p->grp[0];
    } else {
        p->grp[1] = p->grp[0];
        p->grp[2].push_back(me);
    }
    p->direct1 = p->cfg.comm_method != DFFT_ALL2ALL;
    p->direct2 = (decomp == DFFT_PENCIL ? p->cfg.comm_method2 : p->cfg.comm_method) != DFFT_ALL2ALL;
    if (decomp == DFFT_SLAB_ZY_THEN_X) p->direct1 = true;   // trivial group
    if (decomp == DFFT_SLAB_Z_THEN_YX) p->direct2 = true;
    p->any_direct = (p->direct1 && p->grp[1].size() > 1) || (p->direct2 && p->grp[2].size() > 1);
    p->slots = plan_slots(p->direct1 || p->grp[1].size() == 1, p->direct2 || p->grp[2].size() == 1);
    if (p->boxed()) {
        // the reshapes: over peer memory with comm_method Peer2Peer (which needs the peer mapping and the entry rendezvous),
        // else through the all-to-all slots; and their staging slot BX
        p->box_direct = p->cfg.comm_method != DFFT_ALL2ALL;
        if (p->box_direct) p->any_direct = true;
        else if (p->slots.SS < 0) { p->slots.SS = p->slots.count++; p->slots.SR = p->slots.count++; }
        p->slots.BX = p->slots.count++;
    }
    // in place on one rank the caller's buffer is the schedules' first slot (D1; both transpositions are local there)
    p->buf_slot = inplace && P == 1;
    p->nslots = p->slots.count - (p->buf_slot ? 1 : 0);
    size_t dom = 0;
    for (int r = 0; r < P; ++r) dom = std::max({dom, g.domain_elems(r), box_elems(r), chunk_elems(r)});
    p->slot_bytes = ((dom * p->esize * comps + 255) / 256) * 256;
    p->work_bytes = p->slot_bytes * p->nslots;
    {
        const char* e = getenv("DFFT_XCHG_CTAS");
        // untuned default, not measured on H100s: two thirds of an H100's 132 SMs for the exchanging pass, the rest for
        // the local passes (dfft_plan_tune replaces it by the best of its measured candidates)
        p->xchg_ctas = e ? atoi(e) : 88;
        // Blocked intermediate layout for the slab's y -> x hand-over: [Nzc/CH][Nx][Ny_q][CH].  The rows a y-pass tile
        // sends to one destination are adjacent (512-byte warp stores instead of 64-byte rows: what NVLink needs),
        // and the x pass reads rows 16 KB apart instead of one row per 2 MB page (tools/layout_probe.py).
        // The Nzc % CH leftover columns (one for R2C plans: Nzc = Nz/2+1) travel in a small plain-layout tail region
        // behind the blocked part, handled by two tiny extra launches.  DFFT_BLOCKED=0 disables.
        // NVLink store efficiency grows with the contiguous run per row (64-byte rows waste much of every write
        // packet, 128-byte rows and longer runs do not): exchanging passes prefer the wide tile even though it is
        // slower as a purely local pass.  DFFT_XCHG_WIDE=0 keeps the narrow tile.
        if (const char* eg = getenv("DFFT_OVL_GROUPS")) p->ovl_groups = std::max(1, std::min(16, atoi(eg)));
        if (const char* ec = getenv("DFFT_OVL_CHUNKS")) p->ovl_chunks = std::max(1, std::min(16, atoi(ec)));
        const char* et = getenv("DFFT_RENDEZVOUS_TIMEOUT_S");
        const double tsec = et ? atof(et) : 300.0;
        p->rendezvous_timeout_cycles = tsec > 0 ? (long long)(tsec * 1.9e9) : 0;  // clock64 ticks at <= 1.98 GHz (H100 SXM)
        const char* ebs = getenv("DFFT_BULK_STORE");
        p->bulk_store = (ebs && atoi(ebs) != 0) ? 1 : 0;
        const char* ew = getenv("DFFT_XCHG_WIDE");
        p->xchg_tile_pref = (ew && atoi(ew) == 0) ? 1 : 2;
        if (const char* ebi = getenv("DFFT_BLOCKED_INV")) p->blocked_inv = atoi(ebi) != 0;
        // one rank: x innermost up to 512-point y lines; for 1024-point y lines its output rows lie one per 2 MB page,
        // so the general blocked layout is used there (design choice, to be confirmed on the H100)
        p->single_rank_layout = ny < 1024 ? 1 : 0;
        if (const char* en1 = getenv("DFFT_N1_LAYOUT")) p->single_rank_layout = atoi(en1) != 0;
        if (const char* esw = getenv("DFFT_X_SWZ")) p->x_swz = std::max(0, std::min(4, atoi(esw)));
        const char* eb = getenv("DFFT_BLOCKED");
        // block width = the widest tile the y and x passes use for these lengths (fft_kernels.cuh: Shape::TBT —
        // 4096 points per tile, rows of at least 64 bytes, at most 32 columns), never below 8 elements
        auto tile_cols = [&](size_t n) {
            size_t w = 4096 / n, lo = precision == DFFT_F64 ? 4 : 8;
            return w < lo ? lo : (w > 32 ? size_t(32) : w);
        };
        int ch = int(std::max<size_t>(8, std::max(tile_cols(ny), tile_cols(nx))));
        // DCT / DST: the R2R tile holds that many column pairs, so the block is twice as many reals wide
        if (is_r2r(transform)) ch = int(2 * std::max(tile_cols(ny), tile_cols(nx)));
        if (eb) ch = atoi(eb);
        size_t min_nz = g.kzc;  // smallest z extent any rank holds between the y and x passes
        if (decomp == DFFT_PENCIL)
            for (size_t v : g.sz.size) min_nz = std::min(min_nz, v);
        p->blocked_ch = ((decomp == DFFT_SLAB_ZY_THEN_X || decomp == DFFT_PENCIL) && ch > 0 && min_nz >= size_t(4 * ch)) ? ch : 0;
    }
    if (dry) {
        // fake, rank-distinct slot addresses: ((rank + 1) << 44) + slot * slot_bytes; user buffers are offsets
        p->slot_ptr.assign(p->nslots, std::vector<void*>(P, nullptr));
        for (int s_ = 0; s_ < p->nslots; ++s_)
            for (int r = 0; r < P; ++r) p->slot_ptr[s_][r] = (void*)(((unsigned long long)(r + 1) << 44) + (unsigned long long)s_ * p->slot_bytes);
        p->work = p->slot_ptr[0][me];
        *plan = p;
        return DFFT_SUCCESS;
    }
    // The plan's own stream is a BLOCKING stream: like the reference's cuFFT execs on the legacy default stream
    // (mpicufft_slab.cpp:788-807) the synchronous dfft_exec_* calls are ordered behind everything the caller queued on
    // the default stream before the call — a pageable cudaMemcpy whose DMA is still in flight, a kernel that is still
    // filling `in` (the reference's own testcase 4 does exactly that: random_dist_default.cu:719-724).
    cudaError_t ce = cudaStreamCreate(&p->own_stream);
    if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&p->entry_ev, cudaEventDisableTiming);
    if (ce != cudaSuccess) { delete p; return fail(DFFT_ERR_CUDA, "cudaStreamCreate failed"); }
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);  // hi = numerically lowest = highest priority
        if (cudaStreamCreateWithPriority(&p->aux[0], cudaStreamNonBlocking, hi) != cudaSuccess ||
            cudaStreamCreateWithPriority(&p->aux[1], cudaStreamNonBlocking, lo) != cudaSuccess ||
            cudaEventCreateWithFlags(&p->fork_ev, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&p->join_ev[0], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&p->join_ev[1], cudaEventDisableTiming) != cudaSuccess) {
            delete p;
            return fail(DFFT_ERR_CUDA, "stream / event creation failed");
        }
    }
    {
        int l2 = 0;
        if (cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, comm->device) == cudaSuccess && l2 > 0) p->l2_bytes = size_t(l2);
    }
    int rc = plan_setup_flags(p);
    if (rc == DFFT_SUCCESS && allocate) rc = plan_setup_memory(p, nullptr);
    if (rc != DFFT_SUCCESS) {
        std::string keep = g_err;
        dfft_plan_destroy(p);
        g_err = keep;
        return rc;
    }
    p->init_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_init0).count();
    if (!p->bench_dir.empty()) {
        // <dir>/<variant>/test_0_<comm>_<snd>[_<comm2>_<snd2>]_<Nx>_<Ny>_<Nz>_<cuda_aware>_<P | P1_P2>.csv
        const char* variant = decomp == DFFT_PENCIL ? "pencil" : (decomp == DFFT_SLAB_Z_THEN_YX ? "slab_z_then_yx" : "slab_default");
        mkdir(p->bench_dir.c_str(), 0777);
        mkdir((p->bench_dir + "/" + variant).c_str(), 0777);
        std::string f = p->bench_dir + "/" + variant + "/test_0_" + std::to_string(p->cfg.comm_method) + "_" + std::to_string(p->cfg.send_method);
        if (decomp == DFFT_PENCIL) f += "_" + std::to_string(p->cfg.comm_method2) + "_" + std::to_string(p->cfg.send_method2);
        f += "_" + std::to_string(nx) + "_" + std::to_string(ny) + "_" + std::to_string(nz) + "_" + std::to_string(p->cfg.cuda_aware ? 1 : 0);
        if (decomp == DFFT_PENCIL) f += "_" + std::to_string(g.P1) + "_" + std::to_string(g.P2);
        else f += "_" + std::to_string(P);
        p->csv_path = f + ".csv";
        p->csv_warmup_left = p->cfg.warmup_rounds;
        p->timing = true;
    }
    *plan = p;
    return DFFT_SUCCESS;
}

extern "C" {

int dfft_plan_create_batched(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny,
                             size_t nz, size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan) {
    return plan_create(comm, config, PlanSpec(0, decomp, precision, transform, nx, ny, nz, p1, p2, batch), allocate, plan);
}

int dfft_plan_create_inplace(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny,
                             size_t nz, size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan) {
    PlanSpec s(0, decomp, precision, transform, nx, ny, nz, p1, p2, batch);
    s.inplace = true;
    return plan_create(comm, config, s, allocate, plan);
}

int dfft_plan_is_inplace(dfft_plan_t p) { return p && p->inplace ? 1 : 0; }

// Box plans (DESIGN.md section 3.17): six values (lo, hi) per rank on each side that has boxes
int dfft_plan_create_boxes(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny, size_t nz,
                           size_t p1, size_t p2, const size_t* in_boxes, const size_t* out_boxes, size_t batch, int allocate, dfft_plan_t* plan) {
    PlanSpec s(F_BOXES, decomp, precision, transform, nx, ny, nz, p1, p2, batch);
    const size_t* given[2] = {in_boxes, out_boxes};
    for (int side = 0; side < 2; ++side)
        for (int r = 0; given[side] && comm && r < comm->nranks; ++r) {
            Box b;
            for (int a = 0; a < 3; ++a) { b.lo[a] = given[side][6 * r + a]; b.hi[a] = given[side][6 * r + 3 + a]; }
            s.boxes[side].push_back(b);
        }
    return plan_create(comm, config, s, allocate, plan);
}

int dfft_plan_create_padded(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny,
                            size_t nz, size_t kx, size_t ky, size_t kz, size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan) {
    PlanSpec s(F_PADDED, decomp, precision, transform, nx, ny, nz, p1, p2, batch);
    s.k[0] = kx; s.k[1] = ky; s.k[2] = kz;
    return plan_create(comm, config, s, allocate, plan);
}

// Pruned plans (DESIGN.md section 3.19): the data block [0, M) of each axis, zero beyond, and the spectrum of a padded plan.
int dfft_plan_create_pruned(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny,
                            size_t nz, const size_t data[3], const size_t spectral[3], size_t p1, size_t p2, size_t batch, int allocate,
                            dfft_plan_t* plan) {
    PlanSpec s(F_PRUNED, decomp, precision, transform, nx, ny, nz, p1, p2, batch);
    for (int a = 0; a < 3; ++a) {
        s.m[a] = data ? data[a] : s.n[a];
        s.k[a] = spectral ? spectral[a] : s.n[a];
    }
    return plan_create(comm, config, s, allocate, plan);
}

int dfft_plan_get_data_size(dfft_plan_t p, size_t m[3]) {
    if (!p || !m) return fail(DFFT_ERR_INVALID, "null plan / size");
    m[0] = p->g.mx; m[1] = p->g.my; m[2] = p->g.mz;
    return DFFT_SUCCESS;
}

int dfft_plan_create_interleaved(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, int transform, size_t nx, size_t ny,
                                 size_t nz, size_t p1, size_t p2, size_t components, size_t batch, int allocate, dfft_plan_t* plan) {
    PlanSpec s(F_INTERLEAVED, decomp, precision, transform, nx, ny, nz, p1, p2, batch);
    s.comps = components;
    return plan_create(comm, config, s, allocate, plan);
}
size_t dfft_get_components(dfft_plan_t p) { return p ? p->comps : 0; }

int dfft_plan_get_spectral_size(dfft_plan_t p, size_t k[3]) {
    if (!p || !k) return fail(DFFT_ERR_INVALID, "null plan / size");
    k[0] = p->g.kx; k[1] = p->g.ky; k[2] = p->g.kz;
    return DFFT_SUCCESS;
}

int dfft_plan_create_r2r(dfft_comm_t comm, const dfft_config* config, int decomp, int precision, const int kinds[3], size_t nx, size_t ny,
                         size_t nz, size_t p1, size_t p2, size_t batch, int inplace, int allocate, dfft_plan_t* plan) {
    // three DCT (DST) axes make exactly the DCT (DST) plan; type-I and type-IV kinds, like R2HC, make a per-axis plan
    const bool uniform = kinds && kinds[0] == kinds[1] && kinds[1] == kinds[2] && (kinds[0] == DFFT_DCT || kinds[0] == DFFT_DST);
    PlanSpec s(F_KINDS, decomp, precision, uniform ? kinds[0] : DFFT_R2HC, nx, ny, nz, p1, p2, batch);
    s.kinds = kinds;
    s.inplace = inplace != 0;
    return plan_create(comm, config, s, allocate, plan);
}

int dfft_plan_get_r2r_kinds(dfft_plan_t p, int kinds[3]) {
    if (!p || !kinds) return fail(DFFT_ERR_INVALID, "null plan / kinds");
    if (!is_r2r(p->g.transform)) return fail(DFFT_ERR_INVALID, std::string("plan was created for ") + transform_name(p->g.transform));
    for (int a = 0; a < 3; ++a) kinds[a] = p->kinds[a];
    return DFFT_SUCCESS;
}

// 1D plans (DESIGN.md section 3.22).  Default factors: log2 N split into l1 + l2 + l3 with every l in [1, 13] and l1, l2
// at least ceil(log2 P) (N1, N2 >= P: no rank without data), the split with the smallest spread max(l) - min(l), and of
// those the largest l1, then the largest l2 (so N1 >= N2 >= N3 when nothing else decides).  All zero when none exists.
// natural: l3 at least ceil(log2 P) as well (N3 >= P: no rank without output, section 3.23).
static void default_factors(size_t n, int P, size_t f[3], bool natural) {
    f[0] = f[1] = f[2] = 0;
    const int L = ilog2_exact(n);
    int lp = 1;
    while ((1 << lp) < P) ++lp;
    int best = -1;
    for (int l1 = MAX_LOG2N; l1 >= lp; --l1)
        for (int l2 = MAX_LOG2N; l2 >= lp; --l2) {
            const int l3 = L - l1 - l2;
            if (L < 0 || l3 < (natural ? lp : 1) || l3 > MAX_LOG2N) continue;
            const int spread = std::max({l1, l2, l3}) - std::min({l1, l2, l3});
            if (best >= 0 && spread >= best) continue;
            best = spread;
            f[0] = size_t(1) << l1; f[1] = size_t(1) << l2; f[2] = size_t(1) << l3;
        }
}

static int create_1d(dfft_comm_t comm, const dfft_config* config, int precision, size_t n, const size_t factors[3], bool natural, dfft_plan_t* plan) {
    size_t f[3] = {0, 0, 0};
    if (factors) for (int a = 0; a < 3; ++a) f[a] = factors[a];
    else default_factors(n, comm ? comm->nranks : 1, f, natural);
    PlanSpec s(F_1D, DFFT_SLAB_ZY_THEN_X, precision, DFFT_C2C, f[0], f[1], f[2], comm ? size_t(comm->nranks) : 1, 1, 1);
    s.signal = n;
    s.natural = natural;
    return plan_create(comm, config, s, 1, plan);
}

int dfft_plan_create_1d(dfft_comm_t comm, const dfft_config* config, int precision, size_t n, const size_t factors[3], dfft_plan_t* plan) {
    return create_1d(comm, config, precision, n, factors, false, plan);
}

// natural-order output (DESIGN.md section 3.23): the same plan with N3 at least the rank count, and the z pass transposing
int dfft_plan_create_1d_natural(dfft_comm_t comm, const dfft_config* config, int precision, size_t n, const size_t factors[3], dfft_plan_t* plan) {
    return create_1d(comm, config, precision, n, factors, true, plan);
}

int dfft_plan_get_1d_factors(dfft_plan_t p, size_t f[3]) {
    if (!p || !f) return fail(DFFT_ERR_INVALID, "null plan / factors");
    if (!p->n1d) return fail(DFFT_ERR_INVALID, "not a 1D plan (dfft_plan_create_1d)");
    f[0] = p->g.nx; f[1] = p->g.ny; f[2] = p->g.nz;
    return DFFT_SUCCESS;
}

int dfft_plan_destroy(dfft_plan_t p) {
    if (!p) return DFFT_SUCCESS;
    if (p->comm->dry) {
        p->work = nullptr;
        p->tabs.release();
        delete p;
        return DFFT_SUCCESS;
    }
    cudaSetDevice(p->comm->device);
    cudaDeviceSynchronize();
    plan_release_memory(p);
    for (void* q : p->opened_flags) cudaIpcCloseMemHandle(q);
    if (p->flags) cudaFree(p->flags);
    if (p->peer_flags_d) cudaFree(p->peer_flags_d);
    if (p->groups_d) cudaFree(p->groups_d);
    if (p->err_d) cudaFree(p->err_d);
    p->tabs.release();
    for (cudaEvent_t e : p->events) cudaEventDestroy(e);
    for (cudaEvent_t e : p->tl_events) cudaEventDestroy(e);
    for (cudaEvent_t e : p->sync_events) cudaEventDestroy(e);
    if (p->fork_ev) cudaEventDestroy(p->fork_ev);
    for (int a = 0; a < 2; ++a) {
        if (p->join_ev[a]) cudaEventDestroy(p->join_ev[a]);
        if (p->aux[a]) cudaStreamDestroy(p->aux[a]);
    }
    if (p->own_stream) cudaStreamDestroy(p->own_stream);
    if (p->entry_ev) cudaEventDestroy(p->entry_ev);
    delete p;
    return DFFT_SUCCESS;
}

int dfft_set_work_area(dfft_plan_t p, void* device, void* host) {
    (void)host;
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    CK_CUDA(cudaSetDevice(p->comm->device));
    CK_CUDA(cudaDeviceSynchronize());
    return plan_setup_memory(p, device);
}

int dfft_exec_r2c(dfft_plan_t p, void* out, const void* in) { return exec_common(p, out, in, 0, 3, DFFT_R2C, nullptr, true); }
int dfft_exec_c2r(dfft_plan_t p, void* out, const void* in) { return exec_common(p, out, in, 1, 3, DFFT_R2C, nullptr, true); }
int dfft_exec_c2c(dfft_plan_t p, void* out, const void* in, int direction) {
    return exec_common(p, out, in, direction > 0 ? 1 : 0, 3, DFFT_C2C, nullptr, true);
}
int dfft_exec_r2c_partial(dfft_plan_t p, void* out, const void* in, int d) { return exec_common(p, out, in, 0, d, DFFT_R2C, nullptr, true); }
int dfft_exec_c2r_partial(dfft_plan_t p, void* out, const void* in, int d) { return exec_common(p, out, in, 1, d, DFFT_R2C, nullptr, true); }
int dfft_exec_c2c_partial(dfft_plan_t p, void* out, const void* in, int direction, int d) {
    return exec_common(p, out, in, direction > 0 ? 1 : 0, d, DFFT_C2C, nullptr, true);
}
int dfft_exec_r2c_async(dfft_plan_t p, void* out, const void* in, void* stream) { return exec_common(p, out, in, 0, 3, DFFT_R2C, stream, false); }
int dfft_exec_c2r_async(dfft_plan_t p, void* out, const void* in, void* stream) { return exec_common(p, out, in, 1, 3, DFFT_R2C, stream, false); }
int dfft_exec_c2c_async(dfft_plan_t p, void* out, const void* in, int direction, void* stream) {
    return exec_common(p, out, in, direction > 0 ? 1 : 0, 3, DFFT_C2C, stream, false);
}

int dfft_exec_r2r(dfft_plan_t p, void* out, const void* in, int direction) {
    return exec_common(p, out, in, direction > 0 ? 1 : 0, 3, EXEC_R2R, nullptr, true);
}
int dfft_exec_r2r_partial(dfft_plan_t p, void* out, const void* in, int direction, int d) {
    return exec_common(p, out, in, direction > 0 ? 1 : 0, d, EXEC_R2R, nullptr, true);
}
int dfft_exec_r2r_async(dfft_plan_t p, void* out, const void* in, int direction, void* stream) {
    return exec_common(p, out, in, direction > 0 ? 1 : 0, 3, EXEC_R2R, stream, false);
}

int dfft_plan_wait(dfft_plan_t p) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    CK_CUDA(cudaStreamSynchronize(p->last_stream));
    int err = 0;
    CK_CUDA(cudaMemcpy(&err, p->err_d, sizeof(int), cudaMemcpyDeviceToHost));
    if (err) {
        cudaMemset(p->err_d, 0, sizeof(int));
        if (err == ZY_ERR_TIMEOUT)
            return fail(DFFT_ERR_TIMEOUT, "fused z + y stage: a wait for the other phase timed out (DFFT_RENDEZVOUS_TIMEOUT_S); results are "
                                          "invalid and the plan must be destroyed");
        if (err == BATCH_ERR_TIMEOUT)
            return fail(DFFT_ERR_TIMEOUT, "batched stage: a wait for the other phase timed out (DFFT_RENDEZVOUS_TIMEOUT_S); results are "
                                          "invalid and the plan must be destroyed");
        if (err >= 100)
            return fail(DFFT_ERR_TIMEOUT, "a peer rank gave up waiting at a device rendezvous (phase " + std::to_string(err - 100) +
                                              "); results are invalid and the plan must be destroyed");
        return fail(DFFT_ERR_TIMEOUT, "device rendezvous timed out in phase " + std::to_string(err - 1) +
                                          " (a peer rank did not arrive; DFFT_RENDEZVOUS_TIMEOUT_S); results are invalid and the plan must be destroyed");
    }
    return DFFT_SUCCESS;
}

static int layout_of(dfft_plan_t p, int which, size_t size[3], size_t start[3]) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    size_t s[3], o[3];
    caller_block(p, which, s, o);
    for (int k = 0; k < 3; ++k) {
        if (size) size[k] = s[k];
        if (start) start[k] = o[k];
    }
    return DFFT_SUCCESS;
}
int dfft_get_in_size(dfft_plan_t p, size_t size[3]) { return layout_of(p, 0, size, nullptr); }
int dfft_get_in_start(dfft_plan_t p, size_t start[3]) { return layout_of(p, 0, nullptr, start); }
int dfft_get_out_size(dfft_plan_t p, size_t size[3]) { return layout_of(p, 3, size, nullptr); }
int dfft_get_out_start(dfft_plan_t p, size_t start[3]) { return layout_of(p, 3, nullptr, start); }
int dfft_get_partial_size(dfft_plan_t p, int d, size_t size[3]) {
    if (d < 1 || d > 3) return fail(DFFT_ERR_INVALID, "d must be 1..3");
    return layout_of(p, d, size, nullptr);
}
int dfft_get_partial_start(dfft_plan_t p, int d, size_t start[3]) {
    if (d < 1 || d > 3) return fail(DFFT_ERR_INVALID, "d must be 1..3");
    return layout_of(p, d, nullptr, start);
}
size_t dfft_get_domain_size(dfft_plan_t p) { return p ? p->domain_bytes : 0; }
size_t dfft_get_batch(dfft_plan_t p) { return p ? p->batch : 0; }
size_t dfft_get_work_size_device(dfft_plan_t p) { return p ? p->work_bytes : 0; }
size_t dfft_get_work_size_host(dfft_plan_t) { return 0; }
void* dfft_get_work_area_device(dfft_plan_t p) { return p ? p->work : nullptr; }
int dfft_get_rank(dfft_plan_t p) { return p ? p->rank : -1; }
int dfft_get_world_size(dfft_plan_t p) { return p ? p->P : -1; }

int dfft_plan_set_scale(dfft_plan_t p, double forward_scale, double inverse_scale) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (!std::isfinite(forward_scale) || !std::isfinite(inverse_scale)) return fail(DFFT_ERR_INVALID, "scale must be finite");
    p->scale[0] = forward_scale;
    p->scale[1] = inverse_scale;
    // the next exec of either direction may launch kernels that have not been set up yet: run it eagerly before a capture
    for (auto& dir : p->sched)
        for (Schedule& sc : dir) sc.executed = false;
    return DFFT_SUCCESS;
}
int dfft_plan_set_transform_axes(dfft_plan_t p, const int transform[3]) {
    if (!p || !transform) return fail(DFFT_ERR_INVALID, "null plan / transform");
    for (int a = 0; a < 3; ++a)
        if (transform[a] != 0 && transform[a] != 1) return fail(DFFT_ERR_INVALID, "transform axes must be 0 (keep) or 1 (transform)");
    if (p->g.transform == DFFT_R2C && !transform[2]) return fail(DFFT_ERR_INVALID, "R2C / C2R plans transform z (it turns reals into complex)");
    if (!(transform[0] && transform[1] && transform[2]))
        if (int rc = refuse(features(p), F_KEPT_AXES)) return rc;
    // schedules, tuned choices and captured graphs are built for the axes of their time
    if (p->axes_fixed) return fail(DFFT_ERR_STATE, "set the transform axes before the first exec, dfft_plan_tune or dfft_plan_describe");
    for (int a = 0; a < 3; ++a) p->taxes[a] = transform[a];
    return DFFT_SUCCESS;
}
int dfft_plan_get_transform_axes(dfft_plan_t p, int transform[3]) {
    if (!p || !transform) return fail(DFFT_ERR_INVALID, "null plan / transform");
    for (int a = 0; a < 3; ++a) transform[a] = p->taxes[a];
    return DFFT_SUCCESS;
}
int dfft_plan_set_strides(dfft_plan_t p, const long long in_strides[3], const long long out_strides[3]) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (int rc = refuse(features(p) & F_HALF, F_STRIDES)) return rc;  // 16-bit plans before the strides are looked at
    const char* const names[2] = {"in_strides", "out_strides"};
    const long long* const given[2] = {in_strides, out_strides};
    for (int side = 0; side < 2; ++side) {
        const long long* s = given[side];
        if (!s) continue;
        size_t e[3], o[3];
        caller_block(p, side ? 3 : 0, e, o);
        // the field, x and y strides may not let two points of the block (or of two fields) share an element
        const __int128 need[3] = {(__int128)e[0] * s[1], (__int128)e[1] * s[2], (__int128)e[2]};
        for (int k = 0; k < 3; ++k)
            if (s[k] < 1 || s[k] < need[k])
                return fail(DFFT_ERR_INVALID, std::string(names[side]) + ": strides {field, x, y} must be at least {nx * x, ny * y, nz} of this rank's block (" +
                                                  std::to_string(e[0]) + " x " + std::to_string(e[1]) + " x " + std::to_string(e[2]) + ")");
        if (side == 0 && p->g.transform == DFFT_R2C && ((s[0] | s[1] | s[2]) & 1))
            return fail(DFFT_ERR_INVALID, "in_strides: the real side of R2C / C2R moves pairs of reals, so its strides must be even");
    }
    if (int rc = refuse(features(p), F_STRIDES)) return rc;
    if (p->axes_fixed) return fail(DFFT_ERR_STATE, "set the strides before the first exec, dfft_plan_tune or dfft_plan_describe");
    p->in_embedded = in_strides != nullptr;
    p->out_embedded = out_strides != nullptr;
    for (int k = 0; k < 3; ++k) {
        p->in_strides[k] = in_strides ? in_strides[k] : 0;
        p->out_strides[k] = out_strides ? out_strides[k] : 0;
    }
    return DFFT_SUCCESS;
}
int dfft_plan_get_strides(dfft_plan_t p, long long in_strides[3], long long out_strides[3]) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    for (int side = 0; side < 2; ++side) {
        long long* s = side ? out_strides : in_strides;
        if (!s) continue;
        if (side ? p->out_embedded : p->in_embedded) {
            for (int k = 0; k < 3; ++k) s[k] = side ? p->out_strides[k] : p->in_strides[k];
            continue;
        }
        size_t e[3], o[3];  // a dense side: the strides of its dense block
        caller_block(p, side ? 3 : 0, e, o);
        s[2] = (long long)e[2];
        s[1] = (long long)(e[1] * e[2]);
        s[0] = (long long)(e[0] * e[1] * e[2]);
    }
    return DFFT_SUCCESS;
}
#ifdef DFFT_ZY_TRACE
// Trace build only (not part of include/dfft.h): copies the fused z + y stage's stamps of the last 3D exec in one direction
// (fft_kernels.cuh, ZyStamp) to host memory; returns the number of work items, or a negative dfft_status.
int dfft_zy_trace_copy(dfft_plan_t p, int inverse, void* host, size_t bytes) {
    if (!p || !host) return DFFT_ERR_INVALID;
    for (const Step& s : p->sched[inverse ? 1 : 0][2].steps) {
        if (s.kernel != KERNEL_ZY_FUSED || !s.zyf.trace) continue;
        const size_t items = 2 * size_t(p->g.nx) * (p->g.ny * p->g.nz / 4096);
        const size_t need = items * ZY_TRACE_SLOTS * sizeof(unsigned long long);
        if (bytes < need) return DFFT_ERR_INVALID;
        if (cudaMemcpy(host, s.zyf.trace, need, cudaMemcpyDeviceToHost) != cudaSuccess) return DFFT_ERR_CUDA;
        return int(items);
    }
    return DFFT_ERR_STATE;
}
#endif

int dfft_plan_set_weights(dfft_plan_t p, const void* const weights[3]) {
    if (!p || !weights) return fail(DFFT_ERR_INVALID, "null plan / weights");
    if (int rc = refuse(features(p), F_WEIGHTS)) return rc;
    for (int a = 0; a < 3; ++a)
        if ((uintptr_t)weights[a] % p->esize)
            return fail(DFFT_ERR_INVALID, std::string("weights[") + std::to_string(a) + "] must be aligned to its " + std::to_string(p->esize) + "-byte element");
    // the schedules of unweighted plans may run stages that have no weighted twins
    if (!p->weighted && p->axes_fixed)
        return fail(DFFT_ERR_STATE, "set the weights for the first time before the first exec, dfft_plan_tune or dfft_plan_describe");
    for (int a = 0; a < 3; ++a) p->weights[a] = weights[a];
    p->weighted = true;
    // a step whose pointer turns from null to a table launches another kernel: run each direction eagerly before a capture
    for (auto& dir : p->sched)
        for (Schedule& sc : dir) sc.executed = false;
    return DFFT_SUCCESS;
}
int dfft_plan_get_weights(dfft_plan_t p, const void* weights[3]) {
    if (!p || !weights) return fail(DFFT_ERR_INVALID, "null plan / weights");
    for (int a = 0; a < 3; ++a) weights[a] = p->weights[a];
    return DFFT_SUCCESS;
}

int dfft_plan_get_scale(dfft_plan_t p, double* forward_scale, double* inverse_scale) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (forward_scale) *forward_scale = p->scale[0];
    if (inverse_scale) *inverse_scale = p->scale[1];
    return DFFT_SUCCESS;
}

int dfft_timer_enable(dfft_plan_t p, int enable) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    p->timing = enable != 0;
    return DFFT_SUCCESS;
}
int dfft_get_phase_count(dfft_plan_t p) {
    if (!p) return 0;
    int n = 0;
    for (int k = 1; k < p->n_events_used; ++k)
        if (p->ev_names[k]) ++n;
    return n;
}
const char* dfft_get_phase_name(dfft_plan_t p, int i) {
    if (!p) return nullptr;
    int n = 0;
    for (int k = 1; k < p->n_events_used; ++k)
        if (p->ev_names[k]) {
            if (n == i) return p->ev_names[k];
            ++n;
        }
    return nullptr;
}
int dfft_get_phase_times(dfft_plan_t p, double* ms, int capacity) {
    if (!p || !ms) return fail(DFFT_ERR_INVALID, "null argument");
    if (p->n_events_used < 2) return fail(DFFT_ERR_STATE, "no timed exec yet (dfft_timer_enable)");
    CK_CUDA(cudaEventSynchronize(p->events[p->n_events_used - 1]));
    int n = 0;
    for (int k = 1; k < p->n_events_used; ++k)
        if (p->ev_names[k]) {
            if (n < capacity) {
                float f = 0;
                CK_CUDA(cudaEventElapsedTime(&f, p->events[0], p->events[k]));
                ms[n] = f;
            }
            ++n;
        }
    return n;
}
int dfft_get_last_breakdown(dfft_plan_t p, double* fft_ms, double* exchange_ms, double* total_ms) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (p->n_events_used < 2) return fail(DFFT_ERR_STATE, "no timed exec yet (dfft_timer_enable)");
    CK_CUDA(cudaEventSynchronize(p->events[p->n_events_used - 1]));
    double f = 0, x = 0;
    for (int k = 1; k < p->n_events_used; ++k) {
        float d = 0;
        CK_CUDA(cudaEventElapsedTime(&d, p->events[k - 1], p->events[k]));
        if (p->ev_is_fft[k] == 1) f += d;
        else if (p->ev_is_fft[k] == 0) x += d;
    }
    float tot = 0;
    CK_CUDA(cudaEventElapsedTime(&tot, p->events[0], p->events[p->n_events_used - 1]));
    if (fft_ms) *fft_ms = f;
    if (exchange_ms) *exchange_ms = x;
    if (total_ms) *total_ms = tot;
    return DFFT_SUCCESS;
}
int dfft_get_last_launch_count(dfft_plan_t p) { return p ? p->last_launches : 0; }
int dfft_get_step_count(dfft_plan_t p) { return p && p->n_events_used > 1 ? p->n_events_used - 2 : 0; }
const char* dfft_get_step_label(dfft_plan_t p, int i) {
    if (!p || i < 0 || i + 1 >= p->n_events_used - 1) return nullptr;
    return p->ev_labels[i + 1];
}
int dfft_get_step_times(dfft_plan_t p, double* ms, int capacity) {
    if (!p || !ms) return fail(DFFT_ERR_INVALID, "null argument");
    if (p->n_events_used < 2) return fail(DFFT_ERR_STATE, "no timed exec yet (dfft_timer_enable)");
    CK_CUDA(cudaEventSynchronize(p->events[p->n_events_used - 1]));
    int n = 0;
    for (int k = 1; k < p->n_events_used - 1; ++k, ++n) {
        if (n >= capacity) continue;
        float f = 0;
        CK_CUDA(cudaEventElapsedTime(&f, p->events[k - 1], p->events[k]));
        ms[n] = f;
    }
    return n;
}

// Plan-time measurement of the execution schedule (the role FFTW_MEASURE plays for FFTW plans; the reference leaves
// the choice between its Sync and Streams variants to the user's benchmarks).  Runs the plan's transform on the
// caller's buffers with each candidate — the sequential schedule and overlapped schedules with different numbers of
// CTAs for the exchanging pass — and keeps the fastest one, judged by the slowest rank.  Collective; `out` is
// overwritten; the input is left intact.  Only plans created with send_method Streams have alternatives.
static std::string cand_name(int seq, int ctas, int groups, int chunks) {
    if (seq) return "sequential";
    return "overlapped/" + std::to_string(ctas) + " CTAs/" + std::to_string(groups) + " groups/" + std::to_string(chunks) + " chunks";
}
int dfft_plan_tune(dfft_plan_t p, void* out, const void* in, int inverse, int reps) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (p->comm->dry) return fail(DFFT_ERR_STATE, "geometry-only plan");
    if (!p->work || !out || !in) return fail(DFFT_ERR_INVALID, "plan needs its work area and both buffers");
    if (p->inplace && out != in) return fail(DFFT_ERR_INVALID, "in-place plan: out must equal in");
    CK_CUDA(cudaSetDevice(p->comm->device));
    p->axes_fixed = true;
    const int dir = inverse ? 1 : 0;
    if (reps < 1) reps = 3;
    int sms = 0;
    CK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, p->comm->device));
    // candidates: the sequential schedule, and overlapped schedules over a small grid of (CTAs of the exchanging pass,
    // plane groups of the z pass, z chunks of the y / x passes).  One candidate costs reps + 1 transforms (milliseconds).
    struct Cand { int seq; int ctas; int groups; int chunks; };
    std::vector<Cand> cands;
    cands.push_back({1, 0, 0, 0});
    const bool streams = p->cfg.send_method == DFFT_SEND_STREAMS || (p->g.decomp == DFFT_PENCIL && p->cfg.send_method2 == DFFT_SEND_STREAMS);
    const bool has_overlap = streams && p->P > 1 && p->xchg_ctas >= 0 && alt_schedules(p) &&
                             ((p->g.decomp == DFFT_SLAB_ZY_THEN_X && p->direct2) ||
                              (p->g.decomp == DFFT_PENCIL && p->direct1 && p->direct2 && pencil_overlap_enabled()));
    const bool pencil_inv = inverse && p->g.decomp == DFFT_PENCIL;
    const int groups_default = p->ovl_groups, chunks_default = p->ovl_chunks;
    if (has_overlap) {
        const int cta_list[] = {sms / 3, sms / 2, (2 * sms) / 3, (5 * sms) / 6, sms, 2 * sms};
        for (int c : cta_list) {
            if (pencil_inv) {  // plane groups of the y / z passes; the x pass is not chunked
                for (int g_ : {2, 4, 8}) cands.push_back({0, c, g_, 0});
                continue;
            }
            for (int ch : {4, 8}) {
                if (inverse) cands.push_back({0, c, 1, ch});  // the slab inverse has no plane groups (the exchanging x pass comes first)
                else
                    for (int g_ : {1, 2, 4}) cands.push_back({0, c, g_, ch});
            }
        }
    }
    p->tune_report.clear();
    if (cands.size() == 1) {
        const char* why = sequential_only(p);
        p->tune_report = why           ? std::string("sequential schedule (no alternatives for this plan: ") + why + " run the sequential schedule)"
                         : pow2_axes(p) ? "sequential schedule (no alternatives for this plan)"
                                        : "sequential schedule (no alternatives for this plan: an axis length is not a power of two)";
        return 0;
    }
    const bool was_timing = p->timing;
    auto apply = [&](const Cand& c) {
        p->tuned_seq[dir] = c.seq;
        p->tuned_ctas[dir] = c.seq ? -2 : c.ctas;
        p->tuned_chunks[dir] = c.seq ? 0 : c.chunks;
        if (!inverse) p->ovl_groups = (!c.seq && c.groups > 0) ? c.groups : groups_default;
        else if (pencil_inv) p->tuned_groups_inv = c.seq ? 0 : c.groups;
        p->sched[dir][2] = Schedule();
    };
    // whatever way this function is left: events destroyed, the phase timer back on, and — on an error in the middle of
    // the measurements — the plan back on the sequential schedule
    struct Cleanup {
        std::function<void()> f;
        ~Cleanup() { f(); }
    };
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    bool finished = false;
    Cleanup cleanup{[&] {
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
        p->timing = was_timing;
        if (!finished) apply(cands[0]);
    }};
    CK_CUDA(cudaEventCreate(&e0));
    CK_CUDA(cudaEventCreate(&e1));
    p->timing = false;
    int best = 0;
    double best_ms = 1e30;
    std::string rep;
    for (size_t k = 0; k < cands.size(); ++k) {
        apply(cands[k]);
        Schedule* sc = nullptr;
        int rc = get_schedule(p, inverse, 3, &sc);
        if (rc) continue;  // a candidate this geometry cannot build: skip it (every rank takes the same branch)
        for (int it = 0; it < reps + 1; ++it) {
            if (it == 1) CK_CUDA(cudaEventRecord(e0, p->own_stream));
            rc = run_schedule(p, *sc, out, in, p->own_stream, false, 1);  // batched plans: field 0
            if (rc) return rc;
        }
        CK_CUDA(cudaEventRecord(e1, p->own_stream));
        rc = dfft_plan_wait(p);
        if (rc) return rc;
        float ms = 0;
        CK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
        double mine = ms / reps;
        std::vector<char> all;
        rc = nccl_allgather_bytes(p, &mine, sizeof(double), all);
        if (rc) return rc;
        double worst = 0;
        for (int r = 0; r < p->P; ++r) worst = std::max(worst, reinterpret_cast<const double*>(all.data())[r]);
        rep += (k ? ", " : "") + cand_name(cands[k].seq, cands[k].ctas, cands[k].groups, cands[k].chunks) + " " + std::to_string(worst).substr(0, 6) + " ms";
        if (worst < best_ms) { best_ms = worst; best = int(k); }
    }
    apply(cands[best]);
    finished = true;
    (void)chunks_default;
    p->tune_report = std::string(inverse ? "inverse: " : "forward: ") + rep + " -> " +
                     cand_name(cands[best].seq, cands[best].ctas, cands[best].groups, cands[best].chunks);
    return best;
}
const char* dfft_plan_tune_report(dfft_plan_t p) { return p ? p->tune_report.c_str() : nullptr; }

// Timeline of the last timed exec: step i ran on plan stream `stream[i]` (0 caller's, 1 exchange, 2 follow-up) from
// begin_ms[i] to end_ms[i] after the start of the exec.  The way to look at an overlapped (Streams) schedule.
int dfft_get_timeline(dfft_plan_t p, double* begin_ms, double* end_ms, int* stream, int capacity) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    if (p->n_events_used < 2 || p->tl_used < 2) return fail(DFFT_ERR_STATE, "no timed exec yet (dfft_timer_enable)");
    CK_CUDA(cudaEventSynchronize(p->events[p->n_events_used - 1]));
    const int n = p->tl_used / 2;
    for (int i = 0; i < n && i < capacity; ++i) {
        float a = 0, b = 0;
        CK_CUDA(cudaEventSynchronize(p->tl_events[2 * i + 1]));
        CK_CUDA(cudaEventElapsedTime(&a, p->events[0], p->tl_events[2 * i]));
        CK_CUDA(cudaEventElapsedTime(&b, p->events[0], p->tl_events[2 * i + 1]));
        if (begin_ms) begin_ms[i] = a;
        if (end_ms) end_ms[i] = b;
        if (stream) stream[i] = p->tl_streams[2 * i];
    }
    return n;
}
const char* dfft_get_timeline_label(dfft_plan_t p, int i) {
    if (!p || i < 0 || 2 * i >= p->tl_used) return nullptr;
    return p->tl_labels[2 * i];
}
// JSON description of a schedule (test hook: tests/test_schedule_emulation.py replays it with numpy)
static void json_view(std::string& o, const View& v, const Tables& T) {
    o += "{\"nseg\":" + std::to_string(v.nseg) + ",\"sN\":" + std::to_string(v.sN) + ",\"segs\":[";
    for (int i = 0; i < v.nseg; ++i) {
        const Seg& g = v.seg[i];
        if (i) o += ",";
        o += "{\"base\":" + std::to_string((unsigned long long)g.base) + ",\"sA0\":" + std::to_string(g.sA0) + ",\"sA1\":" + std::to_string(g.sA1) +
             ",\"n0\":" + std::to_string(g.n0) + "}";
    }
    o += "],\"seg_of_n\":[";
    if (v.nseg > 1) {
        auto it = T.host_tabs.find(v.seg_of_n);
        if (it != T.host_tabs.end())
            for (size_t i = 0; i < it->second.size(); ++i) { if (i) o += ","; o += std::to_string(int(it->second[i])); }
    }
    o += "]}";
}
// ,"name":[[lx,ly,lz,hx,hy,hz], ...] of box plans; nothing for a side with the natural layout
static std::string json_boxes(const char* name, const std::vector<Box>& boxes) {
    if (boxes.empty()) return std::string();
    std::string o = std::string(",\"") + name + "\":[";
    for (size_t r = 0; r < boxes.size(); ++r) {
        o += r ? ",[" : "[";
        for (int k = 0; k < 6; ++k) o += (k ? "," : "") + std::to_string(k < 3 ? boxes[r].lo[k] : boxes[r].hi[k - 3]);
        o += "]";
    }
    return o + "]";
}
// ,"name":[field,x,y] of a side with strides (dfft_plan_set_strides); nothing for a dense side
static std::string json_strides(const char* name, bool on, const long long s[3]) {
    if (!on) return std::string();
    return std::string(",\"") + name + "\":[" + std::to_string(s[0]) + "," + std::to_string(s[1]) + "," + std::to_string(s[2]) + "]";
}
int dfft_plan_describe(dfft_plan_t p, int inverse, int d, char* buf, size_t capacity, size_t* needed) {
    if (!p || d < 1 || d > 3) return fail(DFFT_ERR_INVALID, "bad arguments");
    Schedule* scp = nullptr;
    {
        int rc = get_schedule(p, inverse, d, &scp);
        if (rc) return rc;
    }
    Schedule& sc = *scp;
    const bool per_axis = p->g.transform == DFFT_R2HC;
    const bool uniform = p->kinds[0] == p->kinds[1] && p->kinds[1] == p->kinds[2];
    std::string o = "{\"rank\":" + std::to_string(p->rank) + ",\"esize\":" + std::to_string(p->esize) + (p->inplace ? ",\"inplace\":true" : "") +
                    (is_half(p->prec) ? std::string(",\"precision\":\"") + (p->prec == DFFT_F16 ? "f16" : "bf16") + "\"" : std::string()) +
                    // "mixed" when the axes differ; per-axis plans also list the kinds, and each R2R pass its own below
                    (is_r2r(p->g.transform) ? std::string(",\"r2r\":\"") + (uniform ? r2r_name(p->kinds[0]) : "mixed") + "\"" : std::string()) +
                    (per_axis ? std::string(",\"r2r_kinds\":[\"") + r2r_name(p->kinds[0]) + "\",\"" + r2r_name(p->kinds[1]) + "\",\"" +
                                    r2r_name(p->kinds[2]) + "\"]"
                              : std::string()) +
                    (all_axes(p) ? std::string()
                                 : ",\"transform_axes\":[" + std::to_string(p->taxes[0]) + "," + std::to_string(p->taxes[1]) + "," +
                                       std::to_string(p->taxes[2]) + "]") +
                    (p->g.padded() ? ",\"spectral\":[" + std::to_string(p->g.kx) + "," + std::to_string(p->g.ky) + "," + std::to_string(p->g.kz) + "]"
                                   : std::string()) +
                    (p->g.pruned() ? ",\"data\":[" + std::to_string(p->g.mx) + "," + std::to_string(p->g.my) + "," + std::to_string(p->g.mz) + "]"
                                   : std::string()) +
                    (p->comps > 1 ? ",\"components\":" + std::to_string(p->comps) : std::string()) +
                    (p->n1d ? ",\"signal\":" + std::to_string(p->n1d) : std::string()) + (p->oz.size.empty() ? "" : ",\"order\":\"natural\"") +
                    (p->weighted ? ",\"weights\":[" + std::to_string(p->weights[0] ? 1 : 0) + "," + std::to_string(p->weights[1] ? 1 : 0) + "," +
                                       std::to_string(p->weights[2] ? 1 : 0) + "]"
                                 : std::string()) +
                    json_boxes("in_boxes", p->in_boxes) + json_boxes("out_boxes", p->out_boxes) +
                    json_strides("in_strides", p->in_embedded, p->in_strides) + json_strides("out_strides", p->out_embedded, p->out_strides) +
                    (p->batch > 1 ? ",\"batch\":" + std::to_string(p->batch) + ",\"field_in\":" + std::to_string(sc.field_in) +
                                        ",\"field_out\":" + std::to_string(sc.field_out)
                                  : std::string()) +
                    ",\"slot_bytes\":" + std::to_string(p->slot_bytes) +
                    ",\"nslots\":" + std::to_string(p->nslots) + ",\"overlapped\":" + (sc.overlapped ? "true" : "false") + ",\"slots\":[";
    for (int s_ = 0; s_ < p->nslots; ++s_) {
        if (s_) o += ",";
        o += "[";
        for (int r = 0; r < p->P; ++r) { if (r) o += ","; o += std::to_string((unsigned long long)p->slot_ptr[s_][r]); }
        o += "]";
    }
    o += "],\"steps\":[";
    bool first = true;
    std::vector<Step> listed;  // the fused z + y stage is listed as its two phases, in the order they consume data
    for (const Step& s_ : sc.steps) {
        if (s_.kernel != KERNEL_ZY_FUSED) { listed.push_back(s_); continue; }
        Step z = s_, y = s_;
        z.kernel = y.kernel = KERNEL_PASS;
        y.kind = PASS_C2C_TILED;
        y.prm = s_.prm_y;
        y.in_user = s_.y_in_user;
        y.out_user = s_.y_out_user;
        y.final_store = false;
        const bool inv = s_.prm.inverse != 0;
        z.label = inv ? "yz pass: z phase" : "zy pass: z phase";
        y.label = inv ? "yz pass: y phase" : "zy pass: y phase";
        if (inv) { listed.push_back(y); listed.push_back(z); }
        else { listed.push_back(z); listed.push_back(y); }
    }
    // Batched plans: the batched stage is listed as its three single-segment views over all fields (in_user 2: it reads
    // the caller's `out`); a per-field schedule is listed once per field, with the caller's buffers shifted to the field
    // and the field in "field".  Between fields an overlapped schedule joins its streams into the caller's and forks
    // them again: the last step of each stream records an event that the first step of every stream of the next field
    // waits for.
    std::vector<long long> field_of(listed.size(), 0);
    if (sc.whole_batch) {
        std::vector<Step> all;
        for (const Step& s_ : listed) {
            if (s_.kernel != KERNEL_BATCH_SMALL) { all.push_back(s_); continue; }
            const long long N = (long long)p->g.nx, N2 = N * N, N3 = N2 * N, B = (long long)p->batch;
            Step z = s_, y = s_, x = s_;
            z.kernel = y.kernel = x.kernel = KERNEL_PASS;
            z.kind = PASS_C2C_CONTIG; z.label = "batched pass: z lines";
            z.prm.A0 = int(B * N); z.prm.A1 = int(N); z.prm.B = 1;
            z.prm.in = z.prm.out = single_view(nullptr, N2, N, 1);
            y.kind = PASS_C2C_TILED; y.label = "batched pass: y lines";
            y.prm.A0 = int(B * N); y.prm.A1 = 1; y.prm.B = int(N);
            y.prm.in = y.prm.out = single_view(nullptr, N2, 0, N);
            x.kind = PASS_C2C_TILED; x.label = "batched pass: x lines";
            x.prm.A0 = int(B); x.prm.A1 = 1; x.prm.B = int(N2);
            x.prm.in = x.prm.out = single_view(nullptr, N3, 0, N2);
            const bool inv = s_.prm.inverse != 0;
            Step* order[3] = {&z, &y, &x};
            if (inv) std::swap(order[0], order[2]);
            for (int k = 0; k < 3; ++k) {
                order[k]->in_user = k == 0 ? 1 : 2;
                order[k]->out_user = 2;
                order[k]->final_store = k == 2;  // the last axis of phase B
                all.push_back(*order[k]);
            }
        }
        listed.swap(all);
        field_of.assign(listed.size(), -1);
    } else if (p->batch > 1) {
        const size_t per = listed.size();
        std::vector<Step> all;
        field_of.clear();
        int join_ev[3] = {-1, -1, -1};
        for (size_t f = 0; f < p->batch; ++f) {
            bool seen[3] = {false, false, false};
            for (size_t k = 0; k < per; ++k) {
                Step s_ = listed[k];
                if (s_.type == STEP_PASS) {
                    if (s_.in_user) s_.prm.in.seg[0].base = (char*)s_.prm.in.seg[0].base + f * (s_.in_user == 1 ? sc.field_in : sc.field_out);
                    if (s_.out_user == 2) s_.prm.out.seg[0].base = (char*)s_.prm.out.seg[0].base + f * sc.field_out;
                }
                if (sc.overlapped && f > 0 && !seen[s_.stream])
                    for (int e : join_ev) if (e >= 0) s_.waits.push_back(e);
                seen[s_.stream] = true;
                all.push_back(s_);
                field_of.push_back((long long)f);
            }
            if (!sc.overlapped) continue;
            for (int st_ = 0; st_ < 3; ++st_) {
                join_ev[st_] = -1;
                for (size_t k = all.size(); k-- > all.size() - per;) {
                    if (all[k].stream != st_) continue;
                    if (all[k].record < 0) all[k].record = sc.nevents + st_;
                    join_ev[st_] = all[k].record;
                    break;
                }
            }
        }
        listed.swap(all);
    }
    for (size_t i = 0; i < listed.size(); ++i) {
        const Step& s_ = listed[i];
        if (!first) o += ",";
        first = false;
        o += "{\"type\":" + std::to_string(int(s_.type)) + ",\"label\":\"" + s_.label + "\",\"stream\":" + std::to_string(s_.stream) +
             (p->batch > 1 ? ",\"field\":" + std::to_string(field_of[i]) : std::string()) + ",\"record\":" + std::to_string(s_.record) + ",\"waits\":[";
        for (size_t w = 0; w < s_.waits.size(); ++w) o += (w ? "," : "") + std::to_string(s_.waits[w]);
        o += "]";
        if (s_.type == STEP_PASS) {
            // copy passes (kinds 6 / 7): "n" is the length of the kept axis, "log2n" 0, no "r2r"
            const bool copy = is_copy(s_.kind);
            o += ",\"kind\":" + std::to_string(int(s_.kind)) +
                 (per_axis && !copy ? std::string(",\"r2r\":\"") + r2r_name(s_.r2r) + "\"" : std::string()) +
                 ",\"log2n\":" + std::to_string(s_.log2n) +
                 (s_.bluestein() || copy ? ",\"n\":" + std::to_string(s_.n) : std::string()) +
                 (s_.keep ? ",\"keep\":" + std::to_string(s_.keep) : std::string()) +
                 (s_.data ? ",\"data\":" + std::to_string(s_.data) : std::string()) + (s_.weighted ? ",\"weighted\":1,\"axis\":" + std::to_string(s_.axis) : std::string()) +
                 (s_.twiddle ? std::string(",\"twiddle\":\"") + s_.twiddle + "\",\"tw\":[" + std::to_string(s_.tw.line0) + "," +
                                   std::to_string(s_.tw.c1) + "," + std::to_string(s_.tw.mul) + "]"
                             : std::string()) +
                 // the transposing z pass of natural-order 1D plans: its row side's line stride
                 (s_.tw.sB ? ",\"transposed\":" + std::to_string(s_.tw.sB) : std::string()) +
                 ",\"A0\":" + std::to_string(s_.prm.A0) +
                 ",\"A1\":" + std::to_string(s_.prm.A1) + ",\"B\":" + std::to_string(s_.prm.B) + ",\"inverse\":" + std::to_string(s_.prm.inverse) +
                 ",\"in_user\":" + std::to_string(s_.in_user) + ",\"out_user\":" + std::to_string(s_.out_user) + ",\"in\":";
            json_view(o, s_.prm.in, p->tabs);
            o += ",\"out\":";
            json_view(o, s_.prm.out, p->tabs);
            // the scale as the kernels apply it (f32 plans: rounded to float)
            const double scale = p->prec == DFFT_F32 ? double(float(p->scale[sc.inverse])) : p->scale[sc.inverse];
            // 16-bit plans: the pass's share of the scale instead (step_factor), under its own key
            const double factor = is_half(p->prec) ? step_factor(p, sc, s_) : 1.0;
            if (factor != 1.0) {
                char num[40];
                snprintf(num, sizeof num, "%.17g", factor);
                o += std::string(",\"factor\":") + num;
            }
            if (s_.final_store && p->scale[sc.inverse] != 1.0 && !is_half(p->prec)) {
                char num[40];
                snprintf(num, sizeof num, "%.17g", scale);
                o += std::string(",\"scale\":") + num;
            }
        } else if (s_.type == STEP_RENDEZVOUS) {
            o += ",\"group\":" + std::to_string(s_.group) + ",\"phase_id\":" + std::to_string(s_.phase_id) + ",\"members\":[";
            const std::vector<int>& G = p->grp[s_.group];
            for (size_t q = 0; q < G.size(); ++q) o += (q ? "," : "") + std::to_string(G[q]);
            o += "]";
        } else {
            o += ",\"group\":" + std::to_string(s_.group) + ",\"send_slot\":" + std::to_string(s_.send_slot) + ",\"recv_slot\":" + std::to_string(s_.recv_slot) + ",\"peers\":[";
            const std::vector<int>& G = p->grp[s_.group];
            for (size_t q = 0; q < G.size(); ++q) {
                if (q) o += ",";
                o += "{\"rank\":" + std::to_string(G[q]) + ",\"scount\":" + std::to_string(s_.scount[q]) + ",\"soff\":" + std::to_string(s_.soff[q]) +
                     ",\"rcount\":" + std::to_string(s_.rcount[q]) + ",\"roff\":" + std::to_string(s_.roff[q]) + "}";
            }
            o += "]";
        }
        o += "}";
    }
    o += "]}";
    if (needed) *needed = o.size() + 1;
    if (buf && capacity > o.size()) memcpy(buf, o.c_str(), o.size() + 1);
    else if (buf && capacity) buf[0] = 0;
    return DFFT_SUCCESS;
}
int dfft_timer_gather(dfft_plan_t p) {
    if (!p) return fail(DFFT_ERR_INVALID, "null plan");
    return timer_gather(p);
}
const char* dfft_timer_csv_path(dfft_plan_t p) { return p ? p->csv_path.c_str() : nullptr; }

// ---- single-axis building blocks -----------------------------------------------------------------------
// Tables of the single-axis calls: one Tables per (precision, device), process-wide and never freed
static Tables& fft1d_tables(int prec) {
    static std::map<std::pair<int, int>, Tables> tabs;
    int dev = 0;
    cudaGetDevice(&dev);
    Tables& T = tabs[std::make_pair(prec, dev)];
    T.prec = prec;
    return T;
}

// one pass of n-point lines over prm's views (R2C / C2R: n complex points), with the tables of its length; r2r: the kind of
// R2R passes
static int fft1d_pass(int prec, PassKind kind, size_t n, FftParams prm, void* stream, int r2r_k = DFFT_DCT) {
    void *tw = nullptr, *tw2 = nullptr, *table = nullptr;
    const int rc = pass_tables(fft1d_tables(prec), kind, n, r2r_k, &tw, &tw2, &table);
    if (rc) return rc;
    prm.tw = tw; prm.tw2 = tw2;
    cudaError_t e = launch_fft_pass(prec, kind, n, prm, table, 1.0, (cudaStream_t)stream, r2r_k);
    if (e != cudaSuccess) return fail(DFFT_ERR_CUDA, std::string("launch failed: ") + cudaGetErrorString(e));
    return DFFT_SUCCESS;
}

int dfft_fft1d_contig(int precision, int kind, int direction, size_t n, size_t lines, void* out, size_t out_pitch, const void* in,
                      size_t in_pitch, void* stream) {
    if (precision < DFFT_F32 || precision > DFFT_BF16) return fail(DFFT_ERR_INVALID, "bad precision");
    if (is_half(precision) && kind == 0 && !pow2_length(n)) return fail(DFFT_ERR_UNSUPPORTED, "16-bit storage takes power-of-two lengths only");
    if (kind < 0 || kind > 2) return fail(DFFT_ERR_INVALID, "bad kind");
    const size_t len = kind == 0 ? n : n / 2;
    const int l2 = ilog2_exact(len);
    if (kind == 0 ? !c2c_length(n) : (ilog2_exact(n) < 1 || l2 < 1 || l2 > MAX_LOG2N)) return fail(DFFT_ERR_UNSUPPORTED, "length must be a power of two");
    FftParams prm{};
    prm.A0 = 1; prm.A1 = int(lines); prm.B = 1;
    prm.inverse = (kind == 0 && direction > 0) ? 1 : 0;
    // pitches are in elements of the respective array (reals for real arrays); views are in complex units
    long long ip = (long long)in_pitch, op = (long long)out_pitch;
    if (kind == 1) { if (in_pitch & 1) return fail(DFFT_ERR_INVALID, "real pitch must be even"); ip /= 2; }
    if (kind == 2) { if (out_pitch & 1) return fail(DFFT_ERR_INVALID, "real pitch must be even"); op /= 2; }
    prm.in = single_view(const_cast<void*>(in), 0, ip, 1);
    prm.out = single_view(out, 0, op, 1);
    return fft1d_pass(precision, kind == 0 ? PASS_C2C_CONTIG : (kind == 1 ? PASS_R2C : PASS_C2R), len, prm, stream);
}

int dfft_fft1d_strided(int precision, int direction, size_t a, size_t n, size_t b, void* out, const void* in, void* stream) {
    if (precision < DFFT_F32 || precision > DFFT_BF16) return fail(DFFT_ERR_INVALID, "bad precision");
    if (is_half(precision) && !pow2_length(n)) return fail(DFFT_ERR_UNSUPPORTED, "16-bit storage takes power-of-two lengths only");
    if (!c2c_length(n)) return fail(DFFT_ERR_UNSUPPORTED, "length must be a power of two in [2, 8192] or any length in [3, 4096]");
    FftParams prm{};
    prm.A0 = int(a); prm.A1 = 1; prm.B = int(b);
    prm.inverse = direction > 0 ? 1 : 0;
    prm.in = single_view(const_cast<void*>(in), (long long)(n * b), 0, (long long)b);
    prm.out = single_view(out, (long long)(n * b), 0, (long long)b);
    return fft1d_pass(precision, PASS_C2C_TILED, n, prm, stream);
}

int dfft_fft1d_r2r(int precision, int transform, int direction, size_t n, size_t a, size_t b, void* out, const void* in, void* stream) {
    if (is_half(precision)) return refuse_half("real-to-real transforms");
    if (precision != DFFT_F32 && precision != DFFT_F64) return fail(DFFT_ERR_INVALID, "bad precision");
    if (!is_r2r_kind(transform))
        return fail(DFFT_ERR_INVALID, "transform must be DFFT_DCT, DFFT_DST, DFFT_R2HC, DFFT_DCT1, DFFT_DST1, DFFT_DCT4 or DFFT_DST4");
    if (!r2r_kind_length(transform, n))
        return fail(DFFT_ERR_UNSUPPORTED, transform == DFFT_DCT1   ? "DCT-I length must be 2^k + 1 in [3, 8193]"
                                          : transform == DFFT_DST1 ? "DST-I length must be 2^k - 1 in [3, 8191]"
                                          : is_type4(transform)    ? "DCT-IV / DST-IV length must be a power of two in [4, 8192]"
                                                                   : "length must be a power of two in [2, 8192]");
    if (a == 0 || b == 0) return DFFT_SUCCESS;
    if (a * b > size_t(0x7fffffff) || n * b > size_t(1) << 62) return fail(DFFT_ERR_INVALID, "array too large");
    FftParams prm{};
    prm.inverse = direction > 0 ? 1 : 0;
    if (b == 1) {  // CONTIG: a lines of n reals
        prm.A0 = 1; prm.A1 = int(a); prm.B = 1;
        prm.in = single_view(const_cast<void*>(in), 0, (long long)n, 1);
        prm.out = single_view(out, 0, (long long)n, 1);
    } else {       // TILED: [a][n][b], b contiguous
        prm.A0 = int(a); prm.A1 = 1; prm.B = int(b);
        prm.in = single_view(const_cast<void*>(in), (long long)(n * b), 0, (long long)b);
        prm.out = single_view(out, (long long)(n * b), 0, (long long)b);
    }
    return fft1d_pass(precision, b == 1 ? PASS_R2R_CONTIG : PASS_R2R_TILED, n, prm, stream, transform);
}

int dfft_fft1d_general(int precision, int direction, size_t n, size_t a0, size_t a1, size_t b, void* out, const long long out_strides[3],
                       const void* in, const long long in_strides[3], void* stream) {
    if (precision < DFFT_F32 || precision > DFFT_BF16) return fail(DFFT_ERR_INVALID, "bad precision");
    if (is_half(precision) && !pow2_length(n)) return fail(DFFT_ERR_UNSUPPORTED, "16-bit storage takes power-of-two lengths only");
    if (!c2c_length(n)) return fail(DFFT_ERR_UNSUPPORTED, "length must be a power of two in [2, 8192] or any length in [3, 4096]");
    FftParams prm{};
    prm.A0 = int(a0); prm.A1 = int(a1); prm.B = int(b);
    prm.inverse = direction > 0 ? 1 : 0;
    prm.in = single_view(const_cast<void*>(in), in_strides[0], in_strides[1], in_strides[2]);
    prm.out = single_view(out, out_strides[0], out_strides[1], out_strides[2]);
    return fft1d_pass(precision, PASS_C2C_TILED, n, prm, stream);
}

// One pass step of a geometry-only plan on the current device, for replaying every rank's schedule on one GPU.  Slot
// addresses ((r+1) << 44) + off become work[r] + off, the caller's views are offsets into in / out as in an exec.  Every
// segment's element range is checked against the buffer it lands in before anything is launched.
int dfft_debug_run_step(dfft_plan_t p, int inverse, int d, size_t field, int step, void* const* work, size_t work_bytes, void* out,
                        size_t out_bytes, const void* in, size_t in_bytes, void* stream) {
    if (!p || d < 1 || d > 3 || !work) return fail(DFFT_ERR_INVALID, "bad arguments");
    if (!p->comm->dry) return fail(DFFT_ERR_STATE, "only geometry-only plans (dfft_comm_create_dry) run single steps");
    Schedule* scp = nullptr;
    {
        int rc = get_schedule(p, inverse, d, &scp);
        if (rc) return rc;
    }
    const Schedule& sc = *scp;
    if (step < 0 || size_t(step) >= sc.steps.size() || field >= (sc.whole_batch ? 1 : p->batch)) return fail(DFFT_ERR_INVALID, "no such step or field");
    Step s = sc.steps[size_t(step)];
    if (s.type != STEP_PASS || s.kernel != KERNEL_PASS) return fail(DFFT_ERR_UNSUPPORTED, "only single pass steps run on their own");
    const size_t len = s.n ? s.n : size_t(1) << s.log2n;  // points per line (R2C / C2R: complex points of the real side)
    if (!is_copy(s.kind)) {
        void *tw = nullptr, *tw2 = nullptr, *blu = nullptr;
        const int rc = pass_tables(fft1d_tables(p->prec), s.kind, len, s.r2r, &tw, &tw2, &blu);
        if (rc) return rc;
        s.prm.tw = tw;
        s.prm.tw2 = tw2;
        s.blu = blu;
        if (s.twiddle && fft1d_tables(p->prec).get_tw1d(s.tw.log2n, const_cast<void**>(&s.tw.table)) != cudaSuccess)
            return fail(DFFT_ERR_CUDA, "twiddle table allocation failed");
    }
    // the views as the kernel sees them: slot addresses on the work areas, the caller's on in / out; each segment's range
    struct Range { const char *lo, *hi, *buf; size_t bytes; };
    std::vector<Range> ranges;
    std::vector<std::pair<View*, const std::vector<unsigned char>*>> tables;
    // bytes per view element: reals on the real side of the R2C / C2R pass of interleaved plans
    auto resolve = [&](View& v, int user, size_t n_len, View& launched, size_t ebytes) -> int {
        if (v.nseg < 1 || v.nseg > MAXSEG || (user && v.nseg != 1)) return fail(DFFT_ERR_STATE, "internal: view segments");
        const std::vector<unsigned char>* tab = nullptr;
        if (v.nseg > 1) {
            auto it = p->tabs.host_tabs.find(v.seg_of_n);
            if (it == p->tabs.host_tabs.end() || it->second.size() < n_len) return fail(DFFT_ERR_STATE, "internal: segment table");
            tab = &it->second;
            tables.emplace_back(&launched, tab);
        }
        launched = v;
        if (user) user_view(launched, user, sc, field, out, in);
        for (int g = 0; g < v.nseg; ++g) {
            Seg& sg = launched.seg[g];
            const char* buf = user == 1 ? static_cast<const char*>(in) : static_cast<const char*>(out);
            size_t bytes = user == 1 ? in_bytes : out_bytes;
            if (!user) {
                const unsigned long long a = (unsigned long long)v.seg[g].base, r = (a >> 44) - 1;
                if ((a >> 44) == 0 || r >= (unsigned long long)p->P || !work[r]) return fail(DFFT_ERR_INVALID, "a view lies in no rank's work area");
                buf = static_cast<const char*>(work[r]);
                bytes = work_bytes;
                sg.base = const_cast<char*>(buf) + (a & ((1ull << 44) - 1));
            }
            // n of this segment, then the lowest and highest element offset over (a0, a1, n, b)
            long long n_lo = -1, n_hi = -1;
            for (size_t n = 0; n < n_len; ++n)
                if (v.nseg == 1 || (*tab)[n] == g) { if (n_lo < 0) n_lo = (long long)n; n_hi = (long long)n; }
            if (n_lo < 0 || s.prm.A0 <= 0 || s.prm.A1 <= 0 || s.prm.B <= 0) continue;  // the segment holds no element
            // b is contiguous, except on the row side of the transposing z pass of natural-order 1D plans (lines tw.sB apart)
            const bool row = s.tw.sB && &v == (s.prm.inverse ? &s.prm.out : &s.prm.in);
            long long lo = 0, hi = (long long)(s.prm.B - 1) * (row ? s.tw.sB : 1);
            for (const long long t : {(long long)(s.prm.A0 - 1) * sg.sA0, (long long)(s.prm.A1 - 1) * sg.sA1}) { lo += std::min(0ll, t); hi += std::max(0ll, t); }
            const long long t0 = (n_lo - sg.n0) * v.sN, t1 = (n_hi - sg.n0) * v.sN;
            lo += std::min(t0, t1);
            hi += std::max(t0, t1);
            const char* b = static_cast<const char*>(sg.base);
            ranges.push_back({b + lo * (long long)ebytes, b + (hi + 1) * (long long)ebytes, buf, bytes});
        }
        return DFFT_SUCCESS;
    };
    // points along n of each view: padded passes hold `keep` on their spectral side and pruned passes `data` on their
    // physical side (the interleaved R2C / C2R pass: Nz reals, Nz / 2 + 1 complex points)
    size_t in_len = 0, out_len = 0;
    s.view_lens(&in_len, &out_len);
    if (s.kind == PASS_R2C_ILV) out_len = len / 2 + 1;
    if (s.kind == PASS_C2R_ILV) in_len = len / 2 + 1;
    const size_t es = p->esize;
    Step t = s;  // the step with resolved views: its user flags are cleared, so run_pass_step leaves them as they are
    t.in_user = t.out_user = 0;
    int rc = resolve(s.prm.in, s.in_user, in_len, t.prm.in, s.kind == PASS_R2C_ILV ? es / 2 : es);
    if (!rc) rc = resolve(s.prm.out, s.out_user, out_len, t.prm.out, s.kind == PASS_C2R_ILV ? es / 2 : es);
    if (rc) return rc;
    for (const Range& r : ranges)
        if (!r.buf || r.lo < r.buf || r.hi > r.buf + r.bytes)
            return fail(DFFT_ERR_INVALID, "a view reaches outside the buffer it lies in");
    // segment tables of multi-segment views: uploaded for this call
    std::vector<void*> dev;
    auto release = [&]() { for (void* q : dev) cudaFree(q); };
    for (auto& vt : tables) {
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, vt.second->size());
        if (e == cudaSuccess) dev.push_back(q);
        if (e == cudaSuccess) e = cudaMemcpy(q, vt.second->data(), vt.second->size(), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) { release(); return fail(DFFT_ERR_CUDA, std::string("segment table upload: ") + cudaGetErrorString(e)); }
        vt.first->seg_of_n = static_cast<const unsigned char*>(q);
    }
    bool launched = false;
    cudaError_t e = run_pass_step(p, sc, t, field, out, in, (cudaStream_t)stream, &launched);
    if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
    release();
    if (e != cudaSuccess) return fail(DFFT_ERR_CUDA, std::string("pass step: ") + cudaGetErrorString(e));
    return DFFT_SUCCESS;
}

}  // extern "C"
