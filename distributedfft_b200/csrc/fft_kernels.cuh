// fft_kernels.cuh — sm_90a batched 1D FFT kernels over "segmented strided views".
//
// One launch = one axis pass of the distributed 3D transform, i.e. one cufftExec* of the reference
// (/root/reference/src/slab/default/mpicufft_slab.cpp:788,806,847,856;
//  /root/reference/src/pencil/mpicufft_pencil.cpp:1662,1695-1698,1723) fused with the pack / unpack
// copies around it (mpicufft_slab.cpp:646-655,691-695; mpicufft_pencil.cpp:873-927,1507-1538): the
// store side of a pass can scatter along the transformed axis into up to MAXSEG destination segments
// (local send slots or peer-mapped receive buffers on other GPUs), the load side can gather likewise.
//
// Two thread mappings:
//   CONTIG — the transformed axis is contiguous in memory (z passes, R2C/C2R).  TB lines per CTA;
//            consecutive threads walk along the line, so global accesses are coalesced over n.
//   TILED  — the transformed axis is strided (y and x passes).  A CTA owns an N x TB tile with TB
//            consecutive elements of the contiguous dimension b; consecutive threads walk along b, so
//            every global access is a TB*sizeof(complex) byte run.
// Both stage through shared memory between radix stages only; first-stage loads and last-stage stores
// go registers <-> HBM directly (one read + one write of the array per pass = the algorithmic minimum).
//
// Instruction diet (the kernels are close to issue-bound in fp64): direction is a template parameter,
// single-segment views use one base pointer plus immediate / incremental offsets, multi-segment views
// read a per-line table of segment bases from shared memory, and shared-memory indices are a
// per-thread base plus compile-time constants (SmemLayout in fft_core.cuh).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <type_traits>

#include "fft_core.cuh"
#include "r2r.hpp"
#include "zy_order.hpp"

namespace dfft {

constexpr int MAXSEG = 16;

struct Seg {
    void* base;     // element pointer (complex elements of the pass' precision)
    long long sA0;  // stride of batch index a0 (elements)
    long long sA1;  // stride of batch index a1
    int n0;         // first n covered by this segment
    int pad_;
};

// element (a0, a1, n, b) of segment s lives at  seg[s].base + a0*sA0 + a1*sA1 + (n - n0)*sN + b
struct View {
    const unsigned char* seg_of_n;  // n -> segment id (device memory); ignored when nseg == 1
    long long sN;                   // stride along the transformed axis (same for every segment)
    int nseg;
    int pad_;
    Seg seg[MAXSEG];
};

struct FftParams {
    View in, out;
    int A0, A1;       // batch extents: line id = a0*A1 + a1
    int B;            // TILED: extent of the contiguous dimension; CONTIG: 1
    int inverse;      // 0 forward (e^-), 1 inverse (e^+), both unnormalised like cuFFT
    const void* tw;   // exp(-2*pi*i*m/N), m < N, N = pass length (complex length for R2C/C2R)
    const void* tw2;  // R2C/C2R only: exp(-2*pi*i*k/(2N)), k <= N/2
    int max_ctas;     // > 0: run as a persistent kernel on at most this many CTAs (SM partitioning for the
                      // overlapped schedule: the exchange pass keeps a few SMs, the local passes the rest)
    int tile_pref;    // TILED: 0 automatic, 1 narrow tiles, 2 wide tiles
    int bulk_out;     // TILED, TMA-fed kernel, experiment (DFFT_BULK_STORE=1): store each destination's rows with one
                      // cp.async.bulk from shared memory instead of 16-byte stores from registers
    int tile_swz;     // TILED: log2 G of the tile-order blocking: G x G tiles of (a0, a1) are numbered consecutively, so
                      // that CTAs running at the same time touch neighbouring rows on BOTH sides of a transposing pass
                      // (0 = plain order: b tiles fastest, then a1, then a0)
};

// Output scale (dfft_plan_set_scale).  Every kernel that stores final values has a scaled twin (template flag SCALED)
// that takes FftScaled in place of FftParams and multiplies each finished value by the scale right before its store.
// The unscaled instantiations keep their parameters and code exactly; the twin is launched only for a scale != 1.
struct FftScaled : FftParams {
    double scale;  // rounded to the kernel's precision once (f32: float(scale))
};
template <bool SCALED>
using KParams = std::conditional_t<SCALED, FftScaled, FftParams>;

// PASS_R2R_*: the view mapping of PASS_C2C_* over real elements (fft_r2r_kernel).  PASS_COPY_*: the views of a C2C or R2R
// pass over an axis the plan keeps, moved without a transform (fft_copy_kernel)
// PASS_C2C_ILV: the z pass of an interleaved plan (dfft_plan_create_interleaved), the view mapping of PASS_C2C_TILED with
// b = the component (B = C, sN = C): fft_c2c_ilv_kernel, or the TILED kernel once C fills its tile.  PASS_R2C_ILV /
// PASS_C2R_ILV: its R2C / C2R z pass of Nz-point lines, one per component (fft_rc_ilv_kernel), the real side counted in reals
enum PassKind {
    PASS_C2C_CONTIG = 0, PASS_C2C_TILED = 1, PASS_R2C = 2, PASS_C2R = 3, PASS_R2R_CONTIG = 4, PASS_R2R_TILED = 5,
    PASS_COPY_CONTIG = 6, PASS_COPY_TILED = 7, PASS_C2C_ILV = 8, PASS_R2C_ILV = 9, PASS_C2R_ILV = 10
};

// ---- tile shape choices (compile time) -----------------------------------------------------------
template <typename T, int LOG2N>
struct Shape {
    // points per thread: 2^LOG2E_MAX (experiment knobs DFFT_LOG2E_F64 / DFFT_LOG2E_F32; 16 points = radix-16
    // butterflies and ~120 registers in f64, 8 points = radix-8 and <= 64 registers, i.e. twice the resident warps)
#ifndef DFFT_LOG2E_F64
#define DFFT_LOG2E_F64 4
#endif
#ifndef DFFT_LOG2E_F32
#define DFFT_LOG2E_F32 4
#endif
    static constexpr int LOG2E_MAX = sizeof(T) == 8 ? DFFT_LOG2E_F64 : DFFT_LOG2E_F32;
    static constexpr int LOG2E = LOG2N < LOG2E_MAX ? LOG2N : LOG2E_MAX;
    static constexpr int N = 1 << LOG2N;
    static constexpr int TPL = N >> LOG2E;
    // CONTIG: lines per CTA.  f64 lines of >= 512 points use 128-thread CTAs (four CTAs per SM interleave their
    // load / compute / store phases), short lines and f32 256 threads (tools/axis_bench.py compares the
    // alternatives).  -DDFFT_CONTIG_THREADS=<n> overrides for experiments.
#ifdef DFFT_CONTIG_THREADS
    static constexpr int CT = DFFT_CONTIG_THREADS;
#else
    static constexpr int CT = (sizeof(T) == 8 && LOG2N >= 9) ? 128 : 256;
#endif
    static constexpr int TBC = (CT / TPL) < 1 ? 1 : ((CT / TPL) > 64 ? 64 : (CT / TPL));
    // TILED: tile width; rows of >= DFFT_MINROW_BYTES where shared memory allows, DFFT_TILE_POINTS_F64 / _F32
    // points per tile (experiment knobs)
#ifndef DFFT_MINROW_BYTES
#define DFFT_MINROW_BYTES 64
#endif
#ifndef DFFT_TILE_POINTS_F64
#define DFFT_TILE_POINTS_F64 4096
#endif
#ifndef DFFT_TILE_POINTS_F32
#define DFFT_TILE_POINTS_F32 4096
#endif
    static constexpr int MINROW = DFFT_MINROW_BYTES / int(2 * sizeof(T));
    static constexpr int WANT = (sizeof(T) == 8 ? DFFT_TILE_POINTS_F64 : DFFT_TILE_POINTS_F32) / N;
    static constexpr int TBT_ = WANT < MINROW ? MINROW : (WANT > 32 ? 32 : WANT);
    // keep the tile within 128 KB of shared memory and 1024 threads
    static constexpr int CAP1 = (128 * 1024) / (N * int(2 * sizeof(T)));
    static constexpr int CAP2 = 1024 / TPL;
    static constexpr int CAP = CAP1 < CAP2 ? CAP1 : CAP2;
    static constexpr int TBT = TBT_ > CAP ? (CAP < 1 ? 1 : CAP) : TBT_;
    // experimental wider tile (DFFT_WIDE_TILES=1): double width if it still fits 128 KB / 1024 threads
    static constexpr int TBT_WIDE = (2 * TBT <= CAP && 2 * TBT <= 32) ? 2 * TBT : TBT;
};

// Resident CTAs per SM the register allocator must leave room for: 128 registers per thread for f64 and 64 for
// f32 (16 points per thread) — without it the grid-stride version of the f32 kernels drifted to 90+ registers and
// lost its second CTA per SM.
template <typename T, int LOG2E = 4>
constexpr int min_ctas_per_sm(int threads) {
    constexpr int regs = (sizeof(T) == 8 ? 128 : 64) >> (LOG2E >= 4 ? 0 : 1);  // 8 points per thread: half the budget
    return (65536 / (threads * regs)) < 1 ? 1 : (65536 / (threads * regs));
}

template <typename T>
__device__ __forceinline__ cx<T> ld_elem(const cx<T>* p) {
    if constexpr (sizeof(T) == 8) {
        double2 r = *reinterpret_cast<const double2*>(p);
        return cx<T>{r.x, r.y};
    } else {
        float2 r = *reinterpret_cast<const float2*>(p);
        return cx<T>{r.x, r.y};
    }
}
template <typename T>
__device__ __forceinline__ void st_elem(cx<T>* p, cx<T> v) {
    if constexpr (sizeof(T) == 8) *reinterpret_cast<double2*>(p) = make_double2(v.x, v.y);
    else *reinterpret_cast<float2*>(p) = make_float2(v.x, v.y);
}

// 16-bit storage (DFFT_F16 / DFFT_BF16): a complex value is a pair of IEEE binary16 (H = __half) or bfloat16 (H =
// __nv_bfloat16) numbers, 4 bytes.  The passes compute in f32: a load widens the pair to float exactly, a store rounds the
// finished float pair once, to nearest even.
template <typename H>
struct alignas(4) cx16 {
    H x, y;
};
template <typename T, typename H>
__device__ __forceinline__ cx<T> ld_elem(const cx16<H>* p) {
    static_assert(sizeof(T) == 4, "16-bit storage computes in f32");
    float2 f;
    if constexpr (std::is_same_v<H, __half>) f = __half22float2(*reinterpret_cast<const __half2*>(p));
    else f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
    return cx<T>{f.x, f.y};
}
template <typename T, typename H>
__device__ __forceinline__ void st_elem(cx16<H>* p, cx<T> v) {
    static_assert(sizeof(T) == 4, "16-bit storage computes in f32");
    if constexpr (std::is_same_v<H, __half>) *reinterpret_cast<__half2*>(p) = __float22half2_rn(make_float2(v.x, v.y));
    else *reinterpret_cast<__nv_bfloat162*>(p) = __float22bfloat162_rn(make_float2(v.x, v.y));
}

// ---- per-thread access to one line of a view ----------------------------------------------------------
// LINES = lines per CTA that need their own segment table (TB for CONTIG, 1 for TILED).  EL: the element the view counts in
// (complex, or T for the real views of R2R passes).
template <typename T, int LINES, typename EL = cx<T>>
struct LineAccess {
    static constexpr int TABLE_ELEMS = LINES * MAXSEG;  // unsigned long long entries in shared memory
    const View& v;
    EL* p0;                     // single segment: element n = 0 of this thread's line (b included)
    const unsigned long long* tab;  // multi segment: tab[s] = address of element n = 0 of segment s (b excluded)
    long long boff;             // multi segment: + b (elements)
    bool multi;

    // fills the shared-memory table (all threads of the CTA call this; a __syncthreads follows outside)
    static __device__ __forceinline__ void fill_table(const View& v, unsigned long long* table, int line_in_cta, int lane_in_line,
                                                      int lanes_per_line, int a0, int a1) {
        if (v.nseg <= 1) return;
        for (int s = lane_in_line; s < v.nseg; s += lanes_per_line) {
            const Seg& g = v.seg[s];
            EL* p = reinterpret_cast<EL*>(g.base) + (a0 * g.sA0 + a1 * g.sA1 - (long long)g.n0 * v.sN);
            table[line_in_cta * MAXSEG + s] = reinterpret_cast<unsigned long long>(p);
        }
    }
    __device__ __forceinline__ LineAccess(const View& v_, const unsigned long long* table, int line_in_cta, int a0, int a1, int b)
        : v(v_) {
        multi = v.nseg > 1;
        const Seg& g = v.seg[0];
        p0 = reinterpret_cast<EL*>(g.base) + (a0 * g.sA0 + a1 * g.sA1 - (long long)g.n0 * v.sN + b);
        tab = table + line_in_cta * MAXSEG;
        boff = b;
    }
    __device__ __forceinline__ EL* at(int n) const {
        if (!multi) return p0 + (long long)n * v.sN;
        const int s = v.seg_of_n[n];
        return reinterpret_cast<EL*>(tab[s]) + ((long long)n * v.sN + boff);
    }
    // unit stride along n (every CONTIG view): no multiply
    __device__ __forceinline__ EL* at1(int n) const {
        if (!multi) return p0 + n;
        const int s = v.seg_of_n[n];
        return reinterpret_cast<EL*>(tab[s]) + (n + boff);
    }
};

// ---- the in-CTA transform ---------------------------------------------------------------------------
struct NoGatherHook {
    template <int ST>
    __device__ __forceinline__ void operator()(std::integral_constant<int, ST>) const {}
};

template <typename T, int LOG2N, int LOG2E, int TB, bool TILED>
struct CtaFft {
    using Core = FftCore<T, LOG2N, LOG2E>;
    using L = SmemLayout<LOG2N, LOG2E, TB, TILED, int(sizeof(cx<T>))>;
    static constexpr int N = Core::N, E = Core::E, TPL = Core::TPL, NST = Core::NST;
    static constexpr int THREADS = TPL * TB;
    static constexpr int LINES = TILED ? 1 : TB;
    static constexpr size_t TILE_BYTES = size_t(L::ELEMS) * sizeof(cx<T>);
    static constexpr size_t TABLE_BYTES = size_t(2) * LINES * MAXSEG * sizeof(unsigned long long) + 16;  // + one mbarrier (TMA-fed kernel)
    static constexpr size_t SMEM_BYTES = TILE_BYTES + TABLE_BYTES;
    static_assert(THREADS >= 1 && THREADS <= 1024, "CTA size out of range");
    static_assert(SMEM_BYTES <= 227 * 1024, "tile does not fit the 227 KB of shared memory a CTA can use on sm_90a");

    static __device__ __forceinline__ int sidx(int n, int t) { return L::idx(n, t); }

    // synchronise the threads that cooperate on one line (CONTIG) or the whole tile (TILED)
    static __device__ __forceinline__ void sync(int t) {
        if constexpr (TILED || TB == 1) {
            __syncthreads();
        } else if constexpr (TPL <= 32) {
            __syncwarp();
        } else if constexpr (TB <= 15) {
            asm volatile("bar.sync %0, %1;" ::"r"(t + 1), "n"(TPL) : "memory");
        } else {
            __syncthreads();
        }
    }

    // gather: v[e] = tile[j + e*TPL]
    static __device__ __forceinline__ void gather(cx<T> (&v)[E], const cx<T>* sm, int j, int t) {
        if constexpr (L::GATHER_SPLIT) {
            const cx<T>* p = sm + L::idx(j, t);
#pragma unroll
            for (int e = 0; e < E; ++e) v[e] = p[L::off(e * TPL)];
        } else {
#pragma unroll
            for (int e = 0; e < E; ++e) v[e] = sm[L::idx(j + e * TPL, t)];
        }
    }

    // after_gather(std::integral_constant<int, ST>): called by every thread once the gather that follows stage ST has left
    // shared memory; after ST = NST - 2 the buffer is free for this thread (the caller synchronises the CTA before it
    // reuses it)
    template <int ST, typename Hook = NoGatherHook>
    static __device__ __forceinline__ void stages(cx<T> (&v)[E], int j, int t, cx<T>* sm, const cx<T>* tw, const Hook& after_gather = {}) {
        Core::template stage_compute<ST>(v, j, tw);
        if constexpr (ST + 1 < NST) {
            if constexpr (ST > 0) sync(t);
            cx<T>* p = sm + L::idx(Core::template scatter_base<ST>(j), t);
#pragma unroll
            for (int e = 0; e < E; ++e) p[L::off(Core::template scatter_off<ST>(e))] = v[e];
            sync(t);
            gather(v, sm, j, t);
            after_gather(std::integral_constant<int, ST>{});
            stages<ST + 1>(v, j, t, sm, tw, after_gather);
        }
    }
};

// linear (a0, a1) tile number -> (a1, a0): plain order (a1 fastest), or G x G blocks of (a0, a1) numbered consecutively
// when p.tile_swz = log2 G > 0
__device__ __forceinline__ void tile_order(const FftParams& p, int a, int& a1, int& a0) {
    if (p.tile_swz > 0) {
        const int lg = p.tile_swz, G = 1 << lg;
        const int lo = a & (G * G - 1), hi = a >> (2 * lg);
        const int w1 = p.A1 >> lg;  // A0, A1 are multiples of G (checked by the launcher)
        a1 = ((hi % w1) << lg) + (lo & (G - 1));
        a0 = ((hi / w1) << lg) + (lo >> lg);
    } else {
        a1 = a % p.A1;
        a0 = a / p.A1;
    }
}

// linear tile number -> (b tile, a1, a0) of a TILED pass
template <int TB>
__device__ __forceinline__ void tiled_decode(const FftParams& p, long long tile, int& bt, int& a1, int& a0) {
    const int nbt = (p.B + TB - 1) / TB;
    bt = int(tile % nbt);
    tile_order(p, int(tile / nbt), a1, a0);
}

// common prologue: thread -> (j, t), tile -> (a0, a1, b), segment tables.  ILV (CONTIG mapping only): the lines are the
// (a0, a1, b) triples with b fastest — the B interleaved components of a row are neighbouring lines of one CTA
template <typename C, bool TILED, int TB, bool ILV = false>
struct TileCoord {
    int j, t, a0, a1, b;
    bool valid;
    __device__ __forceinline__ TileCoord(const FftParams& p, long long tile = blockIdx.x) {
        const int tid = threadIdx.x;
        if constexpr (TILED) { t = tid % TB; j = tid / TB; }
        else { j = tid % C::TPL; t = tid / C::TPL; }
        if constexpr (TILED) {
            int bt;
            tiled_decode<TB>(p, tile, bt, a1, a0);
            b = bt * TB + t;
            valid = b < p.B;
        } else if constexpr (ILV) {
            const long long line = tile * TB + t;
            valid = line < (long long)p.A0 * p.A1 * p.B;
            b = int(line % p.B);
            const long long row = line / p.B;
            a1 = int(row % p.A1);
            a0 = int(row / p.A1);
        } else {
            const long long line = tile * TB + t;
            valid = line < (long long)p.A0 * p.A1;
            a1 = int(line % p.A1);
            a0 = int(line / p.A1);
            b = 0;
        }
    }
    static __device__ __forceinline__ long long num_tiles(const FftParams& p) {
        if constexpr (TILED) return (long long)p.A0 * p.A1 * ((p.B + TB - 1) / TB);
        else if constexpr (ILV) return ((long long)p.A0 * p.A1 * p.B + TB - 1) / TB;
        else return ((long long)p.A0 * p.A1 + TB - 1) / TB;
    }
};

// ---- global-memory access of a C2C tile ------------------------------------------------------------------
// MemPlain: default caching, what every standalone pass uses.  MemHint: per-instruction L2 eviction priorities
// (createpolicy.fractional policies), used by the fused z/y kernel to keep its intermediate in the L2.
// S: the stored element (cx<T>, or cx16<H> for 16-bit storage with T = float).
template <typename T, typename S = cx<T>>
struct MemPlain {
    using Stored = S;
    __device__ __forceinline__ cx<T> ld(const S* p) const { return ld_elem<T>(p); }
    __device__ __forceinline__ void st(S* p, cx<T> v) const { st_elem<T>(p, v); }
};
// the element a memory policy loads and stores: M::Stored where the policy names one, cx<T> otherwise
template <typename T, typename M, typename = void>
struct StoredOf {
    using type = cx<T>;
};
template <typename T, typename M>
struct StoredOf<T, M, std::void_t<typename M::Stored>> {
    using type = typename M::Stored;
};

__device__ __forceinline__ unsigned long long l2_evict_first() {
    unsigned long long pol;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ unsigned long long l2_evict_last() {
    unsigned long long pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ unsigned long long l2_evict_normal() {
    unsigned long long pol;
    asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}

template <typename T>
struct MemHint {
    unsigned long long ld_pol, st_pol;
    __device__ __forceinline__ cx<T> ld(const cx<T>* p) const {
        cx<T> r;
        if constexpr (sizeof(T) == 8)
            asm volatile("ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(r.x), "=d"(r.y) : "l"(p), "l"(ld_pol) : "memory");
        else
            asm volatile("ld.global.L2::cache_hint.v2.f32 {%0, %1}, [%2], %3;" : "=f"(r.x), "=f"(r.y) : "l"(p), "l"(ld_pol) : "memory");
        return r;
    }
    __device__ __forceinline__ void st(cx<T>* p, cx<T> v) const {
        if constexpr (sizeof(T) == 8)
            asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y), "l"(st_pol) : "memory");
        else
            asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"(v.x), "f"(v.y), "l"(st_pol) : "memory");
    }
};

// Real multiply of a finished value by the output scale.  __dmul_rn / __fmul_rn are never contracted into an FMA, so the
// stored value is exactly the unscaled result times s, rounded once in the kernel's precision.
template <typename T>
__device__ __forceinline__ cx<T> cscale(cx<T> v, T s) {
    if constexpr (sizeof(T) == 8) return cx<T>{__dmul_rn(v.x, s), __dmul_rn(v.y, s)};
    else return cx<T>{__fmul_rn(v.x, s), __fmul_rn(v.y, s)};
}

// store policy of the scaled twins: the policy M, with every stored value scaled first
template <typename T, typename M>
struct MemScaled {
    using Stored = typename StoredOf<T, M>::type;
    M m;
    T s;
    __device__ __forceinline__ cx<T> ld(const Stored* p) const { return m.ld(p); }
    __device__ __forceinline__ void st(Stored* p, cx<T> v) const { m.st(p, cscale<T>(v, s)); }
};

// ---- padded and pruned passes (dfft_plan_create_padded, dfft_plan_create_pruned) ---------------------------------------
// A padded pass transforms N-point lines whose spectral side keeps K of the N points, a pruned pass lines whose physical
// side holds M of them, zero beyond.  Each side has a hole [lo, hi) of the line: the pass reads its loaded side's hole as
// zero without a load and never stores its stored side's hole.  Position p outside a hole is element m = p (p < lo) or
// p - (hi - lo) of that side's view, so the view and its segment table are those of a K- (M-) point axis.  Forward the
// loaded side is the physical one, inverse the spectral one.  The padded twins take the scale at run time (one
// instantiation per precision and length).
// Weighted passes (dfft_plan_set_weights) multiply each value of their spectral side by w[m], m the value's index in the
// spectral view (the K stored points of a padded side): forward as it stores, inverse as it loads, before the transform.
// They run the padded twins with WEIGHTED = true: holes (empty for plans without padding) and the scale are runtime
// values, so one instantiation per kind and length serves every weighted plan.  The unweighted twins never read w.
struct FftPadded : FftScaled {
    // Spectral hole: C2C [ceil(K/2), ceil(K/2) + N - K), R2C / C2R [K/2 + 1, N/2 + 1).  Physical hole: C2C [M, N), R2C / C2R
    // the pairs [M/2, N/2).  Empty when lo == hi.
    int ld_lo, ld_hi;  // of the loaded side
    int st_lo, st_hi;  // of the stored side
    const void* w;     // weighted passes: cx<T>[spectral points of the line], Kx, Ky, Kz (C2C) or Kz/2 + 1 (R2C / C2R); else null
    // Twiddled passes of 1D plans (dfft_plan_create_1d, TWIDDLED; DESIGN.md section 3.22): point n of line (a0, a1) is
    // multiplied by W_N^(n * (line0 + a0 + c1 * a1) * mul mod N), W_N = exp(-2 pi i / N), N = 2^log2n: forward as it is
    // loaded, inverse by the conjugate as it is stored.  tw1d: the two-level table of W_N (tw1d_at); else null.
    const void* tw1d;
    long long tw_line0, tw_c1, tw_mul;
    int tw_log2n, tw_lo_bits;
    // TRANSPOSED twiddled passes (the z pass of natural-order 1D plans, DESIGN.md section 3.23): a TILED pass whose row
    // side (forward its loaded, inverse its stored side; one segment, sN = 1) holds line b's point n at b * tw_sB + n, and
    // whose twiddle's line index is tw_line0 + b + tw_c1 * a0.  0: the plain form.
    long long tw_sB;
};
// index in the view of line position n, -1 in the hole
__device__ __forceinline__ int keep_index(int n, int lo, int hi) { return n < lo ? n : (n < hi ? -1 : n - (hi - lo)); }

// W_N^m of a twiddled pass, m reduced mod N = 2^tw_log2n: from the table [W_N^l, l < 2^lo_bits][W_N^(h 2^lo_bits), h < N / 2^lo_bits]
// (built in long double and rounded once), W_N^m = W_N^(m_hi 2^lo_bits) * W_N^(m_lo)
template <typename T>
__device__ __forceinline__ cx<T> tw1d_at(const FftPadded& p, unsigned long long m) {
    const cx<T>* t = reinterpret_cast<const cx<T>*>(p.tw1d);
    m &= (1ull << p.tw_log2n) - 1;
    const unsigned long long lo = m & ((1ull << p.tw_lo_bits) - 1), hi = m >> p.tw_lo_bits;
    return cmul(t[(size_t(1) << p.tw_lo_bits) + hi], t[lo]);
}

// the line index of a twiddled pass's tile: line0 + a0 + c1 a1, or, TRANSPOSED, line0 + b + c1 a0 (b: the thread's column)
template <bool TRANSPOSED, typename TC>
__device__ __forceinline__ unsigned long long tw1d_line(const FftPadded& p, const TC& tc) {
    if constexpr (TRANSPOSED) return (unsigned long long)(p.tw_line0 + tc.b) + (unsigned long long)p.tw_c1 * tc.a0;
    else return (unsigned long long)(p.tw_line0 + tc.a0) + (unsigned long long)p.tw_c1 * tc.a1;
}

// the row side of a TRANSPOSED pass: element n = 0 of line (a0, a1, b) of its one segment, lines tw_sB apart along b
template <typename S>
__device__ __forceinline__ S* row_line(const View& v, int a0, int a1, int b, long long sB) {
    const Seg& g = v.seg[0];
    return reinterpret_cast<S*>(g.base) + (a0 * g.sA0 + a1 * g.sA1 + (long long)b * sB);
}

// The stored row side of a TRANSPOSED pass (the inverse's) where a warp's direct stores would cover less than a 32-byte
// sector of each row (TB lines x 32 / TB points: TB > ROW_LINES): the finished tile goes through shared memory instead.
// Element i = threadIdx.x + e * THREADS of the tile is point n of column bb, a warp covering ROW_LINES columns x ROW_PTS
// consecutive points, so each row takes one 32-byte run (a whole line where it is shorter) and a quarter warp's
// shared-memory reads are consecutive columns.  The forward's row loads stay direct: the other half of a sector one warp
// reads is read by a neighbouring warp of the same tile, from L1, and staging them measured slower (DESIGN.md 3.23).
template <typename T, int N, int TB>
struct RowStage {
    static constexpr int ROW_PTS = 32 / int(sizeof(cx<T>)) < N ? 32 / int(sizeof(cx<T>)) : N;
    static constexpr int ROW_LINES = 32 / ROW_PTS;
    static constexpr bool ON = TB > ROW_LINES;
    static __device__ __forceinline__ void point(int i, int& bb, int& n) {
        constexpr int GB = ON ? TB / ROW_LINES : 1;  // column groups of a tile
        const int rest = i / 32;
        bb = (rest % GB) * ROW_LINES + i % ROW_LINES;
        n = (rest / GB) * ROW_PTS + (i / ROW_LINES) % ROW_PTS;
    }
};

// store policy of the padded twins: plain stores, scaled when s != 1 (a runtime value)
template <typename T>
struct MemRtScaled {
    bool on;
    T s;
    __device__ __forceinline__ cx<T> ld(const cx<T>* p) const { return ld_elem<T>(p); }
    __device__ __forceinline__ void st(cx<T>* p, cx<T> v) const { st_elem<T>(p, on ? cscale<T>(v, s) : v); }
};

// drop a 128-byte L2 line without writing it back (its contents become undefined)
__device__ __forceinline__ void l2_discard(const void* p) { asm volatile("discard.global.L2 [%0], 128;" ::"l"(p) : "memory"); }

// ---- one tile of a C2C pass: load, CtaFft::stages, store --------------------------------------------------
// PADDED: the loaded side keeps the line positions outside the hole [ld_lo, ld_hi), the stored side those outside
// [st_lo, st_hi) (FftPadded); a side with an empty hole takes the plain path.
// ILV (CONTIG mapping): lines of an interleaved z pass, strided by sN along n (TileCoord)
// WEIGHTED: the spectral side's values times w[m] (FftPadded::w), m their index in its view: inverse after the load,
// forward before the store
// TWIDDLED (tp: the FftPadded of a 1D plan's pass): point n of the line times W_N^(n * line index * mul) (tw1d_at):
// forward after the load, inverse its conjugate before the store
// TRANSPOSED (TILED and TWIDDLED): the row side (forward in, inverse out) holds each line contiguously, line b at
// b * tw_sB (row_line); the other side is the plain TILED view, b contiguous.  A warp's direct access covers TB lines x
// 32 / TB consecutive points, whole 32-byte sectors of each row while TB <= sizeof(cx<T>) (16 lines in f64, 8 in f32);
// wider tiles of the inverse store the row side through the tile in shared memory (RowStage).
template <typename T, int LOG2N, int LOG2E, int TB, bool TILED, bool INV, typename M, typename Hook = NoGatherHook, bool PADDED = false,
          bool ILV = false, bool WEIGHTED = false, bool TWIDDLED = false, bool TRANSPOSED = false>
__device__ __forceinline__ void c2c_tile(const FftParams& p, long long tile, cx<T>* sm, unsigned long long* tab_in, unsigned long long* tab_out,
                                         bool multi, const M& mem, const Hook& after_gather = {}, int ld_lo = 0, int ld_hi = 0, int st_lo = 0,
                                         int st_hi = 0, const cx<T>* w = nullptr, const FftPadded* tp = nullptr) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, TILED>;
    using S = typename StoredOf<T, M>::type;
    using LA = LineAccess<T, C::LINES, S>;
    using TC = TileCoord<C, TILED, TB, ILV>;
    constexpr bool STRIDED = TILED || ILV;
    constexpr int E = C::E, TPL = C::TPL;
    static_assert(!TRANSPOSED || (TILED && TWIDDLED && !WEIGHTED), "TRANSPOSED: the TILED twiddled pass");
    using RS = RowStage<T, C::N, TB>;
    constexpr bool STAGED = TRANSPOSED && INV && RS::ON;
    const TC tc(p, tile);
    const int j = tc.j, t = tc.t;
    if (multi) {
        // TILED: one table per CTA (a0, a1 are CTA-uniform), filled by the first threads;
        // CONTIG: one table per line, filled by that line's threads.
        const int line = TILED ? 0 : t;
        const int lane = TILED ? int(threadIdx.x) : j;
        const int lanes = TILED ? C::THREADS : TPL;
        LA::fill_table(p.in, tab_in, line, lane, lanes, tc.a0, tc.a1);
        LA::fill_table(p.out, tab_out, line, lane, lanes, tc.a0, tc.a1);
        __syncthreads();
    }
    const LA in(p.in, tab_in, TILED ? 0 : t, tc.a0, tc.a1, tc.b);
    const LA out(p.out, tab_out, TILED ? 0 : t, tc.a0, tc.a1, tc.b);

    cx<T> v[E];
    if (tc.valid) {
        if constexpr (TRANSPOSED && !INV) {
            const S* q = row_line<const S>(p.in, tc.a0, tc.a1, tc.b, tp->tw_sB) + j;
#pragma unroll
            for (int e = 0; e < E; ++e) v[e] = mem.ld(q + e * TPL);
        } else if (PADDED && ld_lo < ld_hi) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int m = keep_index(j + e * TPL, ld_lo, ld_hi);
                v[e] = m < 0 ? cx<T>{T(0), T(0)} : mem.ld(STRIDED ? in.at(m) : in.at1(m));
            }
        } else if (!in.multi) {
            if constexpr (!STRIDED) {
                // contiguous line: sN == 1, immediate offsets
                const S* q = in.p0 + j;
#pragma unroll
                for (int e = 0; e < E; ++e) v[e] = mem.ld(q + e * TPL);
            } else {
                const long long step = (long long)TPL * p.in.sN;
                const S* q = in.p0 + (long long)j * p.in.sN;
#pragma unroll
                for (int e = 0; e < E; ++e) { v[e] = mem.ld(q); q += step; }
            }
        } else {
#pragma unroll
            for (int e = 0; e < E; ++e) v[e] = mem.ld(STRIDED ? in.at(j + e * TPL) : in.at1(j + e * TPL));
        }
        if constexpr (WEIGHTED && INV) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int m = PADDED && ld_lo < ld_hi ? keep_index(j + e * TPL, ld_lo, ld_hi) : j + e * TPL;
                if (m >= 0) v[e] = cmul(v[e], ld_tw(w, m));
            }
        }
        if constexpr (TWIDDLED && !INV) {
            const unsigned long long step = tw1d_line<TRANSPOSED>(*tp, tc) * (unsigned long long)tp->tw_mul;
#pragma unroll
            for (int e = 0; e < E; ++e) v[e] = cmul(v[e], tw1d_at<T>(*tp, (unsigned long long)(j + e * TPL) * step));
        }
        if constexpr (INV) {
#pragma unroll
            for (int e = 0; e < E; ++e) v[e] = cswap(v[e]);
        }
    } else {
#pragma unroll
        for (int e = 0; e < E; ++e) v[e] = cx<T>{T(0), T(0)};
    }

    C::template stages<0>(v, j, t, sm, reinterpret_cast<const cx<T>*>(p.tw), after_gather);

    if constexpr (WEIGHTED && !INV) {
        if (tc.valid) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int m = PADDED && st_lo < st_hi ? keep_index(j + e * TPL, st_lo, st_hi) : j + e * TPL;
                cx<T>& x = v[C::Core::final_slot(e)];
                if (m >= 0) x = cmul(x, ld_tw(w, m));
            }
        }
    }
    if constexpr (TWIDDLED && INV) {
        // v holds the swapped values (cswap(z) = i conj(z)): multiplying them by W stores conj(W) times the result
        if (tc.valid) {
            const unsigned long long step = tw1d_line<TRANSPOSED>(*tp, tc) * (unsigned long long)tp->tw_mul;
#pragma unroll
            for (int e = 0; e < E; ++e) {
                cx<T>& x = v[C::Core::final_slot(e)];
                x = cmul(x, tw1d_at<T>(*tp, (unsigned long long)(j + e * TPL) * step));
            }
        }
    }
    if constexpr (STAGED) {  // the finished lines through shared memory, then sector-wide rows by every thread
        __syncthreads();              // every thread's last gather has left the tile
        if (tc.valid) {
#pragma unroll
            for (int e = 0; e < E; ++e) sm[C::sidx(j + e * TPL, t)] = cswap(v[C::Core::final_slot(e)]);
        }
        __syncthreads();
        const int b0 = tc.b - t;
        S* q = row_line<S>(p.out, tc.a0, tc.a1, b0, tp->tw_sB);
#pragma unroll
        for (int e = 0; e < E; ++e) {
            int bb, n;
            RS::point(int(threadIdx.x) + e * C::THREADS, bb, n);
            if (b0 + bb < p.B) mem.st(q + (long long)bb * tp->tw_sB + n, sm[C::sidx(n, bb)]);
        }
    } else if (tc.valid) {
        if constexpr (TRANSPOSED && INV) {
            S* q = row_line<S>(p.out, tc.a0, tc.a1, tc.b, tp->tw_sB) + j;
#pragma unroll
            for (int e = 0; e < E; ++e) mem.st(q + e * TPL, cswap(v[C::Core::final_slot(e)]));
        } else if (PADDED && st_lo < st_hi) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int m = keep_index(j + e * TPL, st_lo, st_hi);
                const cx<T> x = v[C::Core::final_slot(e)];
                if (m >= 0) mem.st(STRIDED ? out.at(m) : out.at1(m), INV ? cswap(x) : x);
            }
        } else if (!out.multi) {
            if constexpr (!STRIDED) {
                S* q = out.p0 + j;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const cx<T> x = v[C::Core::final_slot(e)];
                    mem.st(q + e * TPL, INV ? cswap(x) : x);
                }
            } else {
                const long long step = (long long)TPL * p.out.sN;
                S* q = out.p0 + (long long)j * p.out.sN;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const cx<T> x = v[C::Core::final_slot(e)];
                    mem.st(q, INV ? cswap(x) : x);
                    q += step;
                }
            }
        } else {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const cx<T> x = v[C::Core::final_slot(e)];
                mem.st(STRIDED ? out.at(j + e * TPL) : out.at1(j + e * TPL), INV ? cswap(x) : x);
            }
        }
    }
}

// ---- C2C pass ------------------------------------------------------------------------------------------
// Grid-stride over tiles: launched with one CTA per tile it is the plain kernel; launched with fewer CTAs
// (FftParams::max_ctas) it is persistent and occupies only that many CTA slots, which is how the overlapped
// schedule leaves the rest of the GPU to the other passes.
// S: the stored element (MemPlain).
template <typename T, typename S, int LOG2N, int LOG2E, int TB, bool TILED, bool INV, bool SCALED>
__device__ __forceinline__ void c2c_pass(const KParams<SCALED>& p) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, TILED>;
    using TC = TileCoord<C, TILED, TB>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const bool multi = p.in.nseg > 1 || p.out.nseg > 1;
    const long long ntiles = TC::num_tiles(p);

#pragma unroll 1
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if constexpr (SCALED)
            c2c_tile<T, LOG2N, LOG2E, TB, TILED, INV>(p, tile, sm, tab_in, tab_out, multi, MemScaled<T, MemPlain<T, S>>{{}, T(p.scale)});
        else c2c_tile<T, LOG2N, LOG2E, TB, TILED, INV>(p, tile, sm, tab_in, tab_out, multi, MemPlain<T, S>{});
        const int t = TILED ? int(threadIdx.x) % TB : int(threadIdx.x) / C::TPL;
        if (tile + gridDim.x < ntiles) {
            // persistent use: the next tile's first scatter must not overtake this tile's last gather, and
            // the segment tables are rewritten
            if (multi) __syncthreads();
            else if constexpr (C::NST > 1) C::sync(t);
        }
    }
}

// S = cx16<H> (H = __half or __nv_bfloat16, T = float): the C2C pass of 16-bit plans, cx16<H> in memory, the f32 core, tile
// and twiddles of the f32 pass, so each line is the f32 pass's result rounded once to 16 bits (the scaled twin: times
// float(p.scale) first).
template <typename T, typename S, int LOG2N, int LOG2E, int TB, bool TILED, bool INV, bool SCALED>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_c2c_kernel(const __grid_constant__ KParams<SCALED> p) {
    c2c_pass<T, S, LOG2N, LOG2E, TB, TILED, INV, SCALED>(p);
}

// Interleaved z pass (PASS_C2C_ILV, C = p.B components per point, below the TILED tile width): the CONTIG shape with its
// TB lines taken as consecutive (row, component) pairs, so a CTA's lines cover whole runs of [row][N][C] and the strided
// accesses of one component are served by the same sectors as its neighbours'.  Same core, stage plan and tables as the
// CONTIG kernel: bit-identical lines.  Grid-stride like fft_c2c_kernel (max_ctas).
template <typename T, int LOG2N, int LOG2E, int TB, bool INV, bool SCALED>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_c2c_ilv_kernel(const __grid_constant__ KParams<SCALED> p) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, false>;
    using TC = TileCoord<C, false, TB, true>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const bool multi = p.in.nseg > 1 || p.out.nseg > 1;
    const long long ntiles = TC::num_tiles(p);

#pragma unroll 1
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if constexpr (SCALED)
            c2c_tile<T, LOG2N, LOG2E, TB, false, INV, MemScaled<T, MemPlain<T>>, NoGatherHook, false, true>(p, tile, sm, tab_in, tab_out, multi,
                                                                                                       MemScaled<T, MemPlain<T>>{{}, T(p.scale)});
        else c2c_tile<T, LOG2N, LOG2E, TB, false, INV, MemPlain<T>, NoGatherHook, false, true>(p, tile, sm, tab_in, tab_out, multi, MemPlain<T>{});
        if (tile + gridDim.x < ntiles) {
            if (multi) __syncthreads();
            else if constexpr (C::NST > 1) C::sync(int(threadIdx.x) / C::TPL);
        }
    }
}

// R2C / C2R z pass of interleaved plans (PASS_R2C_ILV / PASS_C2R_ILV, C = p.B components per point, r2r.hpp): the CONTIG
// shape with its TB lines taken as consecutive (row, component) items; every component runs its own complex N-point line
// (N = Nz) with a zero imaginary part, so each component's result depends on that component alone.  The real side is one
// segment counted in reals (element (a0, a1, n, c) at base + a0 sA0 + a1 sA1 + n sN + c), the complex side a view with b the
// component (segment tables along z for scatters and gathers).  R2C: after the stages Z goes through the line's shared
// memory once, each thread splits its k <= N/2 with Z[N - k].  C2R: each thread builds Z[k] from X[k] or conj X[N - k],
// straight from global memory.  Grid-stride like fft_c2c_kernel (max_ctas).
template <typename T, int LOG2N, int LOG2E, int TB, bool C2R, bool SCALED>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_rc_ilv_kernel(const __grid_constant__ KParams<SCALED> p) {
    using Cf = CtaFft<T, LOG2N, LOG2E, TB, false>;
    using LA = LineAccess<T, TB>;
    constexpr int E = Cf::E, TPL = Cf::TPL, N = Cf::N;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab = reinterpret_cast<unsigned long long*>(smem_raw + Cf::TILE_BYTES);
    const View& rv = C2R ? p.out : p.in;
    const View& cv = C2R ? p.in : p.out;
    const bool multi = cv.nseg > 1;
    const int C = p.B;
    const long long nlines = (long long)p.A0 * p.A1 * C;
    const long long ntiles = (nlines + TB - 1) / TB;
    const int j = int(threadIdx.x) % TPL, t = int(threadIdx.x) / TPL;
    T s = T(1);
    if constexpr (SCALED) s = T(p.scale);
    const cx<T>* tw = reinterpret_cast<const cx<T>*>(p.tw);

#pragma unroll 1
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const long long line = tile * TB + t;
        const bool valid = line < nlines;
        const int c = int(line % C);
        const long long row = line / C;
        const int a1 = int(row % p.A1), a0 = int(row / p.A1);
        if (multi) {
            LA::fill_table(cv, tab, t, j, TPL, a0, a1);
            __syncthreads();
        }
        const LA x(cv, tab, t, a0, a1, c);
        T* r0 = reinterpret_cast<T*>(rv.seg[0].base) + ((long long)a0 * rv.seg[0].sA0 + (long long)a1 * rv.seg[0].sA1 + c);
        cx<T> v[E];
        if constexpr (!C2R) {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const long long o = (long long)(j + e * TPL) * rv.sN;
                v[e] = cx<T>{valid ? r0[o] : T(0), T(0)};
            }
            Cf::template stages<0>(v, j, t, sm, tw);
            Cf::sync(t);  // the line's last gather has left shared memory
#pragma unroll
            for (int e = 0; e < E; ++e) sm[Cf::sidx(j + e * TPL, t)] = v[Cf::Core::final_slot(e)];
            Cf::sync(t);
            if (valid) {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const int k = j + e * TPL;
                    if (2 * k > N) continue;
                    cx<T> y = rc_line_split<T>(sm[Cf::sidx(k, t)], sm[Cf::sidx((N - k) & (N - 1), t)]);
                    if constexpr (SCALED) y = cscale<T>(y, s);
                    st_elem<T>(x.at(k), y);
                }
            }
        } else {
#pragma unroll
            for (int e = 0; e < E; ++e) {
                const int k = j + e * TPL;
                cx<T> z{T(0), T(0)};
                if (valid) z = rc_line_build<T>(ld_elem<T>(x.at(rc_line_in_k(k, N))), k, N);
                v[e] = cswap(z);
            }
            Cf::template stages<0>(v, j, t, sm, tw);
            if (valid) {
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    T z = cswap(v[Cf::Core::final_slot(e)]).x;
                    if constexpr (SCALED) z *= s;
                    r0[(long long)(j + e * TPL) * rv.sN] = z;
                }
            }
        }
        if (tile + gridDim.x < ntiles) {
            // the next tile's first scatter (and, multi-segment, its tables) must not overtake this tile's shared-memory reads
            if (multi) __syncthreads();
            else Cf::sync(t);
        }
    }
}

// padded twin of fft_c2c_kernel (FftPadded), with WEIGHTED its weighted twin (p.w), with TWIDDLED the twiddled pass of
// 1D plans (p.tw1d), with TRANSPOSED its transposing form (p.tw_sB): one CTA per tile
template <typename T, int LOG2N, int LOG2E, int TB, bool TILED, bool INV, bool WEIGHTED, bool TWIDDLED = false, bool TRANSPOSED = false>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_c2c_padded_kernel(const __grid_constant__ FftPadded p) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, TILED>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const bool multi = p.in.nseg > 1 || p.out.nseg > 1;
    c2c_tile<T, LOG2N, LOG2E, TB, TILED, INV, MemRtScaled<T>, NoGatherHook, true, false, WEIGHTED, TWIDDLED, TRANSPOSED>(
        p, blockIdx.x, sm, tab_in, tab_out, multi, MemRtScaled<T>{p.scale != 1.0, T(p.scale)}, {}, p.ld_lo, p.ld_hi, p.st_lo, p.st_hi,
        WEIGHTED ? reinterpret_cast<const cx<T>*>(p.w) : nullptr, TWIDDLED ? &p : nullptr);
}

// ---- mbarrier of an asynchronous tile copy (fft_c2c_tma_kernel, fft_zy_fused_kernel) ------------------------------
struct TmaBar {
    static __device__ __forceinline__ void init(unsigned long long* bar, unsigned count) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(unsigned(__cvta_generic_to_shared(bar))), "r"(count) : "memory");
    }
    static __device__ __forceinline__ void expect(unsigned long long* bar, unsigned bytes) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(unsigned(__cvta_generic_to_shared(bar))), "r"(bytes) : "memory");
    }
    static __device__ __forceinline__ bool try_wait(unsigned a, unsigned parity) {
        unsigned ok;
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(a), "r"(parity) : "memory");
        return ok != 0;
    }
    // bounded wait: a lost transaction must not hang the GPU (returns false after ~2 s)
    static __device__ __forceinline__ bool wait(unsigned long long* bar, unsigned parity) {
        const unsigned a = unsigned(__cvta_generic_to_shared(bar));
        for (long long spin = 0; spin < (1ll << 26); ++spin)
            if (try_wait(a, parity)) return true;
        return false;
    }
    // wait of at most `cycles` clock64 cycles (0 = no limit); false when they ran out
    static __device__ __forceinline__ bool wait_for(unsigned long long* bar, unsigned parity, long long cycles) {
        const unsigned a = unsigned(__cvta_generic_to_shared(bar));
        const long long t0 = clock64();
        while (!try_wait(a, parity))
            if (cycles > 0 && clock64() - t0 > cycles) return false;
        return true;
    }
};

// ---- fused z + y stage of one-rank slab transforms ---------------------------------------------------------
// One persistent launch runs the z pass (CONTIG, `pz`) and the y pass (TILED, `py`) of the same x-planes, plane group
// by plane group, so that the intermediate one pass writes is still in the L2 when the other reads it (ZyOrder in
// zy_order.hpp).  Forward: phase A = z lines (caller's input -> intermediate slot), phase B = y tiles (slot -> blocked
// hand-over of the x pass).  Inverse (INV): phase A = y tiles (blocked hand-over -> slot), phase B = z lines (slot ->
// caller's output).  Both phases run the per-tile code of fft_c2c_kernel (c2c_tile), so every line is transformed by
// exactly the arithmetic of the standalone passes; only the CTA shape is shared: TB y columns or TB z lines.
//
// L2 policy (per instruction only; no persisting-L2 carve-out, a device-wide setting):
//   * streaming data — phase A's input, phase B's output — is loaded / stored with L2::evict_first;
//   * phase A stores the intermediate with L2::evict_last;
//   * a phase-B CTA discards (discard.global.L2) every 128-byte line of the intermediate it has read, once its tile is
//     stored: the line is dead and is dropped without a write-back to HBM.  That needs every such line to
//     be read by one CTA only — 128-byte y-tile rows (TB * sizeof(complex) a multiple of 128) and z lines of a multiple
//     of 128 bytes, on 128-byte aligned views (ZyFused::discard, checked by the launcher).
//
// Fed by asynchronous copies (FED, the default where the views allow it): every item's N x TB input points arrive by
// cp.async.bulk (z lines) or cp.async.bulk.tensor (y tiles) in shared memory, announced by an mbarrier, and the next
// item's copy is requested as soon as the current item's last gather has left the buffer (fft_zy_fed_kernel).  The
// register-fed form (fft_zy_fused_kernel, c2c_tile) stays for f32 and for views the copies cannot address (16-byte
// alignment); launch_zy_fused chooses.
//
// The parameters of the two persistent two-phase kernels (this one and fft_batch_small_kernel) begin with TicketWork, the
// state of their common ticket loop (ticket_loop).
struct TicketWork {
    unsigned long long* ctr;   // [0] ticket counter, [1 + g] finished phase-A items of group g; zeroed once, never reset
    int* err;                  // the plan's device error flag
    long long timeout_cycles;  // clock64 cycles a dependency wait may take (0 = no limit)
    ZyOrder order;
#ifdef DFFT_ZY_TRACE
    unsigned long long* trace;  // trace build: ZY_TRACE_SLOTS stamps per ticket of the last launch (null: none)
#endif
};

// Trace build (-DDFFT_ZY_TRACE, tools/zy_trace.py): thread 0 of a CTA writes %globaltimer stamps per work item into
// TicketWork::trace[ticket * ZY_TRACE_SLOTS + k].  The default build compiles none of it.
constexpr int ZY_TRACE_SLOTS = 8;
enum ZyStamp {
    ZY_TICKET = 0,      // ticket read from the broadcast slot
    ZY_DEP_MET = 1,     // dependencies met (phase A: at once)
    ZY_INPUTS = 2,      // fed kernel: the item's copy has landed
    ZY_EXCHANGED = 3,   // first exchange through shared memory done (register-fed kernel: its loads have arrived)
    ZY_LAST_GATHER = 4, // last gather done: the buffer is free
    ZY_STORED = 5,      // every store of the item issued (thread 0)
    ZY_DONE = 6,        // counted done / discards issued
    ZY_WHERE = 7        // (smid << 32) | (CTA << 1) | phase
};
#ifdef DFFT_ZY_TRACE
__device__ __forceinline__ void zy_stamp(const TicketWork& f, long long ticket, int k) {
    if (f.trace && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        f.trace[ticket * ZY_TRACE_SLOTS + k] = t;
    }
}
__device__ __forceinline__ void zy_stamp_where(const TicketWork& f, long long ticket, int phase) {
    if (f.trace && threadIdx.x == 0) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        f.trace[ticket * ZY_TRACE_SLOTS + ZY_WHERE] = ((unsigned long long)smid << 32) | ((unsigned long long)blockIdx.x << 1) | unsigned(phase);
    }
}
#define ZY_STAMP(f, ticket, k) zy_stamp(f, ticket, k)
#define ZY_STAMP_WHERE(f, ticket, phase) zy_stamp_where(f, ticket, phase)
#else
#define ZY_STAMP(f, ticket, k) ((void)0)  // the arguments (volatile shared reads among them) are not evaluated
#define ZY_STAMP_WHERE(f, ticket, phase) ((void)0)
#endif
struct ZyFused : TicketWork {
    int discard;  // phase B may discard the intermediate lines it has read
};
constexpr int ZY_ERR_TIMEOUT = 200;   // value of the error flag when a fused-stage wait (dependency or input copy) timed out

// The ticket loop of a persistent two-phase kernel: draws tickets until the work list is done, waits before each phase-B
// item until every phase-A item of its group has finished, and runs item(it, slot) for every work item `it` (all threads;
// *slot holds its ticket).  Shared memory `bcast`: bcast[par] the current ticket; bcast[par ^ 1] the next one, drawn while
// this item runs (the atomic's latency is hidden behind the tile's loads).  Values are re-read from shared memory where
// needed instead of being kept in registers through the tiles.  bcast[2]: give up.  bcast[3], bcast[4]: this launch's
// counter base and epoch, fixed by the CTA's first draw (zy_launch_of) — the kernel takes no per-exec value from the host,
// so a graph can replay it.  A timed-out wait sets the error flag to timeout_err and ends the loop.
// ready(it, ticket): thread 0, once the item's dependencies are met and before the item runs (the fused stage requests the
// item's input there unless it did so earlier).  An item that returns a bool ends the loop by returning false (the same
// value in every thread).
struct NoFeed {
    __device__ __forceinline__ void operator()(const ZyItem&, long long) const {}
};
template <typename Item, typename Ready = NoFeed>
__device__ __forceinline__ void ticket_loop(const TicketWork& f, volatile long long* bcast, int timeout_err, const Item& item, const Ready& ready = {}) {
    const int tid = threadIdx.x;
    const long long total = f.order.total();
    int par = 0;
    if (tid == 0) {
        const unsigned long long raw = atomicAdd(f.ctr, 1ull);
        const ZyLaunch l = zy_launch_of(raw, f.order.draws(gridDim.x));
        bcast[3] = (long long)l.base;
        bcast[4] = (long long)l.epoch;
        bcast[0] = (long long)(raw - l.base);
    }
#pragma unroll 1
    for (;; par ^= 1) {
        __syncthreads();
        const long long ticket = bcast[par];
        if (ticket >= total) break;
        ZY_STAMP(f, ticket, ZY_TICKET);
        if (tid == 0) bcast[par ^ 1] = (long long)(atomicAdd(f.ctr, 1ull) - (unsigned long long)bcast[3]);
        const ZyItem it = f.order.decode(ticket);
        if (it.phase == 1) {
            // Wait until every phase-A item of this group has finished.  This cannot deadlock: tickets are handed out in
            // increasing order and only to CTAs that are already running, and every item a ticket depends on has a lower
            // ticket (zy_order.hpp).  So the lowest unfinished ticket is held by a resident CTA whose earlier item is
            // finished, and all its dependencies are finished: it completes, and by induction so does every ticket —
            // with any number of resident CTAs, also when other work on the GPU leaves this launch fewer CTAs than it
            // asked for.  The wait is still bounded (the plan's rendezvous timeout): a logic error surfaces as an error
            // code, not a hung GPU.
            if (tid == 0) {
                const unsigned long long target = (unsigned long long)bcast[4] * (unsigned long long)f.order.a_items(it.group);
                const unsigned long long* c = f.ctr + 1 + it.group;
                unsigned long long v;
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(c) : "memory");
                long long bail = 0;
                if (v < target) {
                    const long long t0 = clock64();
                    while (true) {
                        __nanosleep(32);
                        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(c) : "memory");
                        if (v >= target) break;
                        if (f.timeout_cycles > 0 && clock64() - t0 > f.timeout_cycles) {
                            atomicExch(f.err, timeout_err);
                            bail = 1;
                            break;
                        }
                    }
                }
                bcast[2] = bail;
                if (!bail) ready(it, ticket);
            }
            __syncthreads();
            if (bcast[2]) break;
        } else if (tid == 0) {
            ready(it, ticket);
        }
        ZY_STAMP(f, ticket, ZY_DEP_MET);
        ZY_STAMP_WHERE(f, ticket, it.phase);
        if constexpr (std::is_same_v<decltype(item(it, bcast + par)), bool>) {
            if (!item(it, bcast + par)) break;
        } else {
            item(it, bcast + par);
        }
    }
}

template <typename T, int LOG2N>
struct ZyShape {
    using S = Shape<T, LOG2N>;
    static constexpr int LOG2E = S::LOG2E, TB = S::TBT;
    using CY = CtaFft<T, LOG2N, LOG2E, TB, true>;
    using CZ = CtaFft<T, LOG2N, LOG2E, TB, false>;
    static constexpr int THREADS = CY::THREADS;
    static_assert(CZ::THREADS == THREADS, "one CTA shape for both phases");
    static_assert(CY::NST >= 2 && CZ::NST >= 2, "the discard hook runs after the first exchange through shared memory");
    static constexpr size_t TILE_BYTES = CY::TILE_BYTES > CZ::TILE_BYTES ? CY::TILE_BYTES : CZ::TILE_BYTES;
    static constexpr size_t TABLE_BYTES = CY::TABLE_BYTES > CZ::TABLE_BYTES ? CY::TABLE_BYTES : CZ::TABLE_BYTES;
    static constexpr size_t SMEM_BYTES = TILE_BYTES + TABLE_BYTES + 48;  // + the ticket broadcast
    // 128-byte lines of the intermediate a phase-B tile owns entirely
    static constexpr bool Y_DISCARD = (TB * sizeof(cx<T>)) % 128 == 0;
    static constexpr bool Z_DISCARD = ((1 << LOG2N) * sizeof(cx<T>)) % 128 == 0;
};

// End of a work item of fft_zy_fused_kernel (all threads, after the tile is stored): a phase-A item counts itself done,
// a phase-B item of the register-fed kernel (DISCARD) drops the intermediate lines it has read.  Kept out of line: the
// kernel runs at its 128-register limit and this bookkeeping, inlined into the loop, made the register allocator spill the
// tile's points.
template <typename T, int LOG2N, bool INV, bool DISCARD>
__device__ __noinline__ void zy_item_done(const FftParams& pz, const FftParams& py, const ZyFused& f, long long ticket) {
    using Z = ZyShape<T, LOG2N>;
    constexpr int TB = Z::TB, N = 1 << LOG2N;
    const ZyItem done = f.order.decode(ticket);
    const int tid = threadIdx.x;
    if (done.phase == 0) {
        // release at gpu scope, after the barrier that ordered every thread's stores of the item before this thread
        if (tid == 0) asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(f.ctr + 1 + done.group) : "memory");
    } else if (DISCARD && f.discard) {
        // Phase B: the intermediate this tile read is dead — drop its 128-byte lines without a write-back.  The
        // register-fed kernel does it here, after the tile, rather than as soon as it is in registers: with the 16
        // points per thread live the extra addressing spilled registers, and a line survives the few microseconds of
        // one tile.  The fed kernel calls this with the item's bytes in shared memory and nothing live.
        if (INV) {  // phase B = z lines
            if constexpr (Z::Z_DISCARD) {
                constexpr int PER_LINE = int(N * sizeof(cx<T>)) / 128;  // TB lines of this tile
                for (int k = tid; k < TB * PER_LINE; k += Z::THREADS) {
                    const long long line = done.tile * TB + k / PER_LINE;
                    const long long a1 = line % pz.A1, a0 = line / pz.A1;
                    const char* q = reinterpret_cast<const char*>(reinterpret_cast<const cx<T>*>(pz.in.seg[0].base) + a0 * pz.in.seg[0].sA0 +
                                                                  a1 * pz.in.seg[0].sA1);
                    l2_discard(q + (k % PER_LINE) * 128);
                }
            }
        } else {
            if constexpr (Z::Y_DISCARD) {
                constexpr int PER_ROW = int(TB * sizeof(cx<T>)) / 128;
                int bt, a1, a0;
                tiled_decode<TB>(py, done.tile, bt, a1, a0);
                const cx<T>* b0 = reinterpret_cast<const cx<T>*>(py.in.seg[0].base) + a0 * py.in.seg[0].sA0 + a1 * py.in.seg[0].sA1 + bt * TB;
                for (int k = tid; k < N * PER_ROW; k += Z::THREADS)
                    l2_discard(reinterpret_cast<const char*>(b0 + (long long)(k / PER_ROW) * py.in.sN) + (k % PER_ROW) * 128);
            }
        }
    }
}

// One work item of the fed stage (all threads): its N x TB points are in shared memory as the copies wrote them — TB dense
// z lines [t][n], or a dense y tile [n][TB].  One gather into registers, then the buffer becomes the padded exchange space
// of CtaFft::stages; from there on the arithmetic is c2c_tile's, so the results are bit-identical.  `ok`: this thread's
// wait for the copy succeeded; false in any thread ends the item in every thread (returns false).
template <typename T, int LOG2N, int LOG2E, int TB, bool TILED, bool INV, typename M, typename Hook>
__device__ __forceinline__ bool zy_fed_tile(const FftParams& p, long long tile, cx<T>* sm, const M& mem, bool ok, const Hook& after_gather) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, TILED>;
    constexpr int E = C::E, TPL = C::TPL, N = C::N;
    const TileCoord<C, TILED, TB> tc(p, tile);
    const int j = tc.j, t = tc.t;
    cx<T> v[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const cx<T> x = TILED ? sm[(j + e * TPL) * TB + t] : sm[t * N + j + e * TPL];
        v[e] = INV ? cswap(x) : x;
    }
    if (__syncthreads_or(!ok)) return false;
    C::template stages<0>(v, j, t, sm, reinterpret_cast<const cx<T>*>(p.tw), after_gather);
    if (tc.valid) {
        const Seg& g = p.out.seg[0];
        cx<T>* q = reinterpret_cast<cx<T>*>(g.base) + (tc.a0 * g.sA0 + tc.a1 * g.sA1 - (long long)g.n0 * p.out.sN + tc.b) + (long long)j * p.out.sN;
        const long long step = (long long)TPL * p.out.sN;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const cx<T> x = v[C::Core::final_slot(e)];
            if constexpr (TILED) {
                mem.st(q, INV ? cswap(x) : x);
                q += step;
            } else {
                mem.st(q + e * TPL, INV ? cswap(x) : x);  // contiguous line: sN == 1
            }
        }
    }
    return true;
}

// global -> shared copies of the fed stage, completing on the mbarrier at shared address mb, with an L2 policy
__device__ __forceinline__ void bulk_load(unsigned dst, const void* src, unsigned bytes, unsigned mb, unsigned long long pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(mb), "l"(pol) : "memory");
}
__device__ __forceinline__ void tensor_load4(unsigned dst, const CUtensorMap* tm, int c0, int c1, int c2, int c3, unsigned mb, unsigned long long pol) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
                 ::"r"(dst), "l"(tm), "r"(mb), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol) : "memory");
}

// SCALED (inverse only): phase B, the z lines that store the caller's output, scales its stores by pz.scale.
// Register-fed form: every item's inputs by 16-byte loads into registers (c2c_tile).
template <typename T, int LOG2N, bool INV, bool SCALED>
__global__ void __launch_bounds__(ZyShape<T, LOG2N>::THREADS, min_ctas_per_sm<T, ZyShape<T, LOG2N>::LOG2E>(ZyShape<T, LOG2N>::THREADS))
fft_zy_fused_kernel(const __grid_constant__ KParams<SCALED> pz, const __grid_constant__ FftParams py, const __grid_constant__ ZyFused f) {
    static_assert(INV || !SCALED, "the forward fused stage stores the intermediate of the x pass only");
    using Z = ZyShape<T, LOG2N>;
    constexpr int TB = Z::TB;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + Z::TILE_BYTES);
    unsigned long long* tab_out = tab_in + (Z::TABLE_BYTES - 16) / 16;
    volatile long long* bcast = reinterpret_cast<volatile long long*>(smem_raw + Z::TILE_BYTES + Z::TABLE_BYTES);
    ticket_loop(f, bcast, ZY_ERR_TIMEOUT, [&](const ZyItem& it, const volatile long long* slot) {
        const bool z_item = (it.phase == 0) == !INV;  // forward: phase A = z; inverse: phase A = y
        const MemHint<T> mem_a{l2_evict_first(), l2_evict_last()};   // streaming input -> intermediate
        const MemHint<T> mem_b{l2_evict_normal(), l2_evict_first()};  // intermediate -> streaming output
        // trace build: the first exchange and the last gather (nothing in the default build)
        auto stamp = [&](auto st) {
            constexpr int ST = decltype(st)::value, NST = CtaFft<T, LOG2N, Z::LOG2E, TB, false>::NST;
            if constexpr (ST == 0) ZY_STAMP(f, *slot, ZY_EXCHANGED);
            if constexpr (ST + 2 == NST) ZY_STAMP(f, *slot, ZY_LAST_GATHER);
        };
        if (z_item) {
            if (it.phase == 0) c2c_tile<T, LOG2N, Z::LOG2E, TB, false, INV>(pz, it.tile, sm, tab_in, tab_out, false, mem_a, stamp);
            else if constexpr (SCALED) c2c_tile<T, LOG2N, Z::LOG2E, TB, false, INV>(pz, it.tile, sm, tab_in, tab_out, false, MemScaled<T, MemHint<T>>{mem_b, T(pz.scale)}, stamp);
            else c2c_tile<T, LOG2N, Z::LOG2E, TB, false, INV>(pz, it.tile, sm, tab_in, tab_out, false, mem_b, stamp);
        } else {
            if (it.phase == 0) c2c_tile<T, LOG2N, Z::LOG2E, TB, true, INV>(py, it.tile, sm, tab_in, tab_out, false, mem_a, stamp);
            else c2c_tile<T, LOG2N, Z::LOG2E, TB, true, INV>(py, it.tile, sm, tab_in, tab_out, false, mem_b, stamp);
        }
        ZY_STAMP(f, *slot, ZY_STORED);
        // the tile is stored and shared memory is free again before the item counts
        __syncthreads();
        zy_item_done<T, LOG2N, INV, true>(pz, py, f, *slot);
        ZY_STAMP(f, *slot, ZY_DONE);
    });
}

// Fed form (complex-double): inputs by asynchronous copies.  tm_y: rank-4 map (b, n, a1, a0) of py.in, box TB x min(N, 256).
template <typename T, int LOG2N, bool INV, bool SCALED>
__global__ void __launch_bounds__(ZyShape<T, LOG2N>::THREADS, min_ctas_per_sm<T, ZyShape<T, LOG2N>::LOG2E>(ZyShape<T, LOG2N>::THREADS))
fft_zy_fed_kernel(const __grid_constant__ KParams<SCALED> pz, const __grid_constant__ FftParams py, const __grid_constant__ ZyFused f,
                  const __grid_constant__ CUtensorMap tm_y) {
    static_assert(INV || !SCALED, "the forward fused stage stores the intermediate of the x pass only");
    using Z = ZyShape<T, LOG2N>;
    constexpr int TB = Z::TB, N = 1 << LOG2N, NST = CtaFft<T, LOG2N, Z::LOG2E, TB, false>::NST;
    constexpr unsigned TILE_TX = unsigned(N) * TB * unsigned(sizeof(cx<T>));  // bytes of one item, either kind
    constexpr int D0 = sizeof(T) == 8 ? 2 : 1;                                // 8-byte map units per complex element
    static_assert(TILE_TX <= Z::TILE_BYTES, "an item's dense landing fits the tile buffer");
    static_assert(NST == CtaFft<T, LOG2N, Z::LOG2E, TB, true>::NST, "one stage count for both phases");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(smem_raw + Z::TILE_BYTES + Z::TABLE_BYTES - 16);  // tables unused
    volatile long long* bcast = reinterpret_cast<volatile long long*>(smem_raw + Z::TILE_BYTES + Z::TABLE_BYTES);
    const int tid = threadIdx.x;
    const long long total = f.order.total();
    long long requested = -1;  // thread 0: the last ticket whose input copy was issued
    unsigned parity = 0;
    if (tid == 0) {
        TmaBar::init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }  // the ticket loop's first barrier orders the init before any use

    // thread 0: arm the barrier and issue the copies of item n (phase A input: evict_first, as the register-fed loads)
    auto request = [&](const ZyItem& n, long long ticket) {
        requested = ticket;
        const unsigned dst = unsigned(__cvta_generic_to_shared(sm));
        const unsigned mb = unsigned(__cvta_generic_to_shared(bar));
        const unsigned long long pol = n.phase == 0 ? l2_evict_first() : l2_evict_normal();
        TmaBar::expect(bar, TILE_TX);
        if ((n.phase == 0) == !INV) {
            // TB consecutive z lines of one a0 (A1 % TB == 0): one range when adjacent, else one copy per line
            const long long line = n.tile * TB;
            const Seg& g = pz.in.seg[0];
            const cx<T>* src = reinterpret_cast<const cx<T>*>(g.base) + ((line / pz.A1) * g.sA0 + (line % pz.A1) * g.sA1 - g.n0);
            if (g.sA1 == N) {
                bulk_load(dst, src, TILE_TX, mb, pol);
            } else {
#pragma unroll 1
                for (int t = 0; t < TB; ++t) bulk_load(dst + t * unsigned(N * sizeof(cx<T>)), src + t * g.sA1, unsigned(N * sizeof(cx<T>)), mb, pol);
            }
        } else {
            int bt, a1, a0;
            tiled_decode<TB>(py, n.tile, bt, a1, a0);
#pragma unroll
            for (int r = 0; r < N; r += 256)
                tensor_load4(dst + unsigned(r) * TB * unsigned(sizeof(cx<T>)), &tm_y, bt * TB * D0, r, a1, a0, mb, pol);
        }
    };
    // ticket loop, thread 0, dependencies met: the item's copy, unless it was issued early.  A phase-B item reads what
    // other CTAs stored through the generic proxy (acquired by the counter wait); the proxy fence orders those stores
    // before this thread's async-proxy read.
    auto ready = [&](const ZyItem& it, long long ticket) {
        if (requested == ticket) return;
        if (it.phase == 1) asm volatile("fence.proxy.async.global;" ::: "memory");
        request(it, ticket);
    };
    ticket_loop(f, bcast, ZY_ERR_TIMEOUT, [&](const ZyItem& it, const volatile long long* slot) -> bool {
        // A timed-out wait (the plan's timeout, seconds) sets the error flag and ends the loop in every thread.  The copy
        // it waited for may then still be in flight into this CTA's shared memory after the CTA has exited; as after a
        // timed-out dependency wait, the plan's device state is undefined once the flag is set (dfft_plan_wait reports it).
        const bool ok = TmaBar::wait_for(bar, parity, f.timeout_cycles);
        parity ^= 1;
        ZY_STAMP(f, *slot, ZY_INPUTS);
        if (!ok) atomicExch(f.err, ZY_ERR_TIMEOUT);
        else if (it.phase == 1) zy_item_done<T, LOG2N, INV, true>(pz, py, f, *slot);  // its intermediate is dead: discard
        // Early request of the next item, once the last gather of this one has left the buffer (every thread, between
        // the last gather and the last stage).  A phase-A item is requested at once.  A phase-B item is requested only
        // if its group counter has reached the target at the first look: thread 0 never waits here while this item is
        // unfinished, otherwise the request waits for the top of the loop, after this item has counted itself done.
        // So ticket_loop's argument holds word for word: the lowest unfinished ticket is held by a resident CTA whose
        // earlier item is finished, all its dependencies are finished, and nothing it waits for depends on later work.
        const volatile long long* next_slot = bcast + ((slot - bcast) ^ 1);
        auto after_gather = [&](auto st) {
            constexpr int ST = decltype(st)::value;
            if constexpr (ST == 0) ZY_STAMP(f, *slot, ZY_EXCHANGED);
            if constexpr (ST + 2 == NST) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic reads of the buffer before the async write
                __syncthreads();
                ZY_STAMP(f, *slot, ZY_LAST_GATHER);
                if (tid == 0) {
                    const long long next = *next_slot;
                    if (next < total) {
                        const ZyItem n = f.order.decode(next);
                        bool go = n.phase == 0;
                        if (!go) {
                            const unsigned long long target = (unsigned long long)bcast[4] * (unsigned long long)f.order.a_items(n.group);
                            unsigned long long v;
                            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(f.ctr + 1 + n.group) : "memory");
                            go = v >= target;
                            if (go) asm volatile("fence.proxy.async.global;" ::: "memory");
                        }
                        if (go) request(n, next);
                    }
                }
            }
        };
        const bool z_item = (it.phase == 0) == !INV;
        const MemHint<T> mem_a{0, l2_evict_last()};    // -> intermediate
        const MemHint<T> mem_b{0, l2_evict_first()};   // -> streaming output
        bool done;
        if (z_item) {
            if (it.phase == 0) done = zy_fed_tile<T, LOG2N, Z::LOG2E, TB, false, INV>(pz, it.tile, sm, mem_a, ok, after_gather);
            else if constexpr (SCALED) done = zy_fed_tile<T, LOG2N, Z::LOG2E, TB, false, INV>(pz, it.tile, sm, MemScaled<T, MemHint<T>>{mem_b, T(pz.scale)}, ok, after_gather);
            else done = zy_fed_tile<T, LOG2N, Z::LOG2E, TB, false, INV>(pz, it.tile, sm, mem_b, ok, after_gather);
        } else {
            if (it.phase == 0) done = zy_fed_tile<T, LOG2N, Z::LOG2E, TB, true, INV>(py, it.tile, sm, mem_a, ok, after_gather);
            else done = zy_fed_tile<T, LOG2N, Z::LOG2E, TB, true, INV>(py, it.tile, sm, mem_b, ok, after_gather);
        }
        if (!done) return false;
        ZY_STAMP(f, *slot, ZY_STORED);
        __syncthreads();  // every store of the item is issued before it counts
        zy_item_done<T, LOG2N, INV, false>(pz, py, f, *slot);
        ZY_STAMP(f, *slot, ZY_DONE);
        return true;
    }, ready);
}

// ---- batches of small cubic fields: one persistent launch per exec ------------------------------------------
// A batch of B fields of N^3 points (N = 32, 64), back to back, transformed in one launch as two phases per field:
//   plane items: the z lines and the y columns of PPI consecutive x-planes (4096 points), staged through shared memory
//                between the two axes;
//   slice items: the x lines of TB consecutive (y, z) columns (4096 points, rows N^2 apart), fft_c2c_kernel's tile code.
// Forward: phase A = plane items (caller's in -> caller's out), phase B = slice items (out -> out, in place).  Inverse, in
// the order of the unbatched plan (x, then y, then z): phase A = slice items (in -> out), phase B = plane items (out -> out,
// in place).  A phase-B item of field f needs every phase-A item of f; the work list is ZyOrder with one group per field,
// so every dependency has a lower ticket (zy_order.hpp) and the kernel runs the ticket loop of fft_zy_fused_kernel.  Each line
// runs FftCore<T, LOG2N, Shape::LOG2E> with the plan's twiddle table, as in the standalone passes: bit-identical results.
// L2 policy as in the fused z + y stage: phase A loads with evict_first and stores the intermediate with evict_last,
// phase B stores with evict_first; a field is read from HBM once and written once.
// TicketWork: one group per field (ctr[1 + f] counts field f), order.nx = fields, gpp = 1, na / nb items per field (filled in
// by the launcher), look-ahead in fields.
struct BatchSmall : TicketWork {
    const void* plane_in;      // plane items read here and write plane_out
    void* plane_out;
    const void* tw;            // exp(-2 pi i m / N), the plan's table
};
constexpr int BATCH_ERR_TIMEOUT = 201;  // value of the error flag when a batched-stage dependency wait timed out

template <typename T, int LOG2N>
struct BatchShape {
    static constexpr int LOG2E = Shape<T, LOG2N>::LOG2E, N = 1 << LOG2N, TPL = N >> LOG2E;
    static constexpr int POINTS = 4096;            // points of one work item
    static constexpr int THREADS = POINTS >> LOG2E;
    static constexpr int PPI = POINTS / (N * N);   // x-planes of a plane item
    static constexpr int TB = POINTS / N;          // z lines / y columns of a plane item, x columns of a slice item
    using CZ = CtaFft<T, LOG2N, LOG2E, TB, false>;
    using CY = CtaFft<T, LOG2N, LOG2E, TB, true>;
    static_assert(CZ::THREADS == THREADS && CY::THREADS == THREADS, "one CTA shape for both items");
    // staged planes: rows of N + TPL points, so that the z-line stores of the TPL threads of consecutive lines fall into
    // distinct banks
    static constexpr int RP = N + TPL;
    static constexpr size_t STAGE_BYTES = size_t(PPI) * N * RP * sizeof(cx<T>);
    static constexpr size_t TILE_BYTES = CZ::TILE_BYTES > CY::TILE_BYTES ? (CZ::TILE_BYTES > STAGE_BYTES ? CZ::TILE_BYTES : STAGE_BYTES)
                                                                         : (CY::TILE_BYTES > STAGE_BYTES ? CY::TILE_BYTES : STAGE_BYTES);
    static constexpr size_t SMEM_BYTES = TILE_BYTES + 48;  // + the ticket broadcast
};
constexpr bool batch_small_length(int log2n) { return log2n == 5 || log2n == 6; }

// One plane item: the 4096 points at src (PPI x-planes, [p][y][z]) -> dst.  Forward z then y; inverse y then z.
template <typename T, int LOG2N, bool INV, typename M>
__device__ __forceinline__ void batch_plane_item(const cx<T>* src, cx<T>* dst, const cx<T>* tw, cx<T>* sm, const M& mem) {
    using BS = BatchShape<T, LOG2N>;
    constexpr int N = BS::N, TPL = BS::TPL, TB = BS::TB, RP = BS::RP, E = BS::CZ::E;
    const int tid = threadIdx.x;
    const int jz = tid % TPL, tz = tid / TPL;          // z lines: thread jz of line tz = (plane, y)
    const int jy = tid / TB, ty = tid % TB;            // y columns: thread jy of column ty = (plane, z)
    const int py = ty / N, zy = ty % N;
    cx<T> v[E];
    if constexpr (!INV) {
        const cx<T>* q = src + tz * N + jz;
#pragma unroll
        for (int e = 0; e < E; ++e) v[e] = mem.ld(q + e * TPL);
        BS::CZ::template stages<0>(v, jz, tz, sm, tw);
        __syncthreads();  // every line's last gather is done: the exchange space becomes the staging buffer
#pragma unroll
        for (int e = 0; e < E; ++e) sm[tz * RP + jz + e * TPL] = v[BS::CZ::Core::final_slot(e)];
        __syncthreads();
#pragma unroll
        for (int e = 0; e < E; ++e) v[e] = sm[(py * N + jy + e * TPL) * RP + zy];
        __syncthreads();  // the staged planes are read before the first exchange overwrites them
        BS::CY::template stages<0>(v, jy, ty, sm, tw);
        cx<T>* o = dst + py * N * N + jy * N + zy;
#pragma unroll
        for (int e = 0; e < E; ++e) mem.st(o + e * TPL * N, v[BS::CY::Core::final_slot(e)]);
    } else {
        // re/im stay swapped between the two axes: the standalone passes swap on store and swap back on load
        const cx<T>* q = src + py * N * N + jy * N + zy;
#pragma unroll
        for (int e = 0; e < E; ++e) v[e] = cswap(mem.ld(q + e * TPL * N));
        BS::CY::template stages<0>(v, jy, ty, sm, tw);
        __syncthreads();
#pragma unroll
        for (int e = 0; e < E; ++e) sm[(py * N + jy + e * TPL) * RP + zy] = v[BS::CY::Core::final_slot(e)];
        __syncthreads();
#pragma unroll
        for (int e = 0; e < E; ++e) v[e] = sm[tz * RP + jz + e * TPL];
        __syncthreads();
        BS::CZ::template stages<0>(v, jz, tz, sm, tw);
        cx<T>* o = dst + tz * N + jz;
#pragma unroll
        for (int e = 0; e < E; ++e) mem.st(o + e * TPL, cswap(v[BS::CZ::Core::final_slot(e)]));
    }
}

// px: the slice items' view (A0 = fields, sA0 = N^3, n = x with sN = N^2, B = N^2; forward out -> out, inverse in -> out)
// SCALED: phase B (forward the slice items, inverse the plane items) scales its stores by px.scale; phase A's stores into
// the caller's output are intermediate and stay unscaled.
template <typename T, int LOG2N, bool INV, bool SCALED>
__global__ void __launch_bounds__(BatchShape<T, LOG2N>::THREADS, min_ctas_per_sm<T, BatchShape<T, LOG2N>::LOG2E>(BatchShape<T, LOG2N>::THREADS))
fft_batch_small_kernel(const __grid_constant__ KParams<SCALED> px, const __grid_constant__ BatchSmall f) {
    using BS = BatchShape<T, LOG2N>;
    constexpr int TB = BS::TB;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* no_tab = reinterpret_cast<unsigned long long*>(smem_raw);  // single-segment views need no tables
    volatile long long* bcast = reinterpret_cast<volatile long long*>(smem_raw + BS::TILE_BYTES);
    const cx<T>* plane_in = reinterpret_cast<const cx<T>*>(f.plane_in);
    cx<T>* plane_out = reinterpret_cast<cx<T>*>(f.plane_out);
    // the ticket loop of fft_zy_fused_kernel, with one group per field
    ticket_loop(f, bcast, BATCH_ERR_TIMEOUT, [&](const ZyItem& it, const volatile long long*) {
        const bool slice = (it.phase == 0) == INV;
        const MemHint<T> mem_a{l2_evict_first(), l2_evict_last()};   // streaming input -> intermediate
        const MemHint<T> mem_b{l2_evict_normal(), l2_evict_first()};  // intermediate -> streaming output
        if (slice) {
            if (it.phase == 0) c2c_tile<T, LOG2N, BS::LOG2E, TB, true, INV>(px, it.tile, sm, no_tab, no_tab, false, mem_a);
            else if constexpr (SCALED) c2c_tile<T, LOG2N, BS::LOG2E, TB, true, INV>(px, it.tile, sm, no_tab, no_tab, false, MemScaled<T, MemHint<T>>{mem_b, T(px.scale)});
            else c2c_tile<T, LOG2N, BS::LOG2E, TB, true, INV>(px, it.tile, sm, no_tab, no_tab, false, mem_b);
        } else {
            const long long off = it.tile * BS::POINTS;
            const cx<T>* tw = reinterpret_cast<const cx<T>*>(f.tw);
            if (it.phase == 0) batch_plane_item<T, LOG2N, INV>(plane_in + off, plane_out + off, tw, sm, mem_a);
            else if constexpr (SCALED) batch_plane_item<T, LOG2N, INV>(plane_in + off, plane_out + off, tw, sm, MemScaled<T, MemHint<T>>{mem_b, T(px.scale)});
            else batch_plane_item<T, LOG2N, INV>(plane_in + off, plane_out + off, tw, sm, mem_b);
        }
        // the item is stored and shared memory is free again before it counts
        __syncthreads();
        if (it.phase == 0 && threadIdx.x == 0) asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(f.ctr + 1 + it.group) : "memory");
    });
}

// ---- C2C TILED pass fed by TMA ----------------------------------------------------------------------------
// Same tile, same stages, but the N x TB input tile is fetched by the TMA engine (cp.async.bulk.tensor, SASS UTMALDG)
// straight into the tile buffer and announced through an mbarrier, instead of 16 LDG.128 per thread:
//   * the loads no longer pass through the LSU / L1TEX data pipe — the busiest unit of the register-fed kernel
//     (about half of its wavefronts are the 64-byte-row global accesses);
//   * no registers are tied to bytes in flight, so the kernel is persistent and the NEXT tile is requested as soon
//     as the last gather of the current tile has left the buffer: it lands while the last radix stage and the stores
//     run (and while the second resident CTA computes).
// Input view: single segment; described by a rank-4 tensor map (b, n, a1, a0) built by the launcher, box TB x 256.
// Output: either 16-byte stores from registers through any (segmented) view, or — `bulk_out`, blocked hand-over
// layouts whose rows per destination are adjacent — one cp.async.bulk (UBLKCP) per destination from the buffer.
// (TmaBar: above, with the fused z + y stage.)

// SCALED: every finished value is scaled by p.scale in registers, before the 16-byte stores or the staging for bulk_out.
template <typename T, int LOG2N, int LOG2E, int TB, bool INV, bool SCALED>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_c2c_tma_kernel(const __grid_constant__ KParams<SCALED> p, const __grid_constant__ CUtensorMap tm_in) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, true>;
    using Core = typename C::Core;
    using L = typename C::L;
    using LA = LineAccess<T, 1>;
    using TC = TileCoord<C, true, TB>;
    constexpr int E = C::E, TPL = C::TPL, N = C::N, NST = C::NST;
    static_assert(NST >= 2, "the TMA-fed kernel is for lines that exchange through shared memory");
    constexpr unsigned TILE_TX = unsigned(N) * TB * unsigned(sizeof(cx<T>));
    constexpr int ROWS_PER_OP = N < 256 ? N : 256;  // box height (a TMA box dimension is at most 256)
    constexpr int D0 = sizeof(T) == 8 ? 2 : 1;      // inner-dimension units per complex element (8-byte units)
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + MAXSEG;
    unsigned long long* bar = tab_out + MAXSEG;
    const long long ntiles = TC::num_tiles(p);
    const bool out_multi = p.out.nseg > 1;
    const bool bulk = p.bulk_out != 0;
    const int tid = threadIdx.x;
    auto finish = [&](cx<T> x) {  // the stored form of a finished value
        if constexpr (INV) x = cswap(x);
        if constexpr (SCALED) x = cscale<T>(x, T(p.scale));
        return x;
    };

    auto request = [&](long long tile) {  // one thread: arm the barrier and ask the TMA engine for the tile
        const TC tc(p, tile);
        const int b0 = (tc.b - tc.t) * D0;
        TmaBar::expect(bar, TILE_TX);
        const unsigned dst = unsigned(__cvta_generic_to_shared(sm));
        const unsigned mb = unsigned(__cvta_generic_to_shared(bar));
#pragma unroll
        for (int r = 0; r < N; r += ROWS_PER_OP)
            asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                         ::"r"(dst + unsigned(r) * TB * unsigned(sizeof(cx<T>))), "l"(&tm_in), "r"(mb), "r"(b0), "r"(r), "r"(tc.a1), "r"(tc.a0)
                         : "memory");
    };

    if (tid == 0) {
        TmaBar::init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0 && (long long)blockIdx.x < ntiles) request(blockIdx.x);
    unsigned parity = 0;

#pragma unroll 1
    for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const TC tc(p, tile);
        const int j = tc.j, t = tc.t;
        const long long next = tile + gridDim.x;
        if (out_multi && !bulk) LA::fill_table(p.out, tab_out, 0, tid, C::THREADS, tc.a0, tc.a1);
        if (bulk)
            for (int s = tid; s < p.out.nseg; s += C::THREADS) {
                const Seg& g = p.out.seg[s];
                cx<T>* q = reinterpret_cast<cx<T>*>(g.base) + (tc.a0 * g.sA0 + tc.a1 * g.sA1 - (long long)g.n0 * p.out.sN);
                tab_out[s] = reinterpret_cast<unsigned long long>(q);
            }
        if (!TmaBar::wait(bar, parity)) __trap();
        parity ^= 1;

        cx<T> v[E];
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const cx<T> x = sm[(j + e * TPL) * TB + t];  // dense [n][TB], as the TMA engine wrote it
            v[e] = INV ? cswap(x) : x;
        }
        __syncthreads();  // everyone has its inputs: the buffer turns into the (padded) exchange space; tables visible

        // the stages of CtaFft::stages, with a hook where the buffer is free again (after the last gather)
        auto run = [&](auto self, auto st_tag) -> void {
            constexpr int ST = decltype(st_tag)::value;
            Core::template stage_compute<ST>(v, j, reinterpret_cast<const cx<T>*>(p.tw));
            if constexpr (ST + 1 < NST) {
                if constexpr (ST > 0) __syncthreads();
                cx<T>* q = sm + L::idx(Core::template scatter_base<ST>(j), t);
#pragma unroll
                for (int e = 0; e < E; ++e) q[L::off(Core::template scatter_off<ST>(e))] = v[e];
                __syncthreads();
                C::gather(v, sm, j, t);
                if constexpr (ST + 2 == NST) {
                    if (!bulk) {
                        // generic-proxy reads of the buffer are ordered before the async-proxy write of the next tile
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        __syncthreads();
                        if (tid == 0 && next < ntiles) request(next);
                    }
                }
                self(self, std::integral_constant<int, ST + 1>{});
            }
        };
        run(run, std::integral_constant<int, 0>{});

        if (!bulk) {
            if (tc.valid) {
                const LA out(p.out, tab_out, 0, tc.a0, tc.a1, tc.b);
                if (!out.multi) {
                    const long long step = (long long)TPL * p.out.sN;
                    cx<T>* q = out.p0 + (long long)j * p.out.sN;
#pragma unroll
                    for (int e = 0; e < E; ++e) {
                        st_elem<T>(q, finish(v[Core::final_slot(e)]));
                        q += step;
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < E; ++e) st_elem<T>(out.at(j + e * TPL), finish(v[Core::final_slot(e)]));
                }
            }
            if (out_multi) __syncthreads();  // the segment table is rewritten by the next tile
        } else {
            __syncthreads();  // last gather finished everywhere: stage the finished tile, natural order [n][TB]
#pragma unroll
            for (int e = 0; e < E; ++e) sm[(j + e * TPL) * TB + t] = finish(v[Core::final_slot(e)]);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (tid == 0) {
                for (int s = 0; s < p.out.nseg; ++s) {
                    const int n0 = p.out.nseg > 1 ? p.out.seg[s].n0 : 0;
                    const int n1 = (s + 1 < p.out.nseg) ? p.out.seg[s + 1].n0 : N;
                    const unsigned bytes = unsigned(n1 - n0) * TB * unsigned(sizeof(cx<T>));
                    if (!bytes) continue;
                    const unsigned src = unsigned(__cvta_generic_to_shared(sm + n0 * TB));
                    const unsigned long long dst = tab_out[s] + (unsigned long long)n0 * TB * sizeof(cx<T>);
                    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
                }
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // the buffer has been read: it may be refilled
                if (next < ntiles) request(next);
            }
            __syncthreads();  // tab_out is rewritten by the next tile
        }
    }
    if (bulk && tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // all bulk stores performed before exit
}


// complex value from another lane of the warp
template <typename T>
__device__ __forceinline__ cx<T> shfl_cx(cx<T> v, int src_lane) {
    return cx<T>{__shfl_sync(0xffffffffu, v.x, src_lane), __shfl_sync(0xffffffffu, v.y, src_lane)};
}

// ---- R2C pass (CONTIG): real line of 2M points -> M+1 complex points ------------------------------------
// The real line is read as M complex points z[m] = x[2m] + i x[2m+1], transformed with the length-M
// core and split into even/odd spectra in shared memory:  X[k] = Xe[k] + W_2M^k Xo[k].
// PADDED (P = FftPadded): the pairs m >= p.ld_lo read as zero, the points k >= p.st_lo are not stored; the scale is
// p.scale at run time.
// S: the stored element, of both sides (the real side in pairs: cx16<H> holds two 16-bit reals).
// WEIGHTED (P = FftPadded with p.w): X[k] times p.w[k] as it is stored.
template <typename T, int LOG2M, int LOG2E, int TB, bool SCALED, bool PADDED, typename P, typename S = cx<T>, bool WEIGHTED = false>
__device__ __forceinline__ void r2c_lines(const P& p) {
    using C = CtaFft<T, LOG2M, LOG2E, TB, false>;
    using LA = LineAccess<T, C::LINES, S>;
    constexpr int E = C::E, TPL = C::TPL, M = C::N, NST = C::NST;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const TileCoord<C, false, TB> tc(p);
    const int j = tc.j, t = tc.t;
    const bool valid = tc.valid;
    if (p.out.nseg > 1) {
        LA::fill_table(p.out, tab_out, t, j, TPL, tc.a0, tc.a1);
        __syncthreads();
    }
    const LA in(p.in, tab_in, t, tc.a0, tc.a1, 0);
    const LA out(p.out, tab_out, t, tc.a0, tc.a1, 0);

    cx<T> v[E];
    if (valid) {
        const S* q = in.p0 + j;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            if constexpr (PADDED) v[e] = j + e * TPL < p.ld_lo ? ld_elem<T>(q + e * TPL) : cx<T>{T(0), T(0)};
            else v[e] = ld_elem<T>(q + e * TPL);
        }
    } else {
#pragma unroll
        for (int e = 0; e < E; ++e) v[e] = cx<T>{T(0), T(0)};
    }
    C::template stages<0>(v, j, t, sm, reinterpret_cast<const cx<T>*>(p.tw));

    const cx<T>* tw2 = reinterpret_cast<const cx<T>*>(p.tw2);
    // (A shuffle-based split like fft_c2r_kernel's would need 16 extra twiddle multiplies per thread in this direction
    // to save one shared-memory round trip; the forward kernel keeps the shared-memory split, not yet compared on the
    // H100.)
    // Z in natural order -> shared memory
    if constexpr (NST > 1) C::sync(t);
#pragma unroll
    for (int e = 0; e < E; ++e) sm[C::sidx(j + e * TPL, t)] = v[C::Core::final_slot(e)];
    C::sync(t);

    auto emit = [&](int k) {
        const int kk = (M - k) & (M - 1);
        const cx<T> zk = sm[C::sidx(k, t)], zp = cconj(sm[C::sidx(kk, t)]);
        const cx<T> xe = cx<T>{T(0.5) * (zk.x + zp.x), T(0.5) * (zk.y + zp.y)};
        const cx<T> d = csub(zk, zp);
        const cx<T> xo = cx<T>{T(0.5) * d.y, T(-0.5) * d.x};  // -i/2 * d
        const cx<T> tt = cmul(ld_tw(tw2, k), xo);
        if (valid) {
            if constexpr (WEIGHTED) {
                static_assert(PADDED, "the weighted R2C pass is the padded twin's");
                const cx<T>* w = reinterpret_cast<const cx<T>*>(p.w);
                const MemRtScaled<T> mem{p.scale != 1.0, T(p.scale)};
                if (k < p.st_lo) mem.st(out.at1(k), cmul(cadd(xe, tt), ld_tw(w, k)));
                if (M - k < p.st_lo) mem.st(out.at1(M - k), cmul(cconj(csub(xe, tt)), ld_tw(w, M - k)));
            } else if constexpr (PADDED) {
                const MemRtScaled<T> mem{p.scale != 1.0, T(p.scale)};
                if (k < p.st_lo) mem.st(out.at1(k), cadd(xe, tt));
                if (M - k < p.st_lo) mem.st(out.at1(M - k), cconj(csub(xe, tt)));
            } else if constexpr (SCALED) {
                st_elem<T>(out.at1(k), cscale<T>(cadd(xe, tt), T(p.scale)));
                st_elem<T>(out.at1(M - k), cscale<T>(cconj(csub(xe, tt)), T(p.scale)));
            } else {
                st_elem<T>(out.at1(k), cadd(xe, tt));
                st_elem<T>(out.at1(M - k), cconj(csub(xe, tt)));
            }
        }
    };
#pragma unroll
    for (int e = 0; e < E / 2; ++e) emit(j + e * TPL);
    if (j == 0) emit(M / 2);
}

// S = cx16<H>, T = float: the R2C z pass of 16-bit plans, the f32 line with cx16<H> loads and stores (fft_c2c_kernel)
template <typename T, typename S, int LOG2M, int LOG2E, int TB, bool SCALED>
__global__ void __launch_bounds__((1 << (LOG2M - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2M - LOG2E)) * TB))
fft_r2c_kernel(const __grid_constant__ KParams<SCALED> p) {
    r2c_lines<T, LOG2M, LOG2E, TB, SCALED, false, KParams<SCALED>, S>(p);
}

// padded twin of fft_r2c_kernel: reads the pairs m < p.ld_lo (p.ld_hi = M), keeps the points k < p.st_lo (p.st_hi = M + 1);
// with WEIGHTED its weighted twin (p.w)
template <typename T, int LOG2M, int LOG2E, int TB, bool WEIGHTED>
__global__ void __launch_bounds__((1 << (LOG2M - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2M - LOG2E)) * TB))
fft_r2c_padded_kernel(const __grid_constant__ FftPadded p) {
    r2c_lines<T, LOG2M, LOG2E, TB, false, true, FftPadded, cx<T>, WEIGHTED>(p);
}

// ---- C2R pass (CONTIG): M+1 complex points -> real line of 2M points, unnormalised -----------------------
// PADDED (P = FftPadded): the points k >= p.ld_lo read as zero, their partner loads X[M - k] as well; the pairs
// m >= p.st_lo are not stored; the scale is p.scale at run time.
// WEIGHTED (P = FftPadded with p.w): X[k] and its partner X[M - k] times p.w at their index as they are loaded.
template <typename T, int LOG2M, int LOG2E, int TB, bool SCALED, bool PADDED, typename P, typename S = cx<T>, bool WEIGHTED = false>
__device__ __forceinline__ void c2r_lines(const P& p) {
    using C = CtaFft<T, LOG2M, LOG2E, TB, false>;
    using LA = LineAccess<T, C::LINES, S>;
    constexpr int E = C::E, TPL = C::TPL, M = C::N;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const TileCoord<C, false, TB> tc(p);
    const int j = tc.j, t = tc.t;
    const bool valid = tc.valid;
    if (p.in.nseg > 1) {
        LA::fill_table(p.in, tab_in, t, j, TPL, tc.a0, tc.a1);
        __syncthreads();
    }
    const LA in(p.in, tab_in, t, tc.a0, tc.a1, 0);
    const LA out(p.out, tab_out, t, tc.a0, tc.a1, 0);

    const cx<T>* tw2 = reinterpret_cast<const cx<T>*>(p.tw2);
    cx<T> v[E];
    if constexpr (TPL <= 32) {
        // The line lives in one warp (TPL lanes): thread j loads X[j + e*TPL] (coalesced), fetches the partners X[M - k] from lane TPL - j
        // (slot E-1-e; lane 0: its own slot E-e, and X[M] for k = 0) with one shuffle each, and builds
        //   Z[k] = (X[k] + conj X[M-k]) + i conj(W_2M^k) (X[k] - conj X[M-k])
        // directly in the register layout the first stage expects — no staging through shared memory.
        cx<T> xk[E];
        cx<T> xM{T(0), T(0)};
        if (valid) {
            if constexpr (PADDED) {
#pragma unroll
                for (int e = 0; e < E; ++e) xk[e] = j + e * TPL < p.ld_lo ? ld_elem<T>(in.at1(j + e * TPL)) : cx<T>{T(0), T(0)};
                if (j == 0 && M < p.ld_lo) xM = ld_elem<T>(in.at1(M));
                if constexpr (WEIGHTED) {
                    const cx<T>* w = reinterpret_cast<const cx<T>*>(p.w);
#pragma unroll
                    for (int e = 0; e < E; ++e)
                        if (j + e * TPL < p.ld_lo) xk[e] = cmul(xk[e], ld_tw(w, j + e * TPL));
                    if (j == 0 && M < p.ld_lo) xM = cmul(xM, ld_tw(w, M));
                }
            } else {
#pragma unroll
                for (int e = 0; e < E; ++e) xk[e] = ld_elem<T>(in.at1(j + e * TPL));
                if (j == 0) xM = ld_elem<T>(in.at1(M));
            }
        } else {
#pragma unroll
            for (int e = 0; e < E; ++e) xk[e] = cx<T>{T(0), T(0)};
        }
        const int lane = threadIdx.x & 31;
        const int src = (lane & ~(TPL - 1)) + ((TPL - j) & (TPL - 1));
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const cx<T> other = shfl_cx<T>(xk[E - 1 - e], src);
            const cx<T> self = e == 0 ? xM : xk[(E - e) & (E - 1)];
            const cx<T> xm = cconj(j == 0 ? self : other);
            const int k = j + e * TPL;
            cx<T> wc;  // conj(W_2M^k)
            if (2 * k <= M) wc = cconj(ld_tw(tw2, k));
            else { const cx<T> u = ld_tw(tw2, M - k); wc = cx<T>{-u.x, -u.y}; }
            const cx<T> xe = cadd(xk[e], xm);
            const cx<T> xo = cmul(wc, csub(xk[e], xm));
            // stored with re/im swapped: the inverse transform is run as swap(fwd(swap(.)))
            v[e] = cswap(cx<T>{xe.x - xo.y, xe.y + xo.x});
        }
    } else {
    // Z[k] = (X[k] + conj X[M-k]) + i * conj(W^k) * (X[k] - conj X[M-k]);  Z[M-k] = conj(Xe' - i Xo')
    auto build = [&](int k) {
        cx<T> xk{T(0), T(0)}, xm{T(0), T(0)};
        if (valid) {
            if constexpr (WEIGHTED) {
                const cx<T>* w = reinterpret_cast<const cx<T>*>(p.w);
                if (k < p.ld_lo) xk = cmul(ld_elem<T>(in.at1(k)), ld_tw(w, k));
                if (M - k < p.ld_lo) xm = cconj(cmul(ld_elem<T>(in.at1(M - k)), ld_tw(w, M - k)));
            } else if constexpr (PADDED) {
                if (k < p.ld_lo) xk = ld_elem<T>(in.at1(k));
                if (M - k < p.ld_lo) xm = cconj(ld_elem<T>(in.at1(M - k)));
            } else {
                xk = ld_elem<T>(in.at1(k));
                xm = cconj(ld_elem<T>(in.at1(M - k)));
            }
        }
        const cx<T> xe = cadd(xk, xm);
        const cx<T> xo = cmul(cconj(ld_tw(tw2, k)), csub(xk, xm));
        // stored with re/im swapped: the inverse transform is run as swap(fwd(swap(.)))
        sm[C::sidx(k, t)] = cswap(cx<T>{xe.x - xo.y, xe.y + xo.x});
        if (k != 0) sm[C::sidx(M - k, t)] = cswap(cx<T>{xe.x + xo.y, -(xe.y - xo.x)});
    };
#pragma unroll
    for (int e = 0; e < E / 2; ++e) build(j + e * TPL);
    if (j == 0) build(M / 2);
    C::sync(t);
    C::gather(v, sm, j, t);
    if constexpr (C::NST > 1) C::sync(t);
    }
    C::template stages<0>(v, j, t, sm, reinterpret_cast<const cx<T>*>(p.tw));
    if (valid) {
        S* q = out.p0 + j;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            if constexpr (PADDED) {
                if (j + e * TPL < p.st_lo) MemRtScaled<T>{p.scale != 1.0, T(p.scale)}.st(q + e * TPL, cswap(v[C::Core::final_slot(e)]));
            }
            else if constexpr (SCALED) st_elem<T>(q + e * TPL, cscale<T>(cswap(v[C::Core::final_slot(e)]), T(p.scale)));
            else st_elem<T>(q + e * TPL, cswap(v[C::Core::final_slot(e)]));
        }
    }
}

// S = cx16<H>, T = float: the C2R z pass of 16-bit plans, the f32 line with cx16<H> loads and stores (fft_c2c_kernel)
template <typename T, typename S, int LOG2M, int LOG2E, int TB, bool SCALED>
__global__ void __launch_bounds__((1 << (LOG2M - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2M - LOG2E)) * TB))
fft_c2r_kernel(const __grid_constant__ KParams<SCALED> p) {
    c2r_lines<T, LOG2M, LOG2E, TB, SCALED, false, KParams<SCALED>, S>(p);
}

// padded twin of fft_c2r_kernel: the points k >= p.ld_lo are zero (p.ld_hi = M + 1), the pairs m >= p.st_lo are not stored
// (p.st_hi = M); with WEIGHTED its weighted twin (p.w)
template <typename T, int LOG2M, int LOG2E, int TB, bool WEIGHTED>
__global__ void __launch_bounds__((1 << (LOG2M - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2M - LOG2E)) * TB))
fft_c2r_padded_kernel(const __grid_constant__ FftPadded p) {
    c2r_lines<T, LOG2M, LOG2E, TB, false, true, FftPadded, cx<T>, WEIGHTED>(p);
}

// ---- Bluestein pass: C2C lines of any length n through two transforms of length M = 2^LOG2M >= 2n - 1 ----------------
// X_k = c_k * IDFT_M(DFT_M(y) * K^)_k with c_k = exp(-pi i k^2 / n), y_k = x_k c_k (k < n, 0 up to M), and K^ the M-point
// spectrum of the conjugate chirp, divided by M (host tables, bluestein.hpp).  Both transforms are CtaFft's stages on the
// tile of the power-of-two kernels; the inverse DFT_M is swap(DFT_M(swap(.))), and the inverse direction swaps re/im on
// load and store as every kernel here does, so only forward tables exist.  One CTA per tile: every CTA reads all of its
// points before it stores, and tiles are disjoint, so out == in works.  The parameters of the other kernels are unchanged.
struct FftBluestein : FftParams {
    int n;              // line length
    const void* chirp;  // c_k, k < n
    const void* kspec;  // K^_m, m < M
    double scale;       // output scale, applied when != 1 (rounded to the kernel's precision once)
    const void* w;      // weighted passes (dfft_plan_set_weights, WEIGHTED): w[k], k < n, multiplies X_k forward as it is
                        // stored and x_k inverse as it is loaded; else null
};

template <typename T, int LOG2M, int LOG2E, int TB, bool TILED, bool INV, bool WEIGHTED>
__device__ __forceinline__ void bluestein_lines(const FftBluestein& p) {
    using C = CtaFft<T, LOG2M, LOG2E, TB, TILED>;
    using LA = LineAccess<T, C::LINES>;
    using TC = TileCoord<C, TILED, TB>;
    constexpr int E = C::E, TPL = C::TPL;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const TC tc(p, blockIdx.x);
    const int j = tc.j, t = tc.t, n = p.n;
    if (p.in.nseg > 1 || p.out.nseg > 1) {
        const int line = TILED ? 0 : t;
        const int lane = TILED ? int(threadIdx.x) : j;
        const int lanes = TILED ? C::THREADS : TPL;
        LA::fill_table(p.in, tab_in, line, lane, lanes, tc.a0, tc.a1);
        LA::fill_table(p.out, tab_out, line, lane, lanes, tc.a0, tc.a1);
        __syncthreads();
    }
    const LA in(p.in, tab_in, TILED ? 0 : t, tc.a0, tc.a1, tc.b);
    const LA out(p.out, tab_out, TILED ? 0 : t, tc.a0, tc.a1, tc.b);
    const cx<T>* chirp = reinterpret_cast<const cx<T>*>(p.chirp);
    const cx<T>* kspec = reinterpret_cast<const cx<T>*>(p.kspec);
    const cx<T>* tw = reinterpret_cast<const cx<T>*>(p.tw);

    // y = x * c, zero-padded to M
    cx<T> v[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int k = j + e * TPL;
        v[e] = cx<T>{T(0), T(0)};
        if (tc.valid && k < n) {
            cx<T> x = ld_elem<T>(TILED ? in.at(k) : in.at1(k));
            if constexpr (WEIGHTED && INV) x = cmul(x, ld_tw(reinterpret_cast<const cx<T>*>(p.w), k));
            v[e] = cmul(INV ? cswap(x) : x, ld_tw(chirp, k));
        }
    }
    C::template stages<0>(v, j, t, sm, tw);
    // Y[j + e*TPL] sits in slot final_slot(e); the second transform takes it in slot e, pre-swapped for the inverse DFT
    cx<T> z[E];
#pragma unroll
    for (int e = 0; e < E; ++e) z[e] = cswap(cmul(v[C::Core::final_slot(e)], ld_tw(kspec, j + e * TPL)));
    if constexpr (C::NST > 1) C::sync(t);  // the first transform's last gather is done before the second's first scatter
    C::template stages<0>(z, j, t, sm, tw);

    const bool scaled = p.scale != 1.0;
    const T s = T(p.scale);
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int k = j + e * TPL;
        if (tc.valid && k < n) {
            cx<T> x = cmul(ld_tw(chirp, k), cswap(z[C::Core::final_slot(e)]));
            if (INV) x = cswap(x);
            if constexpr (WEIGHTED && !INV) x = cmul(x, ld_tw(reinterpret_cast<const cx<T>*>(p.w), k));
            if (scaled) x = cscale<T>(x, s);
            st_elem<T>(TILED ? out.at(k) : out.at1(k), x);
        }
    }
}

template <typename T, int LOG2M, int LOG2E, int TB, bool TILED, bool INV, bool WEIGHTED>
__global__ void __launch_bounds__((1 << (LOG2M - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2M - LOG2E)) * TB))
fft_bluestein_kernel(const __grid_constant__ FftBluestein p) {
    bluestein_lines<T, LOG2M, LOG2E, TB, TILED, INV, WEIGHTED>(p);
}

// ---- real-to-real pass: DCT-II / DCT-III, DST-II / DST-III and R2HC / HC2R of real N-point lines ------------------------
// Two real lines a, b are packed into one complex N-point line (r2r.hpp) and transformed by CtaFft's stages on the tile of
// the power-of-two kernels; no half-length core.  The views count in reals (LineAccess<T, ., T>).
//   CONTIG: the pair (2L, 2L+1) of the flattened (a0, a1) line order takes line slot L of the tile, TB slots per CTA.
//   TILED:  the columns (2c, 2c+1) of the contiguous dimension take column c of the tile: a tile is N x 2 TB reals.
// An odd count gives the last line or column a zero partner, whose results are not stored.
// Forward: the permuted loads reach their reals straight from global memory (the two halves of a sector are read by two
// instructions of the same warp, the second from L1); after the stages Z goes through shared memory once, so that point k
// meets Z[N-k].  Inverse: X[k] and X[N-k] are both loaded from global memory and Z is built in registers; the stores are
// permuted.  One CTA per tile and every load before any store, so out == in works.  A scale != 1 multiplies the final
// stores (__dmul_rn / __fmul_rn: the scaled output is the unscaled one times s, bit for bit).
struct FftR2r : FftParams {
    const void* w;  // w_k = exp(-i pi k / 2N), k <= N (the R2C table of length 2N: Tables::get_tw2(log2 N + 1))
    int dst;        // 0 DCT, 1 DST
    double scale;   // output scale, applied when != 1 (rounded to the kernel's precision once)
};

template <typename T, int LOG2N, int LOG2E, int TB, bool TILED>
struct R2rShape {
    using C = CtaFft<T, LOG2N, LOG2E, TB, TILED>;
    static constexpr int LINES = TILED ? 1 : 2 * TB;  // real lines with their own segment table
    static constexpr size_t SMEM_BYTES = C::TILE_BYTES + size_t(2) * LINES * MAXSEG * sizeof(unsigned long long);
    static_assert(SMEM_BYTES <= 227 * 1024, "R2R tile does not fit the shared memory of a CTA");
};

template <typename T>
__device__ __forceinline__ T rscale(T v, T s) {
    if constexpr (sizeof(T) == 8) return __dmul_rn(v, s);
    else return __fmul_rn(v, s);
}

// reals q[0] and (second) q[1]: one 2-element access when q is aligned to it, two scalar ones otherwise (odd strides)
template <typename T>
__device__ __forceinline__ void ld_pair(const T* q, bool second, T& a, T& b) {
    if (second && (reinterpret_cast<unsigned long long>(q) & (2 * sizeof(T) - 1)) == 0) {
        const cx<T> r = ld_elem<T>(reinterpret_cast<const cx<T>*>(q));
        a = r.x; b = r.y;
    } else {
        a = q[0];
        b = second ? q[1] : T(0);
    }
}
template <typename T>
__device__ __forceinline__ void st_pair(T* q, bool second, T a, T b) {
    if (second && (reinterpret_cast<unsigned long long>(q) & (2 * sizeof(T) - 1)) == 0) {
        st_elem<T>(reinterpret_cast<cx<T>*>(q), cx<T>{a, b});
    } else {
        q[0] = a;
        if (second) q[1] = b;
    }
}

// The body of both R2R kernels.  HC: R2HC / HC2R (r2r.hpp) — natural order, no w_k and no sign flips; p.w and p.dst are
// not read.  A compile-time mode keeps the R2HC branches out of the DCT / DST instantiations (and their registers).
template <typename T, int LOG2N, int LOG2E, int TB, bool TILED, bool INV, bool HC>
__device__ __forceinline__ void r2r_pass(const FftR2r& p) {
    using RS = R2rShape<T, LOG2N, LOG2E, TB, TILED>;
    using C = typename RS::C;
    using LA = LineAccess<T, RS::LINES, T>;
    constexpr int E = C::E, TPL = C::TPL, N = C::N;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + RS::LINES * MAXSEG;
    const int tid = threadIdx.x;
    // line a and its partner b: (a0, a1) of each and whether it exists; TILED: b is column `col` + 1 of the same row
    int j, t, a0a, a1a, a0b, a1b, col = 0;
    bool va, vb;
    if constexpr (TILED) {
        t = tid % TB; j = tid / TB;
        const int nbt = ((p.B + 1) / 2 + TB - 1) / TB;  // tiles of TB column pairs
        const int bt = int(blockIdx.x % unsigned(nbt)), a = int(blockIdx.x / unsigned(nbt));
        a1a = a1b = a % p.A1;
        a0a = a0b = a / p.A1;
        col = 2 * (bt * TB + t);
        va = col < p.B;
        vb = col + 1 < p.B;
    } else {
        j = tid % TPL; t = tid / TPL;
        const long long lines = (long long)p.A0 * p.A1;
        const long long la = 2 * ((long long)blockIdx.x * TB + t), lb = la + 1;
        va = la < lines;
        vb = lb < lines;
        a1a = int(la % p.A1); a0a = int(la / p.A1);
        a1b = int(lb % p.A1); a0b = int(lb / p.A1);
    }
    if (p.in.nseg > 1 || p.out.nseg > 1) {
        if constexpr (TILED) {
            LA::fill_table(p.in, tab_in, 0, tid, C::THREADS, a0a, a1a);
            LA::fill_table(p.out, tab_out, 0, tid, C::THREADS, a0a, a1a);
        } else {
            LA::fill_table(p.in, tab_in, 2 * t, j, TPL, a0a, a1a);
            LA::fill_table(p.in, tab_in, 2 * t + 1, j, TPL, a0b, a1b);
            LA::fill_table(p.out, tab_out, 2 * t, j, TPL, a0a, a1a);
            LA::fill_table(p.out, tab_out, 2 * t + 1, j, TPL, a0b, a1b);
        }
        __syncthreads();
    }
    // TILED: line b is the next real of line a's row, so one access object serves both
    const LA ina(p.in, tab_in, TILED ? 0 : 2 * t, a0a, a1a, col), outa(p.out, tab_out, TILED ? 0 : 2 * t, a0a, a1a, col);
    const LA inb(p.in, tab_in, TILED ? 0 : 2 * t + 1, a0b, a1b, 0), outb(p.out, tab_out, TILED ? 0 : 2 * t + 1, a0b, a1b, 0);
    const cx<T>* w = reinterpret_cast<const cx<T>*>(p.w);
    const cx<T>* tw = reinterpret_cast<const cx<T>*>(p.tw);
    const int dst = p.dst;
    const bool scaled = p.scale != 1.0;
    const T s = T(p.scale);
    // reals m of both lines (0 for a missing line)
    auto load2 = [&](int m, T& a, T& b) {
        a = T(0); b = T(0);
        if constexpr (TILED) {
            if (va) ld_pair<T>(ina.at(m), vb, a, b);
        } else {
            if (va) a = *ina.at1(m);
            if (vb) b = *inb.at1(m);
        }
    };
    auto store2 = [&](int m, T a, T b) {
        if (scaled) { a = rscale<T>(a, s); b = rscale<T>(b, s); }
        if constexpr (TILED) {
            if (va) st_pair<T>(outa.at(m), vb, a, b);
        } else {
            if (va) *outa.at1(m) = a;
            if (vb) *outb.at1(m) = b;
        }
    };

    cx<T> v[E];
    if constexpr (HC && !INV) {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            T a, b;
            load2(j + e * TPL, a, b);
            v[e] = cx<T>{a, b};
        }
        C::template stages<0>(v, j, t, sm, tw);
        if constexpr (C::NST > 1) C::sync(t);
#pragma unroll
        for (int e = 0; e < E; ++e) sm[C::sidx(j + e * TPL, t)] = v[C::Core::final_slot(e)];
        C::sync(t);
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            const cx<T> x = r2hc_split<T>(sm[C::sidx(k, t)], sm[C::sidx((N - k) & (N - 1), t)], k, N);
            store2(k, x.x, x.y);
        }
    } else if constexpr (HC) {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            const int nk = r2hc_in_nk(k, N);
            T ak, bk, am = T(0), bm = T(0);
            load2(k, ak, bk);
            if (nk >= 0) load2(nk, am, bm);
            v[e] = cswap(r2hc_build<T>(ak, am, bk, bm, k, N));
        }
        C::template stages<0>(v, j, t, sm, tw);
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const cx<T> z = cswap(v[C::Core::final_slot(e)]);
            store2(j + e * TPL, z.x, z.y);
        }
    } else if constexpr (!INV) {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int m = r2r_perm(j + e * TPL, N);
            const T sg = r2r_sign<T>(m, dst);
            T a, b;
            load2(m, a, b);
            v[e] = cx<T>{sg * a, sg * b};
        }
        C::template stages<0>(v, j, t, sm, tw);
        // Z in natural order -> shared memory, then point k with Z[N-k]
        if constexpr (C::NST > 1) C::sync(t);
#pragma unroll
        for (int e = 0; e < E; ++e) sm[C::sidx(j + e * TPL, t)] = v[C::Core::final_slot(e)];
        C::sync(t);
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            const cx<T> x = r2r_split<T>(sm[C::sidx(k, t)], sm[C::sidx((N - k) & (N - 1), t)], ld_tw(w, k));
            store2(r2r_out_index(k, N, dst), x.x, x.y);
        }
    } else {
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const int k = j + e * TPL;
            const int nk = r2r_in_nk(k, N, dst);
            T ak, bk, am = T(0), bm = T(0);
            load2(r2r_in_k(k, N, dst), ak, bk);
            if (nk >= 0) load2(nk, am, bm);
            // stored with re/im swapped: the inverse transform is run as swap(fwd(swap(.)))
            v[e] = cswap(r2r_build<T>(ak, am, bk, bm, ld_tw(w, k)));
        }
        C::template stages<0>(v, j, t, sm, tw);
#pragma unroll
        for (int e = 0; e < E; ++e) {
            const cx<T> z = cswap(v[C::Core::final_slot(e)]);
            const int m = r2r_perm(j + e * TPL, N);
            const T sg = r2r_sign<T>(m, dst);
            store2(m, sg * z.x, sg * z.y);
        }
    }
}

template <typename T, int LOG2N, int LOG2E, int TB, bool TILED, bool INV>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_r2r_kernel(const __grid_constant__ FftR2r p) {
    r2r_pass<T, LOG2N, LOG2E, TB, TILED, INV, false>(p);
}

// R2HC forward, HC2R inverse: the DCT / DST kernel's tile, pairing, views and scale
template <typename T, int LOG2N, int LOG2E, int TB, bool TILED, bool INV>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_r2hc_kernel(const __grid_constant__ FftR2r p) {
    r2r_pass<T, LOG2N, LOG2E, TB, TILED, INV, true>(p);
}

// ---- type-I real-to-real pass: DCT-I (L = N + 1 reals per line) and DST-I (L = N - 1) -------------------------------------
// One real line per complex N-point line of the tile (r2r.hpp): point m loads e_{2m} and e_{2m+1} of the line's 2N-point
// extension, CtaFft's stages transform z, and the R2C split with the 2N-point table (FftR2r::w = W^k = exp(-i pi k / N),
// k <= N/2: Tables::get_tw2(log2 N)) gives E_k, of which y takes the real part (DCT-I) or minus the imaginary part (DST-I).
// p.dst picks the kind, p.inverse is not read: the transform is its own inverse.  The views count in reals.
//   CONTIG: TB real lines per CTA, one per line slot.
//   TILED:  one real column per tile column (TB columns: the wide tile of the length where shared memory allows it).
// The mirrored loads reach their reals straight from global memory, as the DCT-II pass's permuted loads do; the second
// read of a sector is meant to hit L1 (a design choice, not a measurement).  After the stages Z goes through shared memory
// once; the thread of point k <= N/2 splits Z[k] with Z[N-k] and stores the outputs of E_k and E_{N-k}.  One CTA per tile
// and every load before any store, so out == in works.  A scale != 1 multiplies the stores (__dmul_rn / __fmul_rn: the
// scaled output is the unscaled one times s, bit for bit).
template <typename T, int LOG2N, int LOG2E, int TB, bool TILED>
__global__ void __launch_bounds__((1 << (LOG2N - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2N - LOG2E)) * TB))
fft_r2r1_kernel(const __grid_constant__ FftR2r p) {
    using C = CtaFft<T, LOG2N, LOG2E, TB, TILED>;
    using LA = LineAccess<T, C::LINES, T>;
    constexpr int E = C::E, TPL = C::TPL, N = C::N;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const TileCoord<C, TILED, TB> tc(p);
    const int j = tc.j, t = tc.t;
    if (p.in.nseg > 1 || p.out.nseg > 1) {
        // TILED: one table per CTA, CONTIG: one per line (as in c2c_tile)
        const int line = TILED ? 0 : t, lane = TILED ? int(threadIdx.x) : j, lanes = TILED ? C::THREADS : TPL;
        LA::fill_table(p.in, tab_in, line, lane, lanes, tc.a0, tc.a1);
        LA::fill_table(p.out, tab_out, line, lane, lanes, tc.a0, tc.a1);
        __syncthreads();
    }
    const LA in(p.in, tab_in, TILED ? 0 : t, tc.a0, tc.a1, tc.b), out(p.out, tab_out, TILED ? 0 : t, tc.a0, tc.a1, tc.b);
    const int dst = p.dst;
    auto ext = [&](int i) -> T {  // e_i
        bool neg;
        const int m = r2r1_ext(i, N, dst, neg);
        if (m < 0) return T(0);
        T x;
        if constexpr (TILED) x = *in.at(m);
        else x = *in.at1(m);
        return neg ? -x : x;
    };
    cx<T> v[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int m = j + e * TPL;
        v[e] = tc.valid ? cx<T>{ext(2 * m), ext(2 * m + 1)} : cx<T>{T(0), T(0)};
    }
    C::template stages<0>(v, j, t, sm, reinterpret_cast<const cx<T>*>(p.tw));
    // Z in natural order -> shared memory, then point k with Z[N-k]
    if constexpr (C::NST > 1) C::sync(t);
#pragma unroll
    for (int e = 0; e < E; ++e) sm[C::sidx(j + e * TPL, t)] = v[C::Core::final_slot(e)];
    C::sync(t);
    if (!tc.valid) return;
    const cx<T>* w = reinterpret_cast<const cx<T>*>(p.w);
    const bool scaled = p.scale != 1.0;
    const T s = T(p.scale);
    auto store = [&](int k, cx<T> ek) {
        const int o = r2r1_out_index(k, N, dst);
        if (o < 0) return;
        T y = r2r1_value<T>(ek, dst);
        if (scaled) y = rscale<T>(y, s);
        if constexpr (TILED) *out.at(o) = y;
        else *out.at1(o) = y;
    };
    auto emit = [&](int k) {
        cx<T> ek, enk;
        r2r1_split<T>(sm[C::sidx(k, t)], sm[C::sidx((N - k) & (N - 1), t)], ld_tw(w, k), ek, enk);
        store(k, ek);
        if (2 * k != N) store(N - k, enk);
    };
#pragma unroll
    for (int e = 0; e < E / 2; ++e) emit(j + e * TPL);
    if (j == 0) emit(N / 2);
}

// ---- type-IV real-to-real pass: DCT-IV and DST-IV of N = 2M reals per line ------------------------------------------------
// One real line per complex M-point line of the tile (r2r.hpp): point m loads x_{2m} and x_{N-1-2m} and multiplies by p_m,
// CtaFft's stages transform v (p.tw: the M-point table), and point k multiplies V_k by q_k and stores y_{2k} and y_{N-1-2k}
// straight from its final slot: no shared-memory round trip after the stages.  p.w is the type-IV table [p_m][q_k]
// (Tables::get_r2r4), p.dst picks the kind, p.inverse is not read: the transform is its own inverse.  The views count in
// reals.
//   CONTIG: TB real lines per CTA, one per line slot.
//   TILED:  one real column per tile column (TB columns: the wide tile of the length where shared memory allows it).
// One CTA per tile and every load before any store (the stages synchronise the line's threads), so out == in works.  A
// scale != 1 multiplies the stores (__dmul_rn / __fmul_rn: the scaled output is the unscaled one times s, bit for bit).
template <typename T, int LOG2M, int LOG2E, int TB, bool TILED>
__global__ void __launch_bounds__((1 << (LOG2M - LOG2E)) * TB, min_ctas_per_sm<T, LOG2E>((1 << (LOG2M - LOG2E)) * TB))
fft_r2r4_kernel(const __grid_constant__ FftR2r p) {
    using C = CtaFft<T, LOG2M, LOG2E, TB, TILED>;
    using LA = LineAccess<T, C::LINES, T>;
    constexpr int E = C::E, TPL = C::TPL, M = C::N, N = 2 * M;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    cx<T>* sm = reinterpret_cast<cx<T>*>(smem_raw);
    unsigned long long* tab_in = reinterpret_cast<unsigned long long*>(smem_raw + C::TILE_BYTES);
    unsigned long long* tab_out = tab_in + C::LINES * MAXSEG;
    const TileCoord<C, TILED, TB> tc(p);
    const int j = tc.j, t = tc.t;
    if (p.in.nseg > 1 || p.out.nseg > 1) {
        // TILED: one table per CTA, CONTIG: one per line (as in c2c_tile)
        const int line = TILED ? 0 : t, lane = TILED ? int(threadIdx.x) : j, lanes = TILED ? C::THREADS : TPL;
        LA::fill_table(p.in, tab_in, line, lane, lanes, tc.a0, tc.a1);
        LA::fill_table(p.out, tab_out, line, lane, lanes, tc.a0, tc.a1);
        __syncthreads();
    }
    const LA in(p.in, tab_in, TILED ? 0 : t, tc.a0, tc.a1, tc.b), out(p.out, tab_out, TILED ? 0 : t, tc.a0, tc.a1, tc.b);
    const int dst = p.dst;
    const cx<T>* w = reinterpret_cast<const cx<T>*>(p.w);
    auto at = [&](const LA& a, int n) -> T* {
        if constexpr (TILED) return a.at(n);
        else return a.at1(n);
    };
    cx<T> v[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int m = j + e * TPL;
        const T lo = tc.valid ? *at(in, r2r4_lo(m)) : T(0), hi = tc.valid ? *at(in, r2r4_hi(m, N)) : T(0);
        v[e] = r2r4_pre<T>(lo, hi, ld_tw(w, m), dst);
    }
    C::template stages<0>(v, j, t, sm, reinterpret_cast<const cx<T>*>(p.tw));
    if (!tc.valid) return;
    const bool scaled = p.scale != 1.0;
    const T s = T(p.scale);
#pragma unroll
    for (int e = 0; e < E; ++e) {
        const int k = j + e * TPL;
        T lo, hi;
        r2r4_post<T>(v[C::Core::final_slot(e)], ld_tw(w, M + k), dst, lo, hi);
        if (scaled) { lo = rscale<T>(lo, s); hi = rscale<T>(hi, s); }
        *at(out, r2r4_lo(k)) = lo;
        *at(out, r2r4_hi(k, N)) = hi;
    }
}

// ---- copy pass: an axis the plan keeps (dfft_plan_set_transform_axes) ------------------------------------------------
// Moves element (a0, a1, n, b) of p.in to the same index of p.out for any line length p.n, through the segmented views of
// the FFT pass it replaces (scatters into peer slots, gathers from receive slots, blocked layouts and tails unchanged).
//   CONTIG: a CTA holds `lpc` lines of `tpl` threads each (tpl = 2^ltpl), threads run along n: coalesced over n.
//   TILED:  a CTA holds one (a0, a1) and `tpl` consecutive b (tpl = 2^ltpl), its rows blockDim / tpl apart along n:
//           threads run along the contiguous b, so every row is one coalesced run.  The (a0, a1) tiles run in G x G
//           blocks (p.tile_swz = log2 G, tile_order), so that CTAs running at the same time read and write neighbouring
//           rows on both sides when a0 is near on one side and a1 on the other (the blocked hand-over layouts).
// Each thread loads COPY_ILP elements before it stores them; an element is read by the same thread that writes it, before
// it writes it.  A scale != 1 multiplies each real value with __dmul_rn / __fmul_rn, so a scaled copy is the unscaled
// one times s, bit for bit.  E: float, double (the real views of R2R plans), cx<float> or cx<double>.
struct FftCopy : FftParams {
    int n;         // line length
    int ltpl;      // log2 of the threads per line (CONTIG) or per row (TILED)
    double scale;  // output scale, applied when != 1 (rounded to the element's precision once)
};
constexpr int COPY_THREADS = 512;
// elements in flight per thread (experiment knob -DDFFT_COPY_ILP=<n>)
#ifndef DFFT_COPY_ILP
#define DFFT_COPY_ILP 8
#endif
constexpr int COPY_ILP = DFFT_COPY_ILP;
constexpr int COPY_SWZ = 1;  // log2 G of the TILED tile blocking (DFFT_COPY_SWZ overrides it per launch, 0 = plain order)

template <typename E>
struct CopyElem {
    using R = E;
    static __device__ __forceinline__ E ld(const E* p) { return *p; }
    static __device__ __forceinline__ void st(E* p, E v) { *p = v; }
    static __device__ __forceinline__ E mul(E v, R s) { return rscale<R>(v, s); }
};
template <typename T>
struct CopyElem<cx<T>> {
    using R = T;
    static __device__ __forceinline__ cx<T> ld(const cx<T>* p) { return ld_elem<T>(p); }
    static __device__ __forceinline__ void st(cx<T>* p, cx<T> v) { st_elem<T>(p, v); }
    static __device__ __forceinline__ cx<T> mul(cx<T> v, T s) { return cx<T>{rscale<T>(v.x, s), rscale<T>(v.y, s)}; }
};

// element (a0, a1, n, b) of a view: p0 + n sN for a single-segment view (p0: element n = 0 of the line), through the
// segment of n otherwise
template <typename E>
struct CopyLine {
    E* p0;
    long long sN;
    bool multi;
    __device__ __forceinline__ CopyLine(const View& v, int a0, int a1, int b) {
        const Seg& g = v.seg[0];
        p0 = reinterpret_cast<E*>(g.base) + (a0 * g.sA0 + a1 * g.sA1 - (long long)g.n0 * v.sN + b);
        sN = v.sN;
        multi = v.nseg > 1;
    }
    __device__ __forceinline__ E* at(const View& v, int a0, int a1, int n, int b) const {
        if (!multi) return p0 + n * sN;
        const Seg& g = v.seg[v.seg_of_n[n]];
        return reinterpret_cast<E*>(g.base) + (a0 * g.sA0 + a1 * g.sA1 + (long long)(n - g.n0) * sN + b);
    }
};

template <typename E, bool TILED>
__global__ void __launch_bounds__(COPY_THREADS) fft_copy_kernel(const __grid_constant__ FftCopy p) {
    using CE = CopyElem<E>;
    const int tid = threadIdx.x, tpl = 1 << p.ltpl;
    int a0, a1, b, j, step;
    bool valid;
    if constexpr (TILED) {
        const int nbt = (p.B + tpl - 1) >> p.ltpl;
        const int bt = int(blockIdx.x % unsigned(nbt));
        tile_order(p, int(blockIdx.x / unsigned(nbt)), a1, a0);
        b = (bt << p.ltpl) + (tid & (tpl - 1));
        j = tid >> p.ltpl;
        step = COPY_THREADS >> p.ltpl;
        valid = b < p.B;
    } else {
        const long long line = (long long)blockIdx.x * (COPY_THREADS >> p.ltpl) + (tid >> p.ltpl);
        a1 = int(line % p.A1);
        a0 = int(line / p.A1);
        b = 0;
        j = tid & (tpl - 1);
        step = tpl;
        valid = line < (long long)p.A0 * p.A1;
    }
    if (!valid) return;
    const bool scaled = p.scale != 1.0;
    const typename CE::R s = typename CE::R(p.scale);
    const CopyLine<E> in(p.in, a0, a1, b), out(p.out, a0, a1, b);
    for (int n0 = j; n0 < p.n; n0 += COPY_ILP * step) {
        E v[COPY_ILP];
#pragma unroll
        for (int u = 0; u < COPY_ILP; ++u) {
            const int n = n0 + u * step;
            if (n < p.n) v[u] = CE::ld(in.at(p.in, a0, a1, n, b));
        }
#pragma unroll
        for (int u = 0; u < COPY_ILP; ++u) {
            const int n = n0 + u * step;
            if (n < p.n) CE::st(out.at(p.out, a0, a1, n, b), scaled ? CE::mul(v[u], s) : v[u]);
        }
    }
}

// ---- host launchers (one explicit instantiation per precision and size, see fft_inst.cu) ----------------
// S: the stored element, cx<T>, or cx16<H> with T = float for 16-bit plans (H = __half for DFFT_F16, __nv_bfloat16 for
// DFFT_BF16: kind PASS_C2C_CONTIG, PASS_C2C_TILED, PASS_R2C or PASS_C2R, the f32 kernels' arithmetic).
// scale: the output scale of the pass' stores; 1 launches the unscaled kernels, anything else their scaled twins.
template <typename T, typename S, int LOG2N>
cudaError_t launch_pass(PassKind kind, const FftParams& p, double scale, cudaStream_t stream);

// Each launcher also has a runtime form (fft_dispatch.cu) that takes the precision (DFFT_F64 / DFFT_F32; launch_pass also
// DFFT_F16 / DFFT_BF16) and the log2 length first; it returns cudaErrorInvalidValue for a length that is not instantiated.
cudaError_t launch_pass(int prec, int log2n, PassKind kind, const FftParams& p, double scale, cudaStream_t stream);

// padded pass (FftPadded): kind PASS_C2C_CONTIG, PASS_C2C_TILED, PASS_R2C or PASS_C2R over the views of launch_pass, the
// hole [p.ld_lo, p.ld_hi) of each line on its loaded side and [p.st_lo, p.st_hi) on its stored side (R2C / C2R: both reach
// the end of the line); p.scale scales the stores.  With p.w set (dfft_plan_set_weights) the weighted twins run: p.w
// multiplies the spectral side, whose holes may be empty.
template <typename T, int LOG2N>
cudaError_t launch_twin(PassKind kind, const FftPadded& p, cudaStream_t stream);
cudaError_t launch_twin(int prec, int log2n, PassKind kind, const FftPadded& p, cudaStream_t stream);

// fused z + y stage (fft_zy_fused_kernel), instantiated for the lengths zy_fused_length accepts.  pz: the z pass, py: the y
// pass, f: counters and plane groups (f.order.na / nb are filled in here).  Every launch of one step must use the same
// counters and the same grid (zy_launch_of), which the launcher's fixed grid for a given work list provides.  scale: of the
// last phase's stores, inverse only (the forward stage stores an intermediate).
template <typename T, int LOG2N>
cudaError_t launch_zy_fused(const FftParams& pz, const FftParams& py, const ZyFused& f, double scale, cudaStream_t stream);
cudaError_t launch_zy_fused(int prec, int log2n, const FftParams& pz, const FftParams& py, const ZyFused& f, double scale, cudaStream_t stream);
constexpr bool zy_fused_length(int log2n) { return log2n == 8 || log2n == 9; }

// batched small cubic fields (fft_batch_small_kernel), instantiated for the lengths batch_small_length accepts.  in / out:
// the caller's buffers (fields back to back); f: counters, table and look-ahead (the work list is filled in here).  Every
// launch of one step must use the same counters and the same batch, so that the grid and the draws per launch stay fixed.
// scale: of phase B's stores.
template <typename T, int LOG2N>
cudaError_t launch_batch_small(const void* in, void* out, long long batch, int inverse, const BatchSmall& f, double scale, cudaStream_t stream);
cudaError_t launch_batch_small(int prec, int log2n, const void* in, void* out, long long batch, int inverse, const BatchSmall& f, double scale,
                               cudaStream_t stream);

// Bluestein pass (fft_bluestein_kernel) of p.n-point lines, M = 2^LOG2M >= 2 p.n - 1: kind PASS_C2C_CONTIG or PASS_C2C_TILED
// (the view mapping of the power-of-two pass), one CTA per tile; p.scale scales the stores, p.w (if set) weights them (the
// weighted twin, WEIGHTED = true).  Instantiated for LOG2M 3..13.
template <typename T, int LOG2M>
cudaError_t launch_bluestein(PassKind kind, const FftBluestein& p, cudaStream_t stream);
cudaError_t launch_bluestein(int prec, int log2m, PassKind kind, const FftBluestein& p, cudaStream_t stream);

// R2R pass of 2^LOG2N-point real lines: kind PASS_R2R_CONTIG (sN == 1, line pairs) or PASS_R2R_TILED (column pairs), views
// in reals, one CTA per tile; p.scale scales the stores.  hc: R2HC / HC2R (fft_r2hc_kernel), otherwise DCT / DST
// (fft_r2r_kernel, p.dst).  Instantiated for LOG2N 1..13.
template <typename T, int LOG2N>
cudaError_t launch_r2r(PassKind kind, const FftR2r& p, bool hc, cudaStream_t stream);
cudaError_t launch_r2r(int prec, int log2n, PassKind kind, const FftR2r& p, bool hc, cudaStream_t stream);

// DCT-I / DST-I pass (fft_r2r1_kernel, p.dst) of real lines of 2^LOG2N + 1 or 2^LOG2N - 1 points: kind PASS_R2R_CONTIG
// (sN == 1, TBC lines per CTA) or PASS_R2R_TILED (one real column per tile column), views in reals, one CTA per tile;
// p.w = Tables::get_tw2(LOG2N), p.scale scales the stores.  Instantiated for LOG2N 1..13.
template <typename T, int LOG2N>
cudaError_t launch_r2r1(PassKind kind, const FftR2r& p, cudaStream_t stream);
cudaError_t launch_r2r1(int prec, int log2n, PassKind kind, const FftR2r& p, cudaStream_t stream);

// DCT-IV / DST-IV pass (fft_r2r4_kernel, p.dst) of real lines of 2^(LOG2M + 1) points through M-point complex lines: kinds
// and views as for launch_r2r1; p.tw = Tables::get_tw(LOG2M), p.w = Tables::get_r2r4(LOG2M + 1), p.scale scales the
// stores.  Instantiated for LOG2M 1..12.
template <typename T, int LOG2M>
cudaError_t launch_r2r4(PassKind kind, const FftR2r& p, cudaStream_t stream);
cudaError_t launch_r2r4(int prec, int log2m, PassKind kind, const FftR2r& p, cudaStream_t stream);

// copy pass of p.n-point lines (fft_copy_kernel): kind PASS_COPY_CONTIG or PASS_COPY_TILED, p.ltpl is filled in here.
// Instantiated for E = T and cx<T> in the LOG2N = 1 unit of each precision; the runtime form takes real != 0 for the
// real elements of R2R plans, and moves the 4-byte elements of 16-bit plans as E = float, unscaled.
template <typename E>
cudaError_t launch_copy(PassKind kind, const FftCopy& p, cudaStream_t stream);
cudaError_t launch_copy(int prec, bool real, PassKind kind, const FftCopy& p, cudaStream_t stream);

constexpr int MAX_LOG2N = 13;
constexpr int BLUESTEIN_MAX_N = 4096;  // 2n - 1 <= 2^MAX_LOG2N

}  // namespace dfft
