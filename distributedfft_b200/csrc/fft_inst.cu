// fft_inst.cu — compiled once per (precision, log2 length): -DDFFT_T=double -DDFFT_LOG2N=10, and once per (16-bit format,
// log2 length) of 16-bit plans: -DDFFT_T=float -DDFFT_S=__half (or __nv_bfloat16) -DDFFT_LOG2N=10, which compiles
// launch_pass<float, cx16<DFFT_S>, 10> only.  Splitting the instantiations over translation units lets build.py compile them in parallel.
#include <cstdlib>

#include "fft_kernels.cuh"

#ifndef DFFT_T
#error "compile with -DDFFT_T=<float|double> -DDFFT_LOG2N=<1..13>"
#endif

namespace dfft {

template <typename K>
static cudaError_t set_smem(K kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return cudaSuccess;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
}

static int env_int(const char* name, int dflt) {
    const char* e = getenv(name);  // read per launch (cheap) so that one process can compare variants
    return e ? atoi(e) : dflt;
}

// cuTensorMapEncodeTiled through the runtime (libdfft.so does not link libcuda)
typedef CUresult (*encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static encode_tiled_fn encode_tiled() {
    static encode_tiled_fn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess) { cudaGetLastError(); f = nullptr; }
        return (encode_tiled_fn)f;
    }();
    return fn;
}

// rank-4 tensor map (b, n, a1, a0) of a single-segment view; box TB x min(N, 256) x 1 x 1.  false: the view does not
// meet the TMA constraints (16-byte aligned base and strides) and the register-fed kernel is used instead.
template <typename T>
static bool make_view_map(const View& v, int A0, int A1, int N, int B, int TB, CUtensorMap* tm) {
    encode_tiled_fn enc = encode_tiled();
    if (!enc || v.nseg != 1) return false;
    const unsigned long long es = sizeof(cx<T>);
    const int d0 = sizeof(T) == 8 ? 2 : 1;  // 8-byte units per complex element
    char* base = reinterpret_cast<char*>(v.seg[0].base) - (long long)v.seg[0].n0 * v.sN * (long long)es;
    if (reinterpret_cast<unsigned long long>(base) % 16) return false;
    if (v.sN <= 0 || v.seg[0].sA0 < 0 || v.seg[0].sA1 < 0) return false;
    cuuint64_t dims[4] = {cuuint64_t(B) * d0, cuuint64_t(N), cuuint64_t(A1 > 0 ? A1 : 1), cuuint64_t(A0 > 0 ? A0 : 1)};
    unsigned long long sn = (unsigned long long)v.sN * es;
    unsigned long long s1 = A1 > 1 ? (unsigned long long)v.seg[0].sA1 * es : sn * N;
    unsigned long long s0 = A0 > 1 ? (unsigned long long)v.seg[0].sA0 * es : sn * N;
    if (s1 == 0) s1 = sn * N;
    if (s0 == 0) s0 = sn * N;
    cuuint64_t strides[3] = {sn, s1, s0};
    for (int i = 0; i < 3; ++i)
        if (strides[i] % 16 || strides[i] >= (1ull << 40)) return false;
    if ((cuuint64_t(TB) * d0 * 8) % 16) return false;
    cuuint32_t box[4] = {cuuint32_t(TB * d0), cuuint32_t(N < 256 ? N : 256), 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the parameters of a scaled twin (FftScaled): the pass' parameters and the output scale
static FftScaled with_scale(const FftParams& p, double scale) {
    FftScaled q;
    static_cast<FftParams&>(q) = p;
    q.scale = scale;
    return q;
}

// Launches one instantiation of a kernel template: KF / KI forward / inverse, KFS / KIS their scaled twins, picked by
// p.inverse and scale != 1; `rest` follows the parameters.  Kernels without an inverse flag (R2C, C2R) pass their kernel as
// both KF and KI, kernels without scaled twins nullptr (the Bluestein kernel scales by a runtime value of its parameters).
// The shared-memory attribute of the unscaled pair is set on its first launch, that of the twins on their first launch.
template <auto KF, auto KI, auto KFS, auto KIS, typename P, typename... R>
static cudaError_t launch_kernel(const P& p, double scale, unsigned grid, int threads, size_t smem, cudaStream_t stream, const R&... rest) {
    static const cudaError_t once = set_smem(KF, smem) == cudaSuccess ? set_smem(KI, smem) : cudaErrorInvalidValue;
    if (once != cudaSuccess) return once;
    if constexpr (!std::is_null_pointer_v<decltype(KIS)>) {
        if (scale != 1.0) {
            static const cudaError_t onces = set_smem(KFS, smem) == cudaSuccess ? set_smem(KIS, smem) : cudaErrorInvalidValue;
            if (onces != cudaSuccess) return onces;
            const FftScaled q = with_scale(p, scale);
            if (p.inverse) KIS<<<grid, threads, smem, stream>>>(q, rest...);
            else KFS<<<grid, threads, smem, stream>>>(q, rest...);
            return cudaGetLastError();
        }
    }
    if (p.inverse) KI<<<grid, threads, smem, stream>>>(p, rest...);
    else KF<<<grid, threads, smem, stream>>>(p, rest...);
    return cudaGetLastError();
}

// CTAs of a persistent kernel that fit on the device at once (callers keep the value in a static per instantiation)
template <typename K>
static int resident_ctas(K kernel, int threads, size_t smem) {
    int dev = 0, sms = 0, per = 0;
    set_smem(kernel, smem);  // the occupancy counts with the kernel's shared-memory limit
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, threads, smem) != cudaSuccess || per < 1) per = 1;
    return sms * per;
}

// the tile-order blocking log2 G where the batch extents allow it (G <= 16 divides A0 and A1), plain order otherwise
static int tile_swz_for(int swz, int A0, int A1) {
    return swz > 0 && swz <= 4 && A0 % (1 << swz) == 0 && A1 % (1 << swz) == 0 ? swz : 0;
}

// Wide tiles (S::TBT_WIDE: 128-byte rows, one CTA per SM) or narrow ones (S::TBT) for a TILED pass of 2^LOG2N-point lines.
// Wide when the rows of a tile sit in different 2 MB pages (x passes: a row pitch of es-byte stored elements >= 1 MiB),
// narrow otherwise (y passes); a choice still to be confirmed on the H100 (tools/axis_bench.py).  tma: the pass can run the
// TMA-fed kernel (launch_tiled), which takes the wide tile for near rows as well unless DFFT_TMA=0.  DFFT_WIDE_TILES=1 / -1
// and p.tile_pref force either.  Never a wide tile for a view that is only one narrow tile wide (blocked hand-over with
// CH = TBT): half of its columns would be empty.
template <typename T, int LOG2N>
static bool wide_tile(const FftParams& p, size_t es, bool tma) {
    using S = Shape<T, LOG2N>;
    const int w = env_int("DFFT_WIDE_TILES", 0);
    const bool far_rows = (unsigned long long)p.in.sN * es >= (1ull << 20) || (unsigned long long)p.out.sN * es >= (1ull << 20);
    const bool tma_auto = tma && env_int("DFFT_TMA", -1) != 0 && p.in.nseg == 1;
    const bool wide = w > 0 || p.tile_pref == 2 || (w == 0 && p.tile_pref == 0 && LOG2N >= 10 && (far_rows || tma_auto));
    return wide && w >= 0 && p.tile_pref != 1 && p.B > S::TBT;
}

// S: the stored element; the TMA-fed kernel serves cx<T> passes only
template <typename T, typename S, int LOG2N, int TB>
static cudaError_t launch_tiled(const FftParams& p_in, double scale, cudaStream_t stream, long long lines) {
    FftParams p = p_in;
    const int swz = env_int("DFFT_TILE_SWZ", -1);  // experiment override of the tile-order blocking
    p.tile_swz = tile_swz_for(swz >= 0 ? swz : p.tile_swz, p.A0, p.A1);
    constexpr int LOG2E = Shape<T, LOG2N>::LOG2E;
    using C = CtaFft<T, LOG2N, LOG2E, TB, true>;
    if (p.B <= 0) return cudaSuccess;
    const long long grid = lines * ((p.B + TB - 1) / TB);
    if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    if constexpr (std::is_same_v<S, cx<T>> && C::NST >= 2 && LOG2N >= 7) {
        // TMA-fed persistent kernel (fft_c2c_tma_kernel).  Design rationale, not yet measured on the H100
        // (tools/axis_bench.py times both kernels per pass): the TMA engine relieves the register-fed kernel where its
        // strided 64/128-byte row loads load the L1TEX pipe most, f64 lines of >= 1024 points.  Lines of <= 512 points
        // and f32 tiles keep the register-fed kernel (fewer stages to overlap, or a tile that leaves room for one CTA per
        // SM only), and so do 64-byte rows of the blocked hand-over layout.
        // Default (-1): f64 lines of >= 1024 points, except 64-byte blocked rows; DFFT_TMA=1 forces it on, 0 off.
        const int mode = env_int("DFFT_TMA", -1);
        const bool narrow_blocked = p.B == TB && TB * sizeof(cx<T>) < 128;
        const bool want = mode > 0 || (mode < 0 && sizeof(T) == 8 && LOG2N >= 10 && !narrow_blocked);
        const bool bulk_ok = p.bulk_out && p.out.sN == TB && p.B == TB;
        alignas(64) CUtensorMap tm;
        if (want && p.in.nseg == 1 && (!p.bulk_out || bulk_ok) && make_view_map<T>(p.in, p.A0, p.A1, C::N, p.B, TB, &tm)) {
            constexpr auto tf = fft_c2c_tma_kernel<T, LOG2N, LOG2E, TB, false, false>;
            static const int resident = resident_ctas(tf, C::THREADS, C::SMEM_BYTES);
            long long g = grid < resident ? grid : resident;
            if (p.max_ctas > 0 && g > p.max_ctas) g = p.max_ctas;
            FftParams q = p;
            q.bulk_out = bulk_ok ? 1 : 0;
            return launch_kernel<tf, fft_c2c_tma_kernel<T, LOG2N, LOG2E, TB, true, false>, fft_c2c_tma_kernel<T, LOG2N, LOG2E, TB, false, true>,
                                 fft_c2c_tma_kernel<T, LOG2N, LOG2E, TB, true, true>>(q, scale, unsigned(g), C::THREADS, C::SMEM_BYTES, stream, tm);
        }
    }
    const unsigned g = unsigned((p.max_ctas > 0 && grid > p.max_ctas) ? p.max_ctas : grid);
    return launch_kernel<fft_c2c_kernel<T, S, LOG2N, LOG2E, TB, true, false, false>, fft_c2c_kernel<T, S, LOG2N, LOG2E, TB, true, true, false>,
                         fft_c2c_kernel<T, S, LOG2N, LOG2E, TB, true, false, true>, fft_c2c_kernel<T, S, LOG2N, LOG2E, TB, true, true, true>>(
        p, scale, g, C::THREADS, C::SMEM_BYTES, stream);
}

// S = cx16<H> (16-bit plans): the shapes of the f32 pass, TILED tiles included.  Their TILED rows are the f32 tile's 8
// elements wide from 512-point lines on, 32 bytes of 16-bit pairs: at 512^3 on an H100 the y and x passes took 0.43-0.50 ms
// with them against 0.69-0.72 ms with 64-byte rows (16 elements, twice the threads and shared memory per CTA), DESIGN.md
// section 3.20.  16-bit plans have no interleaved passes.
template <typename T, typename S, int LOG2N>
cudaError_t launch_pass(PassKind kind, const FftParams& p, double scale, cudaStream_t stream) {
    using SH = Shape<T, LOG2N>;
    constexpr int LOG2E = SH::LOG2E;
    constexpr bool PLAIN = std::is_same_v<S, cx<T>>;
    using C = CtaFft<T, LOG2N, LOG2E, SH::TBC, false>;
    const long long lines = (long long)p.A0 * p.A1;
    if (lines <= 0) return cudaSuccess;
    const long long grid = (lines + SH::TBC - 1) / SH::TBC;  // CONTIG, R2C and C2R
    switch (kind) {
        case PASS_C2C_CONTIG:
            if (p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
            if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
            return launch_kernel<fft_c2c_kernel<T, S, LOG2N, LOG2E, SH::TBC, false, false, false>, fft_c2c_kernel<T, S, LOG2N, LOG2E, SH::TBC, false, true, false>,
                                 fft_c2c_kernel<T, S, LOG2N, LOG2E, SH::TBC, false, false, true>, fft_c2c_kernel<T, S, LOG2N, LOG2E, SH::TBC, false, true, true>>(
                p, scale, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
        case PASS_C2C_TILED:
            if (wide_tile<T, LOG2N>(p, sizeof(S), PLAIN && sizeof(T) == 8 && LOG2N >= 10)) return launch_tiled<T, S, LOG2N, SH::TBT_WIDE>(p, scale, stream, lines);
            return launch_tiled<T, S, LOG2N, SH::TBT>(p, scale, stream, lines);
        case PASS_C2C_ILV: {
            if constexpr (!PLAIN) return cudaErrorInvalidValue;
            else {
                // C = B components per point, lines C apart along n.  From the tile width on, the TILED kernel's tiles are
                // full rows of components; below it the interleaved kernel keeps every thread busy.
                if (p.B < 1 || p.in.sN != p.B || p.out.sN != p.B) return cudaErrorInvalidValue;
                if (p.B >= SH::TBT) return launch_tiled<T, S, LOG2N, SH::TBT>(p, scale, stream, lines);
                const long long g = (lines * p.B + SH::TBC - 1) / SH::TBC;
                if (g > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
                const unsigned grid_ilv = unsigned((p.max_ctas > 0 && g > p.max_ctas) ? p.max_ctas : g);
                return launch_kernel<fft_c2c_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, false, false>, fft_c2c_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, true, false>,
                                     fft_c2c_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, false, true>, fft_c2c_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, true, true>>(
                    p, scale, grid_ilv, C::THREADS, C::SMEM_BYTES, stream);
            }
        }
        case PASS_R2C_ILV:
        case PASS_C2R_ILV: {
            if constexpr (!PLAIN) return cudaErrorInvalidValue;
            else {
                // C = B components, one line per component; the real side is one segment
                const bool c2r = kind == PASS_C2R_ILV;
                if (p.B < 1 || (c2r ? p.out.nseg : p.in.nseg) != 1) return cudaErrorInvalidValue;
                const long long g = (lines * p.B + SH::TBC - 1) / SH::TBC;
                if (g > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
                const unsigned grid_rc = unsigned((p.max_ctas > 0 && g > p.max_ctas) ? p.max_ctas : g);
                if (c2r) {
                    constexpr auto k = fft_rc_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, true, false>;
                    constexpr auto ks = fft_rc_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, true, true>;
                    return launch_kernel<k, k, ks, ks>(p, scale, grid_rc, C::THREADS, C::SMEM_BYTES, stream);
                }
                constexpr auto k = fft_rc_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, false, false>;
                constexpr auto ks = fft_rc_ilv_kernel<T, LOG2N, LOG2E, SH::TBC, false, true>;
                return launch_kernel<k, k, ks, ks>(p, scale, grid_rc, C::THREADS, C::SMEM_BYTES, stream);
            }
        }
        case PASS_R2C: {
            if (p.in.nseg != 1 || p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
            if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
            constexpr auto k = fft_r2c_kernel<T, S, LOG2N, LOG2E, SH::TBC, false>;
            constexpr auto ks = fft_r2c_kernel<T, S, LOG2N, LOG2E, SH::TBC, true>;
            return launch_kernel<k, k, ks, ks>(p, scale, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
        }
        case PASS_C2R: {
            if (p.out.nseg != 1 || p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
            if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
            constexpr auto k = fft_c2r_kernel<T, S, LOG2N, LOG2E, SH::TBC, false>;
            constexpr auto ks = fft_c2r_kernel<T, S, LOG2N, LOG2E, SH::TBC, true>;
            return launch_kernel<k, k, ks, ks>(p, scale, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
        }
        default: return cudaErrorInvalidValue;
    }
}

#ifdef DFFT_S
template cudaError_t launch_pass<float, cx16<DFFT_S>, DFFT_LOG2N>(PassKind, const FftParams&, double, cudaStream_t);
#else
template cudaError_t launch_pass<DFFT_T, cx<DFFT_T>, DFFT_LOG2N>(PassKind, const FftParams&, double, cudaStream_t);

// the padded twins (fft_c2c_padded_kernel, fft_r2c_padded_kernel, fft_c2r_padded_kernel), their weighted instantiations
// (WEIGHTED = true) where p.w is set, and the twiddled C2C passes of 1D plans (TWIDDLED = true) where p.tw1d is set, TILED
// ones in their transposing form (TRANSPOSED = true) where p.tw_sB is set: the tiles of launch_pass (TILED: narrow or wide
// by wide_tile, without the TMA-fed kernel), one CTA per tile
template <typename T, int LOG2N>
cudaError_t launch_twin(PassKind kind, const FftPadded& p, cudaStream_t stream) {
    using S = Shape<T, LOG2N>;
    constexpr int LOG2E = S::LOG2E;
    const long long lines = (long long)p.A0 * p.A1;
    if (lines <= 0) return cudaSuccess;
    // points of the loaded and the stored side's line: the spectral side of R2C / C2R has one more
    const bool half = kind == PASS_R2C || kind == PASS_C2R;
    const int n_ld = (1 << LOG2N) + (kind == PASS_C2R ? 1 : 0), n_st = (1 << LOG2N) + (kind == PASS_R2C ? 1 : 0);
    if (p.ld_lo < 0 || p.ld_hi < p.ld_lo || p.ld_hi > n_ld || p.st_lo < 0 || p.st_hi < p.st_lo || p.st_hi > n_st) return cudaErrorInvalidValue;
    // the R2C / C2R twins test k < lo only: their holes reach the end of the line
    if (half && (p.ld_hi != n_ld || p.st_hi != n_st)) return cudaErrorInvalidValue;
    const long long grid = (lines + S::TBC - 1) / S::TBC;  // CONTIG, R2C and C2R
    const auto launch = [&](auto weighted, auto twiddled) -> cudaError_t {
        constexpr bool W = decltype(weighted)::value, TW = decltype(twiddled)::value;
        using C = CtaFft<T, LOG2N, LOG2E, S::TBC, false>;
        // TILED, tiles TB columns wide
        const auto tiled = [&](auto tb) -> cudaError_t {
            constexpr int TB = decltype(tb)::value;
            using CT = CtaFft<T, LOG2N, LOG2E, TB, true>;
            FftPadded q = p;
            q.tile_swz = tile_swz_for(p.tile_swz, p.A0, p.A1);
            const long long g = lines * ((p.B + TB - 1) / TB);
            if (g > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
            if constexpr (TW) {
                if (p.tw_sB) {  // the transposing form: its row side is one segment with contiguous lines
                    const View& row = p.inverse ? p.out : p.in;
                    if (row.nseg != 1 || row.sN != 1 || q.tile_swz) return cudaErrorInvalidValue;
                    return launch_kernel<fft_c2c_padded_kernel<T, LOG2N, LOG2E, TB, true, false, false, true, true>,
                                         fft_c2c_padded_kernel<T, LOG2N, LOG2E, TB, true, true, false, true, true>, nullptr, nullptr>(
                        q, 1.0, unsigned(g), CT::THREADS, CT::SMEM_BYTES, stream);
                }
            }
            return launch_kernel<fft_c2c_padded_kernel<T, LOG2N, LOG2E, TB, true, false, W, TW>, fft_c2c_padded_kernel<T, LOG2N, LOG2E, TB, true, true, W, TW>,
                                 nullptr, nullptr>(q, 1.0, unsigned(g), CT::THREADS, CT::SMEM_BYTES, stream);
        };
        if (p.tw_sB && !(TW && kind == PASS_C2C_TILED)) return cudaErrorInvalidValue;  // TRANSPOSED: twiddled TILED passes only
        switch (kind) {
            case PASS_C2C_CONTIG:
                if (p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
                if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
                return launch_kernel<fft_c2c_padded_kernel<T, LOG2N, LOG2E, S::TBC, false, false, W, TW>,
                                     fft_c2c_padded_kernel<T, LOG2N, LOG2E, S::TBC, false, true, W, TW>, nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
            case PASS_C2C_TILED:
                if (p.B <= 0) return cudaSuccess;
                if (wide_tile<T, LOG2N>(p, sizeof(cx<T>), false)) return tiled(std::integral_constant<int, S::TBT_WIDE>());
                return tiled(std::integral_constant<int, S::TBT>());
            case PASS_R2C:
            case PASS_C2R: {
                if constexpr (TW) return cudaErrorInvalidValue;  // 1D plans are C2C
                if ((kind == PASS_R2C ? p.in.nseg : p.out.nseg) != 1 || p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
                if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
                if (kind == PASS_R2C) {
                    constexpr auto k = fft_r2c_padded_kernel<T, LOG2N, LOG2E, S::TBC, W>;
                    return launch_kernel<k, k, nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
                }
                constexpr auto k = fft_c2r_padded_kernel<T, LOG2N, LOG2E, S::TBC, W>;
                return launch_kernel<k, k, nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
            }
            default: return cudaErrorInvalidValue;
        }
    };
    if (p.tw1d && p.w) return cudaErrorInvalidValue;  // 1D plans have no spectral weights
    if (p.tw1d) return launch(std::false_type(), std::true_type());
    if (p.w) return launch(std::true_type(), std::false_type());
    return launch(std::false_type(), std::false_type());
}

template cudaError_t launch_twin<DFFT_T, DFFT_LOG2N>(PassKind, const FftPadded&, cudaStream_t);

#if DFFT_LOG2N >= 3
// the Bluestein kernel, its weighted instantiation (WEIGHTED = true) where p.w is set
template <typename T, int LOG2M, int TB, bool TILED>
static cudaError_t launch_bluestein_tiles(const FftBluestein& p, long long grid, cudaStream_t stream) {
    constexpr int LOG2E = Shape<T, LOG2M>::LOG2E;
    using C = CtaFft<T, LOG2M, LOG2E, TB, TILED>;
    if (grid <= 0) return cudaSuccess;
    if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    if (p.w)
        return launch_kernel<fft_bluestein_kernel<T, LOG2M, LOG2E, TB, TILED, false, true>, fft_bluestein_kernel<T, LOG2M, LOG2E, TB, TILED, true, true>,
                             nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
    return launch_kernel<fft_bluestein_kernel<T, LOG2M, LOG2E, TB, TILED, false, false>, fft_bluestein_kernel<T, LOG2M, LOG2E, TB, TILED, true, false>,
                         nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
}

template <typename T, int LOG2M>
cudaError_t launch_bluestein(PassKind kind, const FftBluestein& p_in, cudaStream_t stream) {
    using S = Shape<T, LOG2M>;
    if (p_in.n < 1 || 2 * (long long)p_in.n - 1 > (1LL << LOG2M) || !p_in.chirp || !p_in.kspec) return cudaErrorInvalidValue;
    const long long lines = (long long)p_in.A0 * p_in.A1;
    if (lines <= 0) return cudaSuccess;
    FftBluestein p = p_in;
    if (kind == PASS_C2C_CONTIG) {
        if (p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
        return launch_bluestein_tiles<T, LOG2M, S::TBC, false>(p, (lines + S::TBC - 1) / S::TBC, stream);
    }
    if (kind != PASS_C2C_TILED) return cudaErrorInvalidValue;
    p.tile_swz = tile_swz_for(p.tile_swz, p.A0, p.A1);  // the tile-order blocking of launch_tiled
    if (p.B <= 0) return cudaSuccess;
    return launch_bluestein_tiles<T, LOG2M, S::TBT, true>(p, lines * ((p.B + S::TBT - 1) / S::TBT), stream);
}

template cudaError_t launch_bluestein<DFFT_T, DFFT_LOG2N>(PassKind, const FftBluestein&, cudaStream_t);
#endif

template <typename T, int LOG2N, int TB, bool TILED>
static cudaError_t launch_r2r_tiles(const FftR2r& p, bool hc, long long grid, cudaStream_t stream) {
    using RS = R2rShape<T, LOG2N, Shape<T, LOG2N>::LOG2E, TB, TILED>;
    constexpr int LOG2E = Shape<T, LOG2N>::LOG2E;
    if (grid <= 0) return cudaSuccess;
    if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    if (hc)
        return launch_kernel<fft_r2hc_kernel<T, LOG2N, LOG2E, TB, TILED, false>, fft_r2hc_kernel<T, LOG2N, LOG2E, TB, TILED, true>, nullptr, nullptr>(
            p, 1.0, unsigned(grid), RS::C::THREADS, RS::SMEM_BYTES, stream);
    return launch_kernel<fft_r2r_kernel<T, LOG2N, LOG2E, TB, TILED, false>, fft_r2r_kernel<T, LOG2N, LOG2E, TB, TILED, true>, nullptr, nullptr>(
        p, 1.0, unsigned(grid), RS::C::THREADS, RS::SMEM_BYTES, stream);
}

// CONTIG: TBC line pairs per CTA; TILED: the tile of the C2C pass, TBT column pairs wide (2 TBT reals: the blocked
// hand-over width of R2R plans)
template <typename T, int LOG2N>
cudaError_t launch_r2r(PassKind kind, const FftR2r& p, bool hc, cudaStream_t stream) {
    using S = Shape<T, LOG2N>;
    if ((!hc && !p.w) || !p.tw) return cudaErrorInvalidValue;
    const long long lines = (long long)p.A0 * p.A1;
    if (lines <= 0) return cudaSuccess;
    if (kind == PASS_R2R_CONTIG) {
        if (p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
        return launch_r2r_tiles<T, LOG2N, S::TBC, false>(p, hc, ((lines + 1) / 2 + S::TBC - 1) / S::TBC, stream);
    }
    if (kind != PASS_R2R_TILED) return cudaErrorInvalidValue;
    if (p.B <= 0) return cudaSuccess;
    const long long pairs = ((long long)p.B + 1) / 2;
    return launch_r2r_tiles<T, LOG2N, S::TBT, true>(p, hc, lines * ((pairs + S::TBT - 1) / S::TBT), stream);
}

template cudaError_t launch_r2r<DFFT_T, DFFT_LOG2N>(PassKind, const FftR2r&, bool, cudaStream_t);

// The passes that run one real line per complex 2^LOG2N-point line of the tile (type I: fft_r2r1_kernel, type IV:
// fft_r2r4_kernel), KC / KT the kernel's CONTIG / TILED instantiation.  CONTIG: TBC lines per CTA.  TILED: one real per
// tile column, so the wide tile of the length (2 TBT columns where it fits 128 KB and 1024 threads) gives rows of 2 TBT
// reals, the row width of the paired R2R tile (>= 64 bytes); lengths whose wide tile does not fit keep TBT columns.  The
// tile order is the C2C pass's (tile_swz_for).
template <typename T, int LOG2N, auto KC, auto KT>
static cudaError_t launch_real_lines(PassKind kind, const FftR2r& p_in, cudaStream_t stream) {
    using S = Shape<T, LOG2N>;
    constexpr int LOG2E = S::LOG2E;
    if (!p_in.w || !p_in.tw) return cudaErrorInvalidValue;
    const long long lines = (long long)p_in.A0 * p_in.A1;
    if (lines <= 0) return cudaSuccess;
    FftR2r p = p_in;
    p.tile_swz = tile_swz_for(p.tile_swz, p.A0, p.A1);
    if (kind == PASS_R2R_CONTIG) {
        using C = CtaFft<T, LOG2N, LOG2E, S::TBC, false>;
        if (p.in.sN != 1 || p.out.sN != 1) return cudaErrorInvalidValue;
        const long long grid = (lines + S::TBC - 1) / S::TBC;
        if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
        return launch_kernel<KC, KC, nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
    }
    if (kind != PASS_R2R_TILED) return cudaErrorInvalidValue;
    if (p.B <= 0) return cudaSuccess;
    constexpr int TB = S::TBT_WIDE;
    using C = CtaFft<T, LOG2N, LOG2E, TB, true>;
    const long long grid = lines * ((p.B + TB - 1) / TB);
    if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    return launch_kernel<KT, KT, nullptr, nullptr>(p, 1.0, unsigned(grid), C::THREADS, C::SMEM_BYTES, stream);
}

template <typename T, int LOG2N>
cudaError_t launch_r2r1(PassKind kind, const FftR2r& p, cudaStream_t stream) {
    using S = Shape<T, LOG2N>;
    return launch_real_lines<T, LOG2N, fft_r2r1_kernel<T, LOG2N, S::LOG2E, S::TBC, false>, fft_r2r1_kernel<T, LOG2N, S::LOG2E, S::TBT_WIDE, true>>(
        kind, p, stream);
}

template cudaError_t launch_r2r1<DFFT_T, DFFT_LOG2N>(PassKind, const FftR2r&, cudaStream_t);

// N = 2^(LOG2M + 1) reals per line, so the longest line (8192) runs 4096-point complex lines: no LOG2M = 13 unit
#if DFFT_LOG2N < 13
template <typename T, int LOG2M>
cudaError_t launch_r2r4(PassKind kind, const FftR2r& p, cudaStream_t stream) {
    using S = Shape<T, LOG2M>;
    return launch_real_lines<T, LOG2M, fft_r2r4_kernel<T, LOG2M, S::LOG2E, S::TBC, false>, fft_r2r4_kernel<T, LOG2M, S::LOG2E, S::TBT_WIDE, true>>(
        kind, p, stream);
}

template cudaError_t launch_r2r4<DFFT_T, DFFT_LOG2N>(PassKind, const FftR2r&, cudaStream_t);
#endif

#if DFFT_LOG2N == 1
// CONTIG: lines of up to COPY_THREADS threads (the power of two >= n), COPY_THREADS / that many lines per CTA; TILED: rows
// as wide as the power of two >= B, up to 32 elements (a 512-byte row of cx<double>), the CTA's other threads on further n
template <typename E>
cudaError_t launch_copy(PassKind kind, const FftCopy& p_in, cudaStream_t stream) {
    FftCopy p = p_in;
    const long long lines = (long long)p.A0 * p.A1;
    if (lines <= 0 || p.n <= 0) return cudaSuccess;
    const bool tiled = kind == PASS_COPY_TILED;
    if (!tiled && kind != PASS_COPY_CONTIG) return cudaErrorInvalidValue;
    if (tiled && p.B <= 0) return cudaSuccess;
    // TILED: G x G blocks of (a0, a1) tiles, the largest G <= 2^DFFT_COPY_SWZ that divides both extents
    p.tile_swz = 0;
    if (tiled) {
        p.tile_swz = env_int("DFFT_COPY_SWZ", COPY_SWZ);
        while (p.tile_swz > 0 && (p.A0 % (1 << p.tile_swz) || p.A1 % (1 << p.tile_swz))) --p.tile_swz;
    }
    const int span = tiled ? (p.B < 32 ? p.B : 32) : (p.n < COPY_THREADS ? p.n : COPY_THREADS);
    p.ltpl = 0;
    while ((1 << p.ltpl) < span) ++p.ltpl;
    const long long grid = tiled ? lines * ((p.B + (1 << p.ltpl) - 1) >> p.ltpl) : (lines + (COPY_THREADS >> p.ltpl) - 1) / (COPY_THREADS >> p.ltpl);
    if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    if (tiled) fft_copy_kernel<E, true><<<unsigned(grid), COPY_THREADS, 0, stream>>>(p);
    else fft_copy_kernel<E, false><<<unsigned(grid), COPY_THREADS, 0, stream>>>(p);
    return cudaGetLastError();
}

template cudaError_t launch_copy<DFFT_T>(PassKind, const FftCopy&, cudaStream_t);
template cudaError_t launch_copy<cx<DFFT_T>>(PassKind, const FftCopy&, cudaStream_t);
#endif

#if DFFT_LOG2N == 8 || DFFT_LOG2N == 9
static bool aligned128(const void* base, long long elems_a, long long elems_b, long long elems_c) {
    constexpr long long es = sizeof(cx<DFFT_T>);
    return reinterpret_cast<unsigned long long>(base) % 128 == 0 && (elems_a * es) % 128 == 0 && (elems_b * es) % 128 == 0 && (elems_c * es) % 128 == 0;
}

template <typename T, int LOG2N>
cudaError_t launch_zy_fused(const FftParams& pz, const FftParams& py, const ZyFused& f_in, double scale, cudaStream_t stream) {
    static_assert(zy_fused_length(LOG2N), "fused z + y stage: length not instantiated");
    using Z = ZyShape<T, LOG2N>;
    constexpr int TB = Z::TB;
    const bool inv = pz.inverse != 0;
    if (pz.in.nseg != 1 || pz.out.nseg != 1 || py.in.nseg != 1 || py.out.nseg != 1 || pz.in.sN != 1 || pz.out.sN != 1) return cudaErrorInvalidValue;
    if (pz.inverse != py.inverse || py.tile_swz != 0 || pz.A0 != py.A0 || pz.A1 % TB || py.B % TB || f_in.order.nx != pz.A0 || f_in.order.gpp < 1 || f_in.order.ahead < 1)
        return cudaErrorInvalidValue;
    if (scale != 1.0 && !inv) return cudaErrorInvalidValue;  // the forward stage stores the x pass' input
    ZyFused f = f_in;
    const int z_per_plane = pz.A1 / TB, y_per_plane = py.A1 * (py.B / TB);  // tiles = work items
    f.order.na = inv ? y_per_plane : z_per_plane;
    f.order.nb = inv ? z_per_plane : y_per_plane;
    // phase B reads the intermediate: forward the y tiles (rows of TB elements sN apart), inverse the z lines.  A phase B
    // that stores where it reads (in place, as the inverse of an in-place plan does) would drop its own results: no
    // discard then.
    const View& mid = inv ? pz.in : py.in;
    const bool in_place = mid.seg[0].base == (inv ? pz.out : py.out).seg[0].base;
    f.discard = !in_place && (inv ? (Z::Z_DISCARD && aligned128(mid.seg[0].base, mid.seg[0].sA0, mid.seg[0].sA1, 1 << LOG2N))
                                  : (Z::Y_DISCARD && aligned128(mid.seg[0].base, mid.seg[0].sA0, mid.seg[0].sA1, mid.sN)));
    // persistent: as many CTAs as fit at once (tickets hand out the work; fewer resident CTAs are fine as well).  The
    // grid depends on the work list only, so every launch of a step draws the same number of tickets (zy_launch_of) —
    // also when one exec runs the fed kernel and the next the register-fed one: the grid is the smaller residency of both.
    constexpr auto kf_reg = fft_zy_fused_kernel<T, LOG2N, false, false>;
    constexpr auto kis_reg = fft_zy_fused_kernel<T, LOG2N, true, true>;
    static const int resident_reg = resident_ctas(kf_reg, Z::THREADS, Z::SMEM_BYTES);
    int resident = resident_reg;
    const long long total = f.order.total();
    if (total <= 0) return cudaSuccess;
    if constexpr (sizeof(T) == 8) {
        // f64: inputs by asynchronous copies wherever the views are 16-byte aligned — z lines (pz.in) by bulk copies, y tiles
        // by a tensor map of py.in, encoded here per exec because py.in may be the caller's buffer (inverse).  An aligned
        // view whose map cannot be encoded is an error, not a quiet switch to the register-fed kernel.  DFFT_ZY_FEED=0
        // forces the register-fed kernel (comparison of the two).  f32 keeps the register-fed kernel: fed, its
        // 64-register budget spills and the inverse stage was slower (DESIGN.md section 3.4).
        constexpr auto kf = fft_zy_fed_kernel<T, LOG2N, false, false>;
        static const int resident_fed = resident_ctas(kf, Z::THREADS, Z::SMEM_BYTES);
        if (resident_fed < resident) resident = resident_fed;
        const unsigned grid = unsigned(total < resident ? total : resident);
        constexpr unsigned long long es = sizeof(cx<T>);
        const auto a16 = [](unsigned long long v) { return v % 16 == 0; };
        const Seg& gz = pz.in.seg[0];
        const Seg& gy = py.in.seg[0];
        const bool aligned = a16(reinterpret_cast<unsigned long long>(gz.base)) && a16(gz.sA0 * es) && a16(gz.sA1 * es) &&
                             a16(reinterpret_cast<unsigned long long>(gy.base)) && a16(gy.sA0 * es) && a16(gy.sA1 * es) && a16(py.in.sN * es);
        if (env_int("DFFT_ZY_FEED", 1) != 0 && aligned) {
            alignas(64) CUtensorMap tm;
            if (!make_view_map<T>(py.in, py.A0, py.A1, 1 << LOG2N, py.B, TB, &tm)) return cudaErrorNotSupported;
            // only the inverse stage has a scaled twin (a scaled forward stage is refused above)
            constexpr auto kis = fft_zy_fed_kernel<T, LOG2N, true, true>;
            return launch_kernel<kf, fft_zy_fed_kernel<T, LOG2N, true, false>, kis, kis>(pz, scale, grid, Z::THREADS, Z::SMEM_BYTES, stream, py, f, tm);
        }
    }
    const unsigned grid = unsigned(total < resident ? total : resident);
    return launch_kernel<kf_reg, fft_zy_fused_kernel<T, LOG2N, true, false>, kis_reg, kis_reg>(pz, scale, grid, Z::THREADS, Z::SMEM_BYTES, stream, py, f);
}

template cudaError_t launch_zy_fused<DFFT_T, DFFT_LOG2N>(const FftParams&, const FftParams&, const ZyFused&, double, cudaStream_t);
#endif

#if DFFT_LOG2N == 5 || DFFT_LOG2N == 6
template <typename T, int LOG2N>
cudaError_t launch_batch_small(const void* in, void* out, long long batch, int inverse, const BatchSmall& f_in, double scale, cudaStream_t stream) {
    static_assert(batch_small_length(LOG2N), "batched small fields: length not instantiated");
    using BS = BatchShape<T, LOG2N>;
    constexpr long long N = BS::N, N2 = N * N, N3 = N2 * N;
    if (batch < 1 || batch * N > 0x7fffffffLL || f_in.order.ahead < 1 || !f_in.ctr) return cudaErrorInvalidValue;
    BatchSmall f = f_in;
    const int items = int(N3 / BS::POINTS);  // plane items = slice items per field
    f.order.nx = int(batch);
    f.order.gpp = 1;
    f.order.na = items;
    f.order.nb = items;
    f.plane_in = inverse ? out : in;
    f.plane_out = out;
    FftParams px{};
    px.A0 = int(batch); px.A1 = 1; px.B = int(N2);
    px.inverse = inverse;
    px.tw = f.tw;
    for (View* v : {&px.in, &px.out}) {
        v->nseg = 1;
        v->sN = N2;
        v->seg[0].sA0 = N3;
    }
    px.in.seg[0].base = inverse ? const_cast<void*>(in) : out;
    px.out.seg[0].base = out;
    // persistent, as many CTAs as fit at once; the grid depends on the batch only (zy_launch_of)
    constexpr auto kf = fft_batch_small_kernel<T, LOG2N, false, false>;
    static const int resident = resident_ctas(kf, BS::THREADS, BS::SMEM_BYTES);
    const long long total = f.order.total();
    const unsigned grid = unsigned(total < resident ? total : resident);
    return launch_kernel<kf, fft_batch_small_kernel<T, LOG2N, true, false>, fft_batch_small_kernel<T, LOG2N, false, true>,
                         fft_batch_small_kernel<T, LOG2N, true, true>>(px, scale, grid, BS::THREADS, BS::SMEM_BYTES, stream, f);
}

template cudaError_t launch_batch_small<DFFT_T, DFFT_LOG2N>(const void*, void*, long long, int, const BatchSmall&, double, cudaStream_t);
#endif

#endif  // DFFT_S

}  // namespace dfft
