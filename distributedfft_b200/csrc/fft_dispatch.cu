// fft_dispatch.cu — runtime (precision, log2 length) -> compile-time instantiation (see fft_inst.cu).
#include <type_traits>
#include <utility>

#include "../../include/dfft.h"
#include "fft_kernels.cuh"

namespace dfft {

// launch(T(), std::integral_constant<int, L>()) for T = double (prec == DFFT_F64) or float (DFFT_F32) and L = log2n in [LO, HI];
// with HALF, also T = __half (DFFT_F16) and __nv_bfloat16 (DFFT_BF16), the stored type of 16-bit plans.  cudaErrorInvalidValue
// for a length outside the range, and for a 16-bit precision without HALF (the launchers of 16-bit plans: launch_pass only).
template <int LO, int HI, bool HALF, typename F, int... I>
static cudaError_t dispatch(int prec, int log2n, const F& launch, std::integer_sequence<int, I...>) {
    cudaError_t e = cudaErrorInvalidValue;
    auto one = [&](auto l) -> cudaError_t {
        if constexpr (HALF) {
            if (prec == DFFT_F16) return launch(__half(), l);
            if (prec == DFFT_BF16) return launch(__nv_bfloat16(), l);
        }
        if (prec == DFFT_F64) return launch(double(), l);
        if (prec == DFFT_F32) return launch(float(), l);
        return cudaErrorInvalidValue;
    };
    (void)((log2n == LO + I && (e = one(std::integral_constant<int, LO + I>()), true)) || ...);
    return e;
}
template <int LO, int HI, bool HALF = false, typename F>
static cudaError_t dispatch(int prec, int log2n, const F& launch) {
    return dispatch<LO, HI, HALF>(prec, log2n, launch, std::make_integer_sequence<int, HI - LO + 1>());
}

cudaError_t launch_pass(int prec, int log2n, PassKind kind, const FftParams& p, double scale, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N, true>(prec, log2n, [&](auto t, auto l) {
        using T = decltype(t);
        if constexpr (std::is_same_v<T, __half> || std::is_same_v<T, __nv_bfloat16>) return launch_pass<float, cx16<T>, decltype(l)::value>(kind, p, scale, stream);
        else return launch_pass<T, cx<T>, decltype(l)::value>(kind, p, scale, stream);
    });
}

cudaError_t launch_twin(int prec, int log2n, PassKind kind, const FftPadded& p, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N>(prec, log2n, [&](auto t, auto l) { return launch_twin<decltype(t), decltype(l)::value>(kind, p, stream); });
}

cudaError_t launch_bluestein(int prec, int log2m, PassKind kind, const FftBluestein& p, cudaStream_t stream) {
    return dispatch<3, MAX_LOG2N>(prec, log2m, [&](auto t, auto l) { return launch_bluestein<decltype(t), decltype(l)::value>(kind, p, stream); });
}

cudaError_t launch_r2r(int prec, int log2n, PassKind kind, const FftR2r& p, bool hc, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N>(prec, log2n, [&](auto t, auto l) { return launch_r2r<decltype(t), decltype(l)::value>(kind, p, hc, stream); });
}

cudaError_t launch_r2r1(int prec, int log2n, PassKind kind, const FftR2r& p, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N>(prec, log2n, [&](auto t, auto l) { return launch_r2r1<decltype(t), decltype(l)::value>(kind, p, stream); });
}

cudaError_t launch_r2r4(int prec, int log2m, PassKind kind, const FftR2r& p, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N - 1>(prec, log2m, [&](auto t, auto l) { return launch_r2r4<decltype(t), decltype(l)::value>(kind, p, stream); });
}

cudaError_t launch_copy(int prec, bool real, PassKind kind, const FftCopy& p, cudaStream_t stream) {
    // 16-bit plans: complex elements of 4 bytes, never scaled by a copy (dfft_plan_set_scale)
    if (prec == DFFT_F16 || prec == DFFT_BF16) return real || p.scale != 1.0 ? cudaErrorInvalidValue : launch_copy<float>(kind, p, stream);
    if (prec == DFFT_F64) return real ? launch_copy<double>(kind, p, stream) : launch_copy<cx<double>>(kind, p, stream);
    return real ? launch_copy<float>(kind, p, stream) : launch_copy<cx<float>>(kind, p, stream);
}

cudaError_t launch_zy_fused(int prec, int log2n, const FftParams& pz, const FftParams& py, const ZyFused& f, double scale, cudaStream_t stream) {
    return dispatch<8, 9>(prec, log2n, [&](auto t, auto l) { return launch_zy_fused<decltype(t), decltype(l)::value>(pz, py, f, scale, stream); });
}

cudaError_t launch_batch_small(int prec, int log2n, const void* in, void* out, long long batch, int inverse, const BatchSmall& f, double scale,
                               cudaStream_t stream) {
    return dispatch<5, 6>(prec, log2n,
                          [&](auto t, auto l) { return launch_batch_small<decltype(t), decltype(l)::value>(in, out, batch, inverse, f, scale, stream); });
}

}  // namespace dfft
