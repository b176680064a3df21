// fft_dispatch.cu — runtime (precision, log2 length) -> compile-time instantiation (see fft_inst.cu).
#include <type_traits>
#include <utility>

#include "../../include/dfft.h"
#include "fft_kernels.cuh"

namespace dfft {

// launch(T(), std::integral_constant<int, L>()) for T = double (prec == DFFT_F64) or float and L = log2n in [LO, HI];
// cudaErrorInvalidValue for a length outside the range
template <int LO, int HI, typename F, int... I>
static cudaError_t dispatch(int prec, int log2n, const F& launch, std::integer_sequence<int, I...>) {
    cudaError_t e = cudaErrorInvalidValue;
    (void)((log2n == LO + I && (e = prec == DFFT_F64 ? launch(double(), std::integral_constant<int, LO + I>())
                                                      : launch(float(), std::integral_constant<int, LO + I>()),
                                true)) ||
           ...);
    return e;
}
template <int LO, int HI, typename F>
static cudaError_t dispatch(int prec, int log2n, const F& launch) {
    return dispatch<LO, HI>(prec, log2n, launch, std::make_integer_sequence<int, HI - LO + 1>());
}

cudaError_t launch_pass(int prec, int log2n, PassKind kind, const FftParams& p, double scale, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N>(prec, log2n, [&](auto t, auto l) { return launch_pass<decltype(t), decltype(l)::value>(kind, p, scale, stream); });
}

cudaError_t launch_padded(int prec, int log2n, PassKind kind, const FftPadded& p, cudaStream_t stream) {
    return dispatch<1, MAX_LOG2N>(prec, log2n, [&](auto t, auto l) { return launch_padded<decltype(t), decltype(l)::value>(kind, p, stream); });
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
