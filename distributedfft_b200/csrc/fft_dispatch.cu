// fft_dispatch.cu — runtime length -> compile-time instantiation (see fft_inst.cu).
#include "fft_kernels.cuh"

namespace dfft {

#define DFFT_DECL(T, L) extern template cudaError_t launch_pass<T, L>(PassKind, const FftParams&, double, cudaStream_t);
#define DFFT_ALL(M, T) M(T, 1) M(T, 2) M(T, 3) M(T, 4) M(T, 5) M(T, 6) M(T, 7) M(T, 8) M(T, 9) M(T, 10) M(T, 11) M(T, 12) M(T, 13)
DFFT_ALL(DFFT_DECL, double)
DFFT_ALL(DFFT_DECL, float)

#define DFFT_CASE(T, L) \
    case L: return launch_pass<T, L>(kind, p, scale, stream);

cudaError_t launch_pass_f64(int log2n, PassKind kind, const FftParams& p, double scale, cudaStream_t stream) {
    switch (log2n) {
        DFFT_ALL(DFFT_CASE, double)
        default: return cudaErrorInvalidValue;
    }
}
cudaError_t launch_pass_f32(int log2n, PassKind kind, const FftParams& p, double scale, cudaStream_t stream) {
    switch (log2n) {
        DFFT_ALL(DFFT_CASE, float)
        default: return cudaErrorInvalidValue;
    }
}

#define DFFT_BLU_DECL(T, L) extern template cudaError_t launch_bluestein<T, L>(PassKind, const FftBluestein&, cudaStream_t);
#define DFFT_BLU_ALL(M, T) M(T, 3) M(T, 4) M(T, 5) M(T, 6) M(T, 7) M(T, 8) M(T, 9) M(T, 10) M(T, 11) M(T, 12) M(T, 13)
DFFT_BLU_ALL(DFFT_BLU_DECL, double)
DFFT_BLU_ALL(DFFT_BLU_DECL, float)

#define DFFT_BLU_CASE(T, L) \
    case L: return launch_bluestein<T, L>(kind, p, stream);

cudaError_t launch_bluestein_f64(int log2m, PassKind kind, const FftBluestein& p, cudaStream_t stream) {
    switch (log2m) {
        DFFT_BLU_ALL(DFFT_BLU_CASE, double)
        default: return cudaErrorInvalidValue;
    }
}
cudaError_t launch_bluestein_f32(int log2m, PassKind kind, const FftBluestein& p, cudaStream_t stream) {
    switch (log2m) {
        DFFT_BLU_ALL(DFFT_BLU_CASE, float)
        default: return cudaErrorInvalidValue;
    }
}

#define DFFT_ZY_DECL(T, L) \
    extern template cudaError_t launch_zy_fused<T, L>(const FftParams&, const FftParams&, const ZyFused&, double, cudaStream_t);
DFFT_ZY_DECL(double, 8) DFFT_ZY_DECL(double, 9) DFFT_ZY_DECL(float, 8) DFFT_ZY_DECL(float, 9)

cudaError_t launch_zy_fused_f64(int log2n, const FftParams& pz, const FftParams& py, const ZyFused& f, double scale, cudaStream_t stream) {
    switch (log2n) {
        case 8: return launch_zy_fused<double, 8>(pz, py, f, scale, stream);
        case 9: return launch_zy_fused<double, 9>(pz, py, f, scale, stream);
        default: return cudaErrorInvalidValue;
    }
}
cudaError_t launch_zy_fused_f32(int log2n, const FftParams& pz, const FftParams& py, const ZyFused& f, double scale, cudaStream_t stream) {
    switch (log2n) {
        case 8: return launch_zy_fused<float, 8>(pz, py, f, scale, stream);
        case 9: return launch_zy_fused<float, 9>(pz, py, f, scale, stream);
        default: return cudaErrorInvalidValue;
    }
}

#define DFFT_BATCH_DECL(T, L) \
    extern template cudaError_t launch_batch_small<T, L>(const void*, void*, long long, int, const BatchSmall&, double, cudaStream_t);
DFFT_BATCH_DECL(double, 5) DFFT_BATCH_DECL(double, 6) DFFT_BATCH_DECL(float, 5) DFFT_BATCH_DECL(float, 6)

cudaError_t launch_batch_small_f64(int log2n, const void* in, void* out, long long batch, int inverse, const BatchSmall& f, double scale, cudaStream_t stream) {
    switch (log2n) {
        case 5: return launch_batch_small<double, 5>(in, out, batch, inverse, f, scale, stream);
        case 6: return launch_batch_small<double, 6>(in, out, batch, inverse, f, scale, stream);
        default: return cudaErrorInvalidValue;
    }
}
cudaError_t launch_batch_small_f32(int log2n, const void* in, void* out, long long batch, int inverse, const BatchSmall& f, double scale, cudaStream_t stream) {
    switch (log2n) {
        case 5: return launch_batch_small<float, 5>(in, out, batch, inverse, f, scale, stream);
        case 6: return launch_batch_small<float, 6>(in, out, batch, inverse, f, scale, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace dfft
