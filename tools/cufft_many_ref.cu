// cufft_many_ref.cu — cuFFT reference for batched 3D transforms: one cufftPlanMany (rank 3, contiguous fields back to
// back) and its exec.  Measurement and test helper only, compiled at run time into a temporary directory by
// tools/batch_bench.py and tests/test_gpu_batch.py:
//     nvcc -gencode arch=compute_90a,code=sm_90a -shared -Xcompiler -fPIC cufft_many_ref.cu -lcufft -o libcufft_many_ref.so
// kind: 0 forward, 1 inverse (C2C / Z2Z).  prec: 0 f32, 1 f64.  ms: mean time of `reps` execs after one warm-up.
#include <cuda_runtime.h>
#include <cufft.h>

extern "C" int cufft_ref_3d_many(int prec, int kind, int nx, int ny, int nz, int batch, void* out, void* in, float* ms, int reps) {
    cufftHandle plan;
    int n[3] = {nx, ny, nz};
    if (cufftPlanMany(&plan, 3, n, nullptr, 1, nx * ny * nz, nullptr, 1, nx * ny * nz, prec ? CUFFT_Z2Z : CUFFT_C2C, batch) != CUFFT_SUCCESS) return -1;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    int rc = 0;
    if (reps < 1) reps = 1;
    const int dir = kind == 0 ? CUFFT_FORWARD : CUFFT_INVERSE;
    for (int r = 0; r < reps + 1; ++r) {
        if (r == 1) cudaEventRecord(e0);
        const cufftResult res = prec ? cufftExecZ2Z(plan, (cufftDoubleComplex*)in, (cufftDoubleComplex*)out, dir)
                                     : cufftExecC2C(plan, (cufftComplex*)in, (cufftComplex*)out, dir);
        if (res != CUFFT_SUCCESS) rc = -2;
    }
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float t = 0;
    cudaEventElapsedTime(&t, e0, e1);
    if (ms) *ms = t / reps;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cufftDestroy(plan);
    if (cudaDeviceSynchronize() != cudaSuccess) rc = -3;
    return rc;
}
