// graph_capture_test.cu — capture of one-rank plans into a CUDA graph through the C ABI (include/dfft.h) with the raw
// runtime calls a C++ caller uses: cudaStreamBeginCapture / cudaStreamEndCapture / cudaGraphInstantiate /
// cudaGraphLaunch.  A graph holding forward then inverse is replayed on fresh input several times and compared byte for
// byte (memcmp) with eager execs of the same plan on the same input; eager execs and replays alternate on one stream.
// A capture before any eager exec of the direction is refused with DFFT_ERR_STATE, and the plan still works after it.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -Iinclude graph_capture_test.cu -Ldistributedfft_b200 -ldfft
#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "dfft.h"

#define CUDA_CALL(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { std::printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return 2; } } while (0)
#define DFFT_OK(x) do { int r_ = (x); if (r_ != DFFT_SUCCESS) { std::printf("dfft error %d (%s) at %s:%d\n", r_, dfft_last_error_string(), __FILE__, __LINE__); return 2; } } while (0)

static void fill(std::vector<double>& h, unsigned seed) {
    unsigned long long s = 0x9E3779B97F4A7C15ull * (seed + 1);
    for (double& v : h) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        v = double(s >> 11) * (1.0 / 9007199254740992.0) * 255.0;
    }
}

// forward (in -> out) then inverse (out -> back) of one C2C or R2C/C2R plan
static int enqueue(dfft_plan_t plan, bool c2c, void* out, void* back, const void* in, cudaStream_t s) {
    int r = c2c ? dfft_exec_c2c_async(plan, out, in, DFFT_FORWARD, s) : dfft_exec_r2c_async(plan, out, in, s);
    if (r != DFFT_SUCCESS) return r;
    return c2c ? dfft_exec_c2c_async(plan, back, out, DFFT_INVERSE, s) : dfft_exec_c2r_async(plan, back, out, s);
}

// complex-double plans
static int round_trip(dfft_comm_t comm, const char* name, int decomp, int transform, size_t nx, size_t ny, size_t nz) {
    dfft_config cfg{1, 0, DFFT_PEER2PEER, DFFT_SEND_SYNC, nullptr, DFFT_PEER2PEER, DFFT_SEND_SYNC};
    dfft_plan_t plan = nullptr;
    DFFT_OK(dfft_plan_create(comm, &cfg, decomp, DFFT_F64, transform, nx, ny, nz, 1, 1, 1, &plan));
    const bool c2c = transform == DFFT_C2C;
    size_t isz[3];
    DFFT_OK(dfft_get_in_size(plan, isz));
    const size_t in_bytes = isz[0] * isz[1] * isz[2] * sizeof(double) * (c2c ? 2 : 1);
    const size_t dom = dfft_get_domain_size(plan);
    void *in_d, *out_d, *back_d;
    CUDA_CALL(cudaMalloc(&in_d, in_bytes));
    CUDA_CALL(cudaMalloc(&out_d, dom));
    CUDA_CALL(cudaMalloc(&back_d, in_bytes));
    cudaStream_t s;
    CUDA_CALL(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));

    std::vector<double> gen(in_bytes / 8);
    std::vector<unsigned char> ref_out(dom), ref_back(in_bytes), got_out(dom), got_back(in_bytes);
    // on `s`: s does not synchronise with the legacy default stream, and a pageable cudaMemcpy may return before its DMA
    // has landed
    auto refill = [&](unsigned seed) -> cudaError_t {
        fill(gen, seed);
        return cudaMemcpyAsync(in_d, gen.data(), in_bytes, cudaMemcpyHostToDevice, s);
    };

    // warm-up: one eager exec of each direction
    CUDA_CALL(refill(0));
    DFFT_OK(enqueue(plan, c2c, out_d, back_d, in_d, s));
    CUDA_CALL(cudaStreamSynchronize(s));
    DFFT_OK(dfft_plan_wait(plan));
    const int eager_launches = dfft_get_last_launch_count(plan);

    cudaGraph_t graph;
    cudaGraphExec_t exec;
    CUDA_CALL(cudaStreamBeginCapture(s, cudaStreamCaptureModeGlobal));
    const int rc = enqueue(plan, c2c, out_d, back_d, in_d, s);
    CUDA_CALL(cudaStreamEndCapture(s, &graph));
    if (rc != DFFT_SUCCESS) {
        std::printf("%s: capture failed: %d (%s)\n", name, rc, dfft_last_error_string());
        return 1;
    }
    CUDA_CALL(cudaGraphInstantiate(&exec, graph, 0));
    int fails = 0;
    if (dfft_get_last_launch_count(plan) != eager_launches) {
        std::printf("%s: a capture changed the launch count\n", name);
        ++fails;
    }
    for (unsigned rep = 1; rep <= 3; ++rep) {
        CUDA_CALL(refill(rep));
        DFFT_OK(enqueue(plan, c2c, out_d, back_d, in_d, s));  // eager
        CUDA_CALL(cudaMemcpyAsync(ref_out.data(), out_d, dom, cudaMemcpyDeviceToHost, s));
        CUDA_CALL(cudaMemcpyAsync(ref_back.data(), back_d, in_bytes, cudaMemcpyDeviceToHost, s));
        CUDA_CALL(cudaMemsetAsync(out_d, 0, dom, s));
        CUDA_CALL(cudaMemsetAsync(back_d, 0, in_bytes, s));
        CUDA_CALL(cudaGraphLaunch(exec, s));  // replay
        CUDA_CALL(cudaMemcpyAsync(got_out.data(), out_d, dom, cudaMemcpyDeviceToHost, s));
        CUDA_CALL(cudaMemcpyAsync(got_back.data(), back_d, in_bytes, cudaMemcpyDeviceToHost, s));
        CUDA_CALL(cudaStreamSynchronize(s));
        if (std::memcmp(ref_out.data(), got_out.data(), dom) || std::memcmp(ref_back.data(), got_back.data(), in_bytes)) {
            std::printf("%s: replay %u differs from the eager exec\n", name, rep);
            ++fails;
        }
    }
    DFFT_OK(dfft_plan_wait(plan));
    std::printf("%s %zux%zux%zu: %d launches per exec, 3 replays %s\n", name, nx, ny, nz, eager_launches, fails ? "DIFFER" : "bit-identical");
    cudaGraphExecDestroy(exec);
    cudaGraphDestroy(graph);
    cudaStreamDestroy(s);
    cudaFree(in_d); cudaFree(out_d); cudaFree(back_d);
    dfft_plan_destroy(plan);
    return fails ? 1 : 0;
}

// a capture before any eager exec of the direction: refused, nothing captured, the plan works eagerly afterwards
static int refusal(dfft_comm_t comm) {
    dfft_config cfg{1, 0, DFFT_PEER2PEER, DFFT_SEND_SYNC, nullptr, DFFT_PEER2PEER, DFFT_SEND_SYNC};
    dfft_plan_t plan = nullptr;
    const size_t n = 64, bytes = n * n * n * 16;
    DFFT_OK(dfft_plan_create(comm, &cfg, DFFT_SLAB_ZY_THEN_X, DFFT_F64, DFFT_C2C, n, n, n, 1, 1, 1, &plan));
    void *in_d, *out_d;
    CUDA_CALL(cudaMalloc(&in_d, bytes));
    CUDA_CALL(cudaMalloc(&out_d, bytes));
    cudaStream_t s;
    CUDA_CALL(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    CUDA_CALL(cudaMemsetAsync(in_d, 0, bytes, s));
    cudaGraph_t graph;
    CUDA_CALL(cudaStreamBeginCapture(s, cudaStreamCaptureModeGlobal));
    const int rc = dfft_exec_c2c_async(plan, out_d, in_d, DFFT_FORWARD, s);
    CUDA_CALL(cudaStreamEndCapture(s, &graph));
    size_t nodes = 1;
    CUDA_CALL(cudaGraphGetNodes(graph, nullptr, &nodes));
    cudaGraphDestroy(graph);
    int fails = 0;
    if (rc != DFFT_ERR_STATE || nodes != 0) {
        std::printf("capture before an eager exec: rc %d, %zu nodes (expected DFFT_ERR_STATE, 0)\n", rc, nodes);
        ++fails;
    }
    DFFT_OK(dfft_exec_c2c_async(plan, out_d, in_d, DFFT_FORWARD, s));
    CUDA_CALL(cudaStreamSynchronize(s));
    DFFT_OK(dfft_plan_wait(plan));
    std::printf("refusal before warm-up: %s\n", fails ? "WRONG" : "DFFT_ERR_STATE, empty graph, eager exec fine");
    cudaStreamDestroy(s);
    cudaFree(in_d); cudaFree(out_d);
    dfft_plan_destroy(plan);
    return fails ? 1 : 0;
}

int main() {
    dfft_comm_t comm;
    DFFT_OK(dfft_comm_create(0, 1, nullptr, 0, &comm));
    int rc = 0;
    rc |= round_trip(comm, "slab C2C f64 (fused z + y)", DFFT_SLAB_ZY_THEN_X, DFFT_C2C, 64, 512, 512);
    rc |= round_trip(comm, "slab R2C/C2R f64", DFFT_SLAB_ZY_THEN_X, DFFT_R2C, 128, 128, 128);
    rc |= refusal(comm);
    dfft_comm_destroy(comm);
    std::printf(rc ? "FAILED\n" : "PASSED\n");
    return rc;
}
