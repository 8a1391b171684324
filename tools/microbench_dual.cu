// tools/microbench_dual.cu — can the fp64 tensor pipe (DMMA, mma.sync f64) and the fp64 ALU pipe (DFMA) run at the same
// time on sm_90a, and how much of each?  Three arrangements, all register resident (no memory traffic):
//   split : W_T warps of a CTA issue only DMMA, W_A warps only DFMA (warp specialisation);
//   mixed : every warp interleaves R DFMA per DMMA.8x8x4 in its instruction stream;
// Prints one JSON object.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench_dual tools/microbench_dual.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// warps [0, wt) : DMMA; warps [wt, wt + wa) : DFMA.  Roles are interleaved over the 4 SM sub-partitions (warp w runs on
// sub-partition w % 4), so put DMMA warps first: with wt, wa multiples of 4 every sub-partition gets wt/4 + wa/4 warps.
__global__ void split_kernel(double* out, int iters, int wt)
{
    const int warp = threadIdx.x >> 5;
    double s = 0;
    if (warp < wt) {
        double c[16][2];
        for (int i = 0; i < 16; ++i) c[i][0] = c[i][1] = 0.0;
        const double a = 1e-3 * threadIdx.x, b = 2e-3;
        for (int it = 0; it < iters; ++it) {
#pragma unroll
            for (int i = 0; i < 16; ++i) dmma884(c[i][0], c[i][1], a, b);
        }
        for (int i = 0; i < 16; ++i) s += c[i][0] + c[i][1];
    }
    else {
        double c[32];
        for (int i = 0; i < 32; ++i) c[i] = threadIdx.x * 1e-3 + i;
        const double a = 1.0000001, b = 1e-9;
        for (int it = 0; it < iters; ++it) {
#pragma unroll
            for (int i = 0; i < 32; ++i) c[i] = fma(c[i], a, b);
        }
        for (int i = 0; i < 32; ++i) s += c[i];
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// every warp: per iteration 16 DMMA.8x8x4 and 16 * R DFMA (independent accumulators), interleaved
template <int R>
__global__ void mixed_kernel(double* out, int iters)
{
    double c[16][2], f[16 * (R > 0 ? R : 1) > 48 ? 48 : 16 * (R > 0 ? R : 1)];
    constexpr int NF = 16 * (R > 0 ? R : 1) > 48 ? 48 : 16 * (R > 0 ? R : 1);
    for (int i = 0; i < 16; ++i) c[i][0] = c[i][1] = 0.0;
    for (int i = 0; i < NF; ++i) f[i] = threadIdx.x * 1e-3 + i;
    const double a = 1e-3 * threadIdx.x, b = 2e-3, fa = 1.0000001, fb = 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            dmma884(c[i][0], c[i][1], a, b);
#pragma unroll
            for (int r = 0; r < R; ++r) { const int j = (i * R + r) % NF; f[j] = fma(f[j], fa, fb); }
        }
    }
    double s = 0;
    for (int i = 0; i < 16; ++i) s += c[i][0] + c[i][1];
    for (int i = 0; i < NF; ++i) s += f[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

static float time_it(void (*launch)(int), int iters)
{
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch(50);
    cudaDeviceSynchronize();
    float best = 1e30f, ms;
    for (int r = 0; r < 3; ++r) {
        cudaEventRecord(e0);
        launch(iters);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    return best;
}

static double* g_out;
static int g_sms, g_wt, g_wa;
static void launch_split(int iters) { split_kernel<<<g_sms, (g_wt + g_wa) * 32>>>(g_out, iters, g_wt); }
template <int R> static void launch_mixed(int iters) { mixed_kernel<R><<<g_sms * 2, 256>>>(g_out, iters); }

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    g_sms = prop.multiProcessorCount;
    CK(cudaMalloc(&g_out, sizeof(double) * g_sms * 2 * 1024));
    const int iters = 20000;
    printf("{\"gpu\": \"%s\", \"sms\": %d, \"split\": [", prop.name, g_sms);
    const int cfgs[][2] = {{8, 0}, {0, 8}, {8, 8}, {8, 4}, {16, 0}, {0, 16}, {16, 8}, {16, 16}, {8, 16}, {12, 4}, {4, 4}};
    bool first = true;
    for (auto& c : cfgs) {
        g_wt = c[0]; g_wa = c[1];
        float ms = time_it(launch_split, iters);
        CK(cudaGetLastError());
        const double tf_t = (double)g_sms * g_wt * iters * 16.0 * 512.0 / (ms * 1e-3) / 1e12;
        const double tf_a = (double)g_sms * g_wa * 32 * iters * 32.0 * 2.0 / (ms * 1e-3) / 1e12;
        printf("%s{\"dmma_warps\": %d, \"dfma_warps\": %d, \"ms\": %.3f, \"dmma_tflops\": %.2f, \"dfma_tflops\": %.2f, \"total_tflops\": %.2f}", first ? "" : ", ",
            g_wt, g_wa, ms, tf_t, tf_a, tf_t + tf_a);
        first = false;
    }
    printf("], \"mixed\": [");
    auto report = [&](int R, float ms) {
        const double warps = (double)g_sms * 2 * 8;
        const double tf_t = warps * iters * 16.0 * 512.0 / (ms * 1e-3) / 1e12;
        const double tf_a = warps * 32 * iters * 16.0 * R * 2.0 / (ms * 1e-3) / 1e12;
        printf("%s{\"dfma_per_dmma\": %d, \"ms\": %.3f, \"dmma_tflops\": %.2f, \"dfma_tflops\": %.2f, \"total_tflops\": %.2f}", R ? ", " : "", R, ms, tf_t, tf_a,
            tf_t + tf_a);
    };
    report(0, time_it(launch_mixed<0>, iters));
    report(1, time_it(launch_mixed<1>, iters));
    report(2, time_it(launch_mixed<2>, iters));
    report(4, time_it(launch_mixed<4>, iters));
    report(8, time_it(launch_mixed<8>, iters));
    printf("]}\n");
    return 0;
}
