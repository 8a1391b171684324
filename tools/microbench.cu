// tools/microbench.cu — measures the fp64 roofline denominators this backend is
// judged against on the actual box (MEASURED_PEAKS.json only holds HBM copy and
// bf16): DMMA (mma.sync f64) and DFMA peak, HBM write-only and copy bandwidth,
// and the DMMA rate of each f64 mma.sync shape (m8n8k4, m16n8k4/8/16).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench tools/microbench.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__global__ void dmma_kernel(double* out, int iters)
{
    double c[8][4];
    double a[4], b[2];
    for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) c[i][j] = 0.0;
    for (int j = 0; j < 4; ++j) a[j] = 1e-3 * (threadIdx.x + j);
    b[0] = 1e-3 * threadIdx.x; b[1] = 2e-3;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
            asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                         : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
                         : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    }
    double s = 0;
    for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) s += c[i][j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// One f64 mma.sync shape, CH independent accumulator chains per warp (as the GEMM core keeps 2 x NT tiles in flight).
//   S = 0: m8n8k4   S = 1: m16n8k4   S = 2: m16n8k8   S = 3: m16n8k16
template <int S>
struct Shape;
template <>
struct Shape<0> { static constexpr int NA = 1, NB = 1, NC = 2, FLOP = 2 * 8 * 8 * 4; static constexpr const char* name = "m8n8k4"; };
template <>
struct Shape<1> { static constexpr int NA = 2, NB = 1, NC = 4, FLOP = 2 * 16 * 8 * 4; static constexpr const char* name = "m16n8k4"; };
template <>
struct Shape<2> { static constexpr int NA = 4, NB = 2, NC = 4, FLOP = 2 * 16 * 8 * 8; static constexpr const char* name = "m16n8k8"; };
template <>
struct Shape<3> { static constexpr int NA = 8, NB = 4, NC = 4, FLOP = 2 * 16 * 8 * 16; static constexpr const char* name = "m16n8k16"; };

template <int S>
__device__ __forceinline__ void mma_shape(double* c, const double* a, const double* b)
{
    if (S == 0)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                     : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
    else if (S == 1)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if (S == 2)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, "
                     "{%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

template <int S, int CH>
__global__ void dmma_shape_kernel(double* out, int iters)
{
    using SH = Shape<S>;
    double c[CH][SH::NC], a[SH::NA], b[SH::NB];
#pragma unroll
    for (int i = 0; i < CH; ++i)
#pragma unroll
        for (int j = 0; j < SH::NC; ++j) c[i][j] = 0.0;
#pragma unroll
    for (int j = 0; j < SH::NA; ++j) a[j] = 1e-3 * (threadIdx.x + j);
#pragma unroll
    for (int j = 0; j < SH::NB; ++j) b[j] = 1e-3 * (threadIdx.x - j);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < CH; ++i) mma_shape<S>(c[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < CH; ++i)
#pragma unroll
        for (int j = 0; j < SH::NC; ++j) s += c[i][j];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// TFLOP/s of one shape at `wps` warps per SM (128-thread CTAs, wps / 4 of them per SM), best of 3
template <int S, int CH>
static double time_shape(double* out, int sms, int wps, cudaEvent_t e0, cudaEvent_t e1)
{
    const int threads = 128, blocks = sms * wps / 4;
    // the same work per warp for every shape and chain count: 2^29 flop
    const int iters = (int)((1ll << 29) / ((long long)CH * Shape<S>::FLOP));
    dmma_shape_kernel<S, CH><<<blocks, threads>>>(out, iters / 16);
    if (cudaDeviceSynchronize() != cudaSuccess) return -1.0;
    float best = 1e30f, ms = 0.f;
    for (int r = 0; r < 3; ++r) {
        cudaEventRecord(e0);
        dmma_shape_kernel<S, CH><<<blocks, threads>>>(out, iters);
        cudaEventRecord(e1);
        if (cudaEventSynchronize(e1) != cudaSuccess) return -1.0;
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    const double flops = (double)blocks * (threads / 32) * iters * CH * Shape<S>::FLOP;
    return flops / (best * 1e-3) / 1e12;
}

template <int S>
static void print_shape(double* out, int sms, cudaEvent_t e0, cudaEvent_t e1, bool first)
{
    printf("%s\"%s\": {", first ? "" : ", ", Shape<S>::name);
    bool f = true;
    for (int wps : {4, 8, 16}) {
        printf("%s\"w%d_c8\": %.2f", f ? "" : ", ", wps, time_shape<S, 8>(out, sms, wps, e0, e1));
        printf(", \"w%d_c16\": %.2f", wps, time_shape<S, 16>(out, sms, wps, e0, e1));
        f = false;
    }
    printf("}");
}

__global__ void dfma_kernel(double* out, int iters)
{
    double c[16];
    for (int i = 0; i < 16; ++i) c[i] = threadIdx.x * 1e-3 + i;
    double a = 1.0000001, b = 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) c[i] = fma(c[i], a, b);
    }
    double s = 0;
    for (int i = 0; i < 16; ++i) s += c[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void write_kernel(double2* p, size_t n)
{
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) p[i] = make_double2(1.0, 2.0);
}
__global__ void copy_kernel(const double2* __restrict__ s, double2* __restrict__ d, size_t n)
{
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) d[i] = s[i];
}

int main()
{
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    int sms = prop.multiProcessorCount;
    printf("{\"gpu\": \"%s\", \"sms\": %d", prop.name, sms);
    double* out;
    CK(cudaMalloc(&out, sizeof(double) * sms * 8 * 1024));
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms;
    // DMMA: warps per SM sweep
    for (int wps : {4, 8, 16, 32}) {
        int threads = 256, blocks = sms * wps * 32 / threads;
        int iters = 20000;
        dmma_kernel<<<blocks, threads>>>(out, 100);
        CK(cudaDeviceSynchronize());
        float best = 1e30f;
        for (int r = 0; r < 3; ++r) {
            cudaEventRecord(e0);
            dmma_kernel<<<blocks, threads>>>(out, iters);
            cudaEventRecord(e1);
            CK(cudaEventSynchronize(e1));
            cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) best = ms;
        }
        double flops = (double)blocks * (threads / 32) * iters * 8.0 * (16.0 * 8 * 8 * 2);
        printf(", \"dmma_tflops_w%d\": %.2f", wps, flops / (best * 1e-3) / 1e12);
    }
    // per-shape DMMA rate: TFLOP/s at 4 / 8 / 16 warps per SM, 8 / 16 independent accumulators per warp
    printf(", \"dmma_shapes_tflops\": {");
    print_shape<0>(out, sms, e0, e1, true);
    print_shape<1>(out, sms, e0, e1, false);
    print_shape<2>(out, sms, e0, e1, false);
    print_shape<3>(out, sms, e0, e1, false);
    printf("}");
    for (int wps : {8, 16, 32}) {
        int threads = 256, blocks = sms * wps * 32 / threads;
        int iters = 20000;
        dfma_kernel<<<blocks, threads>>>(out, 100);
        CK(cudaDeviceSynchronize());
        float best = 1e30f;
        for (int r = 0; r < 3; ++r) {
            cudaEventRecord(e0);
            dfma_kernel<<<blocks, threads>>>(out, iters);
            cudaEventRecord(e1);
            CK(cudaEventSynchronize(e1));
            cudaEventElapsedTime(&ms, e0, e1);
            if (ms < best) best = ms;
        }
        double flops = (double)blocks * threads * iters * 16.0 * 2;
        printf(", \"dfma_tflops_w%d\": %.2f", wps, flops / (best * 1e-3) / 1e12);
    }
    size_t bytes = (size_t)4 << 30;
    double2 *pa, *pb;
    CK(cudaMalloc(&pa, bytes)); CK(cudaMalloc(&pb, bytes));
    size_t n = bytes / sizeof(double2);
    write_kernel<<<sms * 16, 256>>>(pa, n); write_kernel<<<sms * 16, 256>>>(pb, n);
    CK(cudaDeviceSynchronize());
    float best = 1e30f;
    for (int r = 0; r < 5; ++r) {
        cudaEventRecord(e0);
        write_kernel<<<sms * 16, 256>>>(pa, n);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    printf(", \"hbm_write_gbs\": %.1f", bytes / (best * 1e-3) / 1e9);
    best = 1e30f;
    for (int r = 0; r < 5; ++r) {
        cudaEventRecord(e0);
        copy_kernel<<<sms * 16, 256>>>(pa, pb, n);
        cudaEventRecord(e1);
        CK(cudaEventSynchronize(e1));
        cudaEventElapsedTime(&ms, e0, e1);
        if (ms < best) best = ms;
    }
    printf(", \"hbm_copy_gbs\": %.1f}\n", 2.0 * bytes / (best * 1e-3) / 1e9);
    return 0;
}
