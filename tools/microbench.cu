// tools/microbench.cu — measures the fp64 roofline denominators this backend is
// judged against on the actual box (MEASURED_PEAKS.json only holds HBM copy and
// bf16): DMMA (mma.sync f64) and DFMA peak, HBM write-only and copy bandwidth.
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
