// limbo_b200/csrc/tf32_query.cu — reduced-precision candidate scoring on the Hopper tensor cores (wgmma)
// (BASELINE.json config 4: N = 16384, D = 12, 1M EI candidates; LB_PREC_TF32 / LB_PREC_FP16 / LB_PREC_FP16X3).
//
// The per-candidate variance needs |L^-1 k*|^2, i.e. V = L^-1 K* (M N^2 flops, gp.hpp:618-624 once per
// candidate in the reference).  The fp64 path runs on DMMA (query.cu).  Here the factor is inverted once in fp64 (lml.cu,
// recursive trtri), cast to a row-major tf32 (fp32 container) or fp16 copy, and
//     D[c, n] = sum_{k <= n} Kt[c, k] * Linv[n, k]          (Kt = K*^T, candidates x training points)
// runs on wgmma with fp32 accumulators in registers; D is never written: every consumer thread squares the accumulator
// fragment it holds and adds it to the partial norms of its two candidate rows.
//
// gemm_norm_kernel (persistent, 384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers,
// each issuing m64 wgmmas for 64 of the tile's 128 candidates; a ring of 128-byte SWIZZLE_128B rows in shared memory;
// every mbarrier wait is bounded and raises an error flag instead of hanging the GPU.
//   F16 = false : tf32 operands, 128 x 256 tiles, 4 stages of 48 KB
//   F16 = true  : fp16 operands, same tiles (64 k per stage instead of 32)
//   SPLIT       : fp16 hi + 2^-11 lo operands (LB_PREC_FP16X3), 128 x 128 tiles, 3 stages of 64 KB, two accumulators
// Around it: kstar_t32_kernel (K*^T chunk from fp64 kernel evaluations with the squared distances on the fp64 tensor pipe,
// mean and rounding-bias partials fused), mu_reduce_kernel, sigma2_t32_kernel (clamp / noise of gp.hpp:623,166 and the
// rounding-bias correction), linv_to_rowmajor_kernel (+ absmax / colnorm2 for the fp16 scale and the bias weights).
#include "common.cuh"
#include <cuda.h>
#include <cuda_fp16.h>
#include <cmath>
#include <type_traits>
#include <cstdlib>

namespace tf32q {

constexpr int BM = 128;       // candidates per tile (two consumer warpgroups x wgmma M = 64)
constexpr int BN = 256;       // outputs (rows of L^-1) per tile (wgmma N); split mode: BN / 2
// k elements per stage = 128 B = one swizzle atom row: 32 tf32 or 64 fp16; one stage is always 4 wgmmas (K = 8 tf32 / 16 fp16)
template <bool F16> __host__ __device__ constexpr int bke() { return F16 ? 64 : 32; }
constexpr int MMAS_PER_STAGE = 4;
constexpr int THREADS = 384;
constexpr long long SPIN_LIMIT = 1LL << 24;

// Shared-memory stage of one k-block: [A hi | B hi | A lo | B lo] (lo planes in split mode only).  The split mode halves the
// tile width: two 64-register accumulators per thread instead of one of 128.
template <bool SPLIT>
struct Cfg {
    static constexpr int BNT = SPLIT ? BN / 2 : BN;
    static constexpr int A_BYTES = BM * 128;
    static constexpr int B_BYTES = BNT * 128;
    static constexpr int STAGE_BYTES = (SPLIT ? 2 : 1) * (A_BYTES + B_BYTES);
    static constexpr int STAGES = SPLIT ? 3 : 4;
    static constexpr size_t SMEM_BYTES = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t n)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(lb_smem_u32(b)), "r"(n));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(lb_smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(lb_smem_u32(b)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* b, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(lb_smem_u32(b)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: returns false (and raises *err) instead of spinning forever
// The error flag (global memory) is polled only every 1024 attempts: a volatile load per spin from every spinning thread
// would saturate the SM's load/store path.
__device__ __forceinline__ bool mbar_wait(uint64_t* b, uint32_t parity, int* err)
{
    long long spins = 0;
    while (!mbar_try(b, parity)) {
        if ((++spins & 1023) == 0 && (spins > SPIN_LIMIT || *(volatile int*)err)) {
            atomicExch(err, 1);
            return false;
        }
    }
    return true;
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                     lb_smem_u32(dst)),
                 "l"(map), "r"(c0), "r"(c1), "r"(lb_smem_u32(bar))
                 : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (PTX ISA, "Matrix Descriptor Format"):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major: 1) |
//   [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024 B -> 64) | [62,64) layout = 1 (SWIZZLE_128B)
// Every operand tile starts on a 1024-byte boundary, so the base-offset field stays 0.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R])
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// m64 x N x k wgmmas, A and B from K-major shared memory, fp32 accumulators; accumulate == 0 overwrites d.
// Accumulator fragment: d[i] is row (warp % 4) * 16 + lane / 4 + 8 * ((i >> 1) & 1), column (i >> 2) * 8 + 2 * (lane % 4) + (i & 1).
__device__ __forceinline__ void wgmma_tf32_n256(float (&d)[128], uint64_t a, uint64_t b, int accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_n256(float (&d)[128], uint64_t a, uint64_t b, int accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t a, uint64_t b, int accumulate)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
}

template <bool F16>
__device__ __forceinline__ void wgmma_n256(float (&d)[128], uint64_t a, uint64_t b, int accumulate)
{
    if (F16) wgmma_f16_n256(d, a, b, accumulate);
    else wgmma_tf32_n256(d, a, b, accumulate);
}

// D[c, n] = sum_k A[c, k] B[n, k]; tri != 0: k only up to the end of the n-tile (B lower triangular).
// norm2[c] = sum_n D[c, n]^2 (float; double in split mode); Dout (optional, row-major M x N, not in split mode) receives D
// for validation.  Split mode: D = A_hi B_hi + 2^-11 (A_hi B_lo + A_lo B_hi) from three fp16 wgmmas per k-step into two
// accumulators (the 2^-22 A_lo B_lo term is dropped), combined and squared in fp64.
template <bool F16, bool SPLIT>
__global__ void __launch_bounds__(THREADS, 1)
gemm_norm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
    const __grid_constant__ CUtensorMap mapAlo, const __grid_constant__ CUtensorMap mapBlo, int64_t M, int64_t N, int64_t K, int tri,
    void* __restrict__ norm2_, float* __restrict__ Dout, int* __restrict__ err)
{
    static_assert(F16 || !SPLIT, "split operands are fp16");
    using C = Cfg<SPLIT>;
    using NormT = typename std::conditional<SPLIT, double, float>::type;
    constexpr int BNT = C::BNT, BKE = bke<F16>(), NACC = BNT / 2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023); // SWIZZLE_128B needs 1024-byte alignment
    uint64_t* full = (uint64_t*)(smem + (size_t)C::STAGES * C::STAGE_BYTES);
    uint64_t* empty = full + C::STAGES;

    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int m_tiles = (int)(M / BM), n_tiles = (int)(N / BNT);
    auto kblocks_of = [&](int nt) {
        const int64_t kend = tri ? (int64_t)(nt + 1) * BNT : K;
        return (int)((kend < K ? kend : K) / BKE);
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); } // empty: one arrival per consumer warpgroup
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // ===== TMA producer =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            int s = 0; uint32_t ph = 0; bool ok = true;
            for (int mt = blockIdx.x; mt < m_tiles && ok; mt += gridDim.x) {
                for (int nt = 0; nt < n_tiles && ok; ++nt) {
                    const int kblocks = kblocks_of(nt);
                    for (int kb = 0; kb < kblocks; ++kb) {
                        if (!mbar_wait(&empty[s], ph ^ 1, err)) { ok = false; break; }
                        uint8_t* sa = smem + (size_t)s * C::STAGE_BYTES;
                        mbar_expect_tx(&full[s], C::STAGE_BYTES);
                        tma_load_2d(sa, &mapA, kb * BKE, mt * BM, &full[s]);
                        tma_load_2d(sa + C::A_BYTES, &mapB, kb * BKE, nt * BNT, &full[s]);
                        if (SPLIT) {
                            tma_load_2d(sa + C::A_BYTES + C::B_BYTES, &mapAlo, kb * BKE, mt * BM, &full[s]);
                            tma_load_2d(sa + 2 * C::A_BYTES + C::B_BYTES, &mapBlo, kb * BKE, nt * BNT, &full[s]);
                        }
                        if (++s == C::STAGES) { s = 0; ph ^= 1; }
                    }
                }
            }
        }
    }
    else {
        // ===== consumers: warpgroup c owns candidate rows [64 c, 64 c + 64) of the tile =====
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int c = wg - 1;
        const int r0 = c * 64 + warp * 16 + (lane >> 2); // this thread's rows: r0 and r0 + 8
        const bool signal = (warp == 0 && lane == 0);    // releases a stage for its warpgroup
        float acc[NACC];
        float acc1[SPLIT ? NACC : 1];
        // A timed-out wait never leaves the loops: what follows it is warpgroup-collective (wgmma, wgmma.wait_group) and
        // warp-collective (the quad shuffles), so every thread keeps walking the same trip counts, which depend only on the
        // shapes and blockIdx.  It only marks its results invalid; once *err is raised every later wait gives up after one
        // polling interval, and operands left stale in shared memory feed results that are never written.
        int s = 0; uint32_t ph = 0; bool ok = true;
        for (int mt = blockIdx.x; mt < m_tiles; mt += gridDim.x) {
            NormT n0 = 0, n1 = 0;
            for (int nt = 0; nt < n_tiles; ++nt) {
                const int kblocks = kblocks_of(nt);
                int prev = -1;
                for (int kb = 0; kb < kblocks; ++kb) {
                    if (!mbar_wait(&full[s], ph, err)) ok = false;
                    const uint32_t sa = lb_smem_u32(smem + (size_t)s * C::STAGE_BYTES);
                    const uint64_t ad = make_desc(sa + c * 64 * 128), bd = make_desc(sa + C::A_BYTES);
                    acc_fence(acc);
                    if (SPLIT) acc_fence(acc1);
                    wg_fence();
                    if constexpr (SPLIT) {
                        const uint64_t ald = make_desc(sa + C::A_BYTES + C::B_BYTES + c * 64 * 128),
                                       bld = make_desc(sa + 2 * C::A_BYTES + C::B_BYTES);
#pragma unroll
                        for (int k = 0; k < MMAS_PER_STAGE; ++k) { // +32 B per wgmma inside the 128 B swizzle row: +2 in the >>4 address field
                            wgmma_f16_n128(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kb | k) != 0);
                            wgmma_f16_n128(acc1, ad + (uint64_t)(2 * k), bld + (uint64_t)(2 * k), (kb | k) != 0);
                            wgmma_f16_n128(acc1, ald + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), 1);
                        }
                    }
                    else {
#pragma unroll
                        for (int k = 0; k < MMAS_PER_STAGE; ++k)
                            wgmma_n256<F16>(acc, ad + (uint64_t)(2 * k), bd + (uint64_t)(2 * k), (kb | k) != 0);
                    }
                    wg_commit();
                    wg_wait<1>(); // the previous stage's wgmmas have read their operands
                    acc_fence(acc);
                    if (SPLIT) acc_fence(acc1);
                    if (prev >= 0 && signal) mbar_arrive(&empty[prev]);
                    prev = s;
                    if (++s == C::STAGES) { s = 0; ph ^= 1; }
                }
                wg_wait<0>();
                acc_fence(acc);
                if (SPLIT) acc_fence(acc1);
                if (signal) mbar_arrive(&empty[prev]);
#pragma unroll
                for (int i = 0; i < NACC; ++i) {
                    const bool hi_row = (i >> 1) & 1;
                    if constexpr (SPLIT) {
                        const double d = fma((double)acc1[i], 1.0 / 2048.0, (double)acc[i]);
                        if (hi_row) n1 = fma(d, d, n1);
                        else n0 = fma(d, d, n0);
                    }
                    else {
                        if (hi_row) n1 = fmaf(acc[i], acc[i], n1);
                        else n0 = fmaf(acc[i], acc[i], n0);
                    }
                }
                if (!SPLIT && Dout) {
#pragma unroll
                    for (int i = 0; i < NACC; ++i)
                        Dout[((int64_t)mt * BM + r0 + 8 * ((i >> 1) & 1)) * N + (int64_t)nt * BNT + (i >> 2) * 8 + 2 * (lane & 3) + (i & 1)] = acc[i];
                }
            }
            // the four threads of a quad hold the same two rows
            n0 += __shfl_xor_sync(0xffffffffu, n0, 1);
            n0 += __shfl_xor_sync(0xffffffffu, n0, 2);
            n1 += __shfl_xor_sync(0xffffffffu, n1, 1);
            n1 += __shfl_xor_sync(0xffffffffu, n1, 2);
            if (ok && (lane & 3) == 0) {
                NormT* norm2 = reinterpret_cast<NormT*>(norm2_);
                norm2[(int64_t)mt * BM + r0] = n0;
                norm2[(int64_t)mt * BM + r0 + 8] = n1;
            }
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// row-major (rows x K) fp32 matrix, boxes of 32 k x box_rows rows, 128-byte swizzle, tf32 rounding on load
static int make_map(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int64_t ld, int box_rows, bool f16)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) return LB_ERR_UNSUPPORTED;
    cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t gstr[1] = {(cuuint64_t)ld * (f16 ? 2 : 4)};
    cuuint32_t box[2] = {(cuuint32_t)(f16 ? 64 : 32), (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 2, (void*)base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? LB_OK : LB_ERR_CUDA;
}

// A: M x K (ld lda), B: N x K (ld ldb), row-major; lo planes (split mode) with the same shapes.  M % 128 == 0,
// N % (256, split: 128) == 0, K % 64 == 0.  grid: persistent CTAs (at most one per 128-candidate tile).
template <bool F16, bool SPLIT>
static int launch_gemm_norm(cudaStream_t st, const void* dA, const void* dAlo, int64_t lda, const void* dB, const void* dBlo, int64_t ldb,
    int64_t M, int64_t N, int64_t K, int tri, void* dNorm2, float* dDout, int* dErr, int grid)
{
    using C = Cfg<SPLIT>;
    if (M % BM || N % C::BNT || K % 64) return LB_ERR_ARG;
    static LbOncePerDevice attr_once;
    if (attr_once.need()) {
        LB_CUDA(cudaFuncSetAttribute(gemm_norm_kernel<F16, SPLIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    }
    alignas(64) CUtensorMap mA, mB, mAlo, mBlo;
    int rc;
    if ((rc = make_map(&mA, dA, M, K, lda, BM, F16))) return rc;
    if ((rc = make_map(&mB, dB, N, K, ldb, C::BNT, F16))) return rc;
    mAlo = mA;
    mBlo = mB;
    if (SPLIT) {
        if ((rc = make_map(&mAlo, dAlo, M, K, lda, BM, true))) return rc;
        if ((rc = make_map(&mBlo, dBlo, N, K, ldb, C::BNT, true))) return rc;
    }
    const int m_tiles = (int)(M / BM);
    if (grid > m_tiles) grid = m_tiles;
    gemm_norm_kernel<F16, SPLIT><<<grid, THREADS, C::SMEM_BYTES, st>>>(mA, mB, mAlo, mBlo, M, N, K, tri, dNorm2, dDout, dErr);
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

} // namespace tf32q

// A: M x K (ld lda), B: N x K (ld ldb), row-major fp32 (tf32 MMA) or fp16 in device memory; M % 128 == 0, N % 256 == 0, K % 64 == 0.
int lb_launch_tf32_gemm_norm(cudaStream_t st, const void* dA, int64_t lda, const void* dB, int64_t ldb, int64_t M, int64_t N, int64_t K,
    int tri, float* dNorm2, float* dDout, int* dErr, int grid, int f16)
{
    using namespace tf32q;
    return f16 ? launch_gemm_norm<true, false>(st, dA, nullptr, lda, dB, nullptr, ldb, M, N, K, tri, dNorm2, dDout, dErr, grid)
               : launch_gemm_norm<false, false>(st, dA, nullptr, lda, dB, nullptr, ldb, M, N, K, tri, dNorm2, dDout, dErr, grid);
}

// Split-operand launch (fp16 hi / lo planes): dA*: M x K, dB*: N x K row-major halves; M % 128 == 0, N % 128 == 0; dNorm2: M doubles.
static int lb_launch_split_gemm_norm(cudaStream_t st, const void* dAh, const void* dAl, int64_t lda, const void* dBh, const void* dBl,
    int64_t ldb, int64_t M, int64_t N, int64_t K, int tri, double* dNorm2, int* dErr, int grid)
{
    return tf32q::launch_gemm_norm<true, true>(st, dAh, dAl, lda, dBh, dBl, ldb, M, N, K, tri, dNorm2, nullptr, dErr, grid);
}

__global__ void debug_exp_kernel(const double* in, double* out, long long n)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i < n) out[i] = lb_exp_nonpos(in[i]);
}

// test hook: out[i] = lb_exp_nonpos(in[i]) (device pointers)
extern "C" int lb_debug_exp(const double* dIn, double* dOut, long long n)
{
    debug_exp_kernel<<<(unsigned)((n + 255) / 256), 256>>>(dIn, dOut, n);
    LB_CUDA(cudaGetLastError());
    LB_CUDA(cudaDeviceSynchronize());
    return LB_OK;
}

extern "C" int lb_debug_tf32_gemm(const void* dA, const void* dB, long long M, long long N, long long K, int tri, float* dNorm2,
    float* dDout, int grid, int f16)
{
    int* dErr = nullptr;
    LB_CUDA(cudaMalloc(&dErr, sizeof(int)));
    LB_CUDA(cudaMemset(dErr, 0, sizeof(int)));
    int rc = lb_launch_tf32_gemm_norm(0, dA, K, dB, K, M, N, K, tri, dNorm2, dDout, dErr, grid, f16);
    if (rc) { cudaFree(dErr); return rc; }
    LB_CUDA(cudaDeviceSynchronize());
    int herr = 0;
    LB_CUDA(cudaMemcpy(&herr, dErr, sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(dErr);
    return herr ? LB_ERR_TIMEOUT : LB_OK;
}

// ===========================================================================
// TF32 prediction path: K*^T (fp32, K-major) build, mu GEMV, L^-1 cast/transposed, sigma^2 from the row norms.
// ===========================================================================
namespace tf32q {

// fp32 -> tf32 with round-to-nearest: the tf32 wgmma ignores the low 13 mantissa bits of its operands, i.e. truncates;
// a truncated operand is biased low, and the bias of |L^-1 k*|^2 does not average out over the N terms of the sum.
__device__ __forceinline__ float tf32_rna(float v)
{
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    return __uint_as_float(u);
}

constexpr int DCH_WIDE = 16; // input dimensions staged per pass

// Kt[c * ldk + n] = (float) k(x_n, q_c)  for one tile of 128 candidates x 128 training points; zero for n >= N.
// grid: (Np/128, Mc/128).  Same thread mapping as kbuild_kernel: the two consecutive "rows" of a thread are two
// consecutive n, stored as one float2 (n is the contiguous, K-major index of the GEMM's A operand).
// F16: the stored values are k / sigma_f^2 (in (0, 1]) as half.  EDGE: the tile crosses N or M (zero beyond).
// Tiles [i_first, i_first + ni) x [j_first, j_first + nj) are walked with a grid-stride loop (training index fastest), so the
// same kernel runs one tile per CTA or as a small persistent grid.
// Squared distances on the fp64 TENSOR pipe: z_cn = |q_c|^2 + |x_n|^2 - 2 q_c . x_n with the cross term as an
// mma.m8n8k4.f64 (candidates = M side, training points = N side, input dimensions = K, zero padded to a multiple of 4).
// Moving the D-loop (24 of ~55 fp64 operations per pair at D = 12) to DMMA leaves the fp64 ALU pipe to exp / scaling / the
// mean and bias partials.  The cancellation costs ~1e-16 (|q|^2 +
// |x|^2) absolute on z, i.e. <= 1e-13 relative on k: inside the 1e-9 bar this path states for mu.
// A thread ends up with candidate g (+ 8 mb) x training points 2t, 2t+1 (+ 8 nb): two consecutive K-major elements = one
// half2 / float2 store.
constexpr int XP = LB_TILE + 4; // pitch of the staged point tiles: the (d = t, point = g) fragment loads of a half-warp hit 16 distinct banks

template <int KID, bool F16, bool EDGE, int DCH>
__device__ __forceinline__ void kstar_t32_body(const double* __restrict__ Xs, int64_t Np, int64_t N, const double* __restrict__ Qs, int64_t Mp,
    int64_t M, void* __restrict__ Kt_, int64_t ldk, const KernParams& kp, const double* __restrict__ alpha, int P,
    double* __restrict__ mu_part, int64_t i_first, int64_t j_first, int64_t ni, int64_t nj, const double* __restrict__ colw,
    void* __restrict__ Kt_lo = nullptr)
{
    static_assert(DCH % 4 == 0, "k4 steps");
    __shared__ __align__(128) double sxi[DCH][XP]; // training points of the tile, dimension-major
    __shared__ __align__(128) double sxj[DCH][XP]; // candidates
    __shared__ double sni[LB_TILE], snj[LB_TILE];  // squared norms of the staged coordinates
    __shared__ double spm[8][64];
    __shared__ __align__(8) uint64_t bar;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int D = kp.D;
    if (tid == 0) {
        lb_mbar_init(&bar, 1);
        lb_fence_barrier_init();
    }
    __syncthreads();
    uint32_t phase = 0;
    const int npass = (D + DCH - 1) / DCH;
    for (int64_t tile = blockIdx.x; tile < ni * nj; tile += gridDim.x) {
    const int64_t ti = i_first + tile % ni; // training tile index (also the slot of the mean partial)
    const int64_t i0 = ti * LB_TILE, j0 = (j_first + tile / ni) * LB_TILE; // i: training, j: candidates
    __syncthreads(); // the previous tile's epilogue has read the norms
    if (tid < LB_TILE) sni[tid] = 0.0;
    else snj[tid - LB_TILE] = 0.0;
    for (int h = 0; h < 2; ++h) {
        double acc[8][2][2]; // [candidate block mb][training block nb][2 consecutive training points]
#pragma unroll
        for (int mb = 0; mb < 8; ++mb)
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) acc[mb][nb][0] = acc[mb][nb][1] = 0.0;
        for (int pass = 0; pass < npass; ++pass) {
            const int d0 = pass * DCH;
            const int dc = min(DCH, D - d0), dc4 = (dc + 3) & ~3;
            if (!(npass == 1 && h == 1)) {
                __syncthreads();
                if (tid == 0) {
                    lb_fence_proxy_async();
                    lb_mbar_expect_tx(&bar, (uint32_t)(2 * dc * LB_TILE * sizeof(double)));
                    for (int d = 0; d < dc; ++d) {
                        lb_bulk_g2s(&sxi[d][0], Xs + (int64_t)(d0 + d) * Np + i0, LB_TILE * sizeof(double), &bar);
                        lb_bulk_g2s(&sxj[d][0], Qs + (int64_t)(d0 + d) * Mp + j0, LB_TILE * sizeof(double), &bar);
                    }
                }
                for (int d = dc; d < dc4; ++d) { // zero rows up to the k4 boundary
                    if (tid < LB_TILE) sxi[d][tid] = 0.0;
                    else sxj[d][tid - LB_TILE] = 0.0;
                }
                lb_mbar_wait(&bar, phase);
                phase ^= 1;
                if (h == 0) { // squared norms, accumulated over the passes (one point per thread)
                    double s = 0.0;
                    if (tid < LB_TILE) {
                        for (int d = 0; d < dc; ++d) s = fma(sxi[d][tid], sxi[d][tid], s);
                        sni[tid] += s;
                    }
                    else {
                        for (int d = 0; d < dc; ++d) s = fma(sxj[d][tid - LB_TILE], sxj[d][tid - LB_TILE], s);
                        snj[tid - LB_TILE] += s;
                    }
                }
                __syncthreads();
            }
            for (int ks = 0; ks < dc4; ks += 4) {
                const double b0 = sxi[ks + t][warp * 16 + g], b1 = sxi[ks + t][warp * 16 + 8 + g];
#pragma unroll
                for (int mb = 0; mb < 8; ++mb) {
                    const double a = sxj[ks + t][h * 64 + mb * 8 + g];
                    lb_dmma_8x8x4(acc[mb][0][0], acc[mb][0][1], a, b0);
                    lb_dmma_8x8x4(acc[mb][1][0], acc[mb][1][1], a, b1);
                }
            }
        }
        // kernel values (kept in acc for the partial sums), K-major stores
#pragma unroll
        for (int mb = 0; mb < 8; ++mb) {
            const int cl = h * 64 + mb * 8 + g; // candidate within the tile
            const int64_t gj = j0 + cl;
            const double nq = snj[cl];
#pragma unroll
            for (int nb = 0; nb < 2; ++nb) {
                const int tl = warp * 16 + nb * 8 + 2 * t; // training point within the tile (even)
                const int64_t gi = i0 + tl;
                float v[2];
                double uu[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const double z = fmax(nq + sni[tl + e] - 2.0 * acc[mb][nb][e], 0.0);
                    double u = lb_unit_kernel_from_z<KID>(z, kp);
                    if (EDGE) {
                        if (gi + e >= N || gj >= M) u = 0.0;
                    }
                    const double k = kp.sf2 * u;
                    acc[mb][nb][e] = k;
                    uu[e] = u;
                    v[e] = (float)(F16 ? u : k);
                }
                if (F16) {
                    const __half2 hi = __floats2half2_rn(v[0], v[1]);
                    *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(Kt_) + gj * ldk + gi) = hi;
                    if (Kt_lo) { // split operands (LB_PREC_FP16X3): lo = (u - hi) * 2^11, the next 11 bits of the value
                        const float2 hf = __half22float2(hi);
                        *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(Kt_lo) + gj * ldk + gi)
                            = __floats2half2_rn((float)((uu[0] - (double)hf.x) * 2048.0), (float)((uu[1] - (double)hf.y) * 2048.0));
                    }
                }
                else *reinterpret_cast<float2*>(reinterpret_cast<float*>(Kt_) + gj * ldk + gi) = make_float2(tf32_rna(v[0]), tf32_rna(v[1]));
            }
        }
        // mean partials from the fp64 kernel values: mu_part[(p * ntiles + tile) * Mp + candidate] = sum over this tile's
        // 128 training points (lanes -> warps in a fixed order; the tiles are summed in order by mu_reduce_kernel).
        // Pass p == P (when colw != nullptr): sum_k k*_k^2 |L^-1 e_k|^2, the weight of the rounding-noise bias of |L^-1 k*|^2
        // (sigma2_t32_kernel subtracts its expectation).
        for (int p = 0; p < P + (colw ? 1 : 0); ++p) {
            const bool bias = (p == P);
            const double* wv = (bias ? colw : alpha + (int64_t)p * Np) + i0 + warp * 16 + 2 * t;
            const double w00 = wv[0], w01 = wv[1], w10 = wv[8], w11 = wv[9];
#pragma unroll
            for (int mb = 0; mb < 8; ++mb) {
                double sm;
                if (bias)
                    sm = fma(acc[mb][0][0] * acc[mb][0][0], w00, fma(acc[mb][0][1] * acc[mb][0][1], w01,
                        fma(acc[mb][1][0] * acc[mb][1][0], w10, acc[mb][1][1] * acc[mb][1][1] * w11)));
                else
                    sm = fma(acc[mb][0][0], w00, fma(acc[mb][0][1], w01, fma(acc[mb][1][0], w10, acc[mb][1][1] * w11)));
                sm += __shfl_xor_sync(0xffffffffu, sm, 1);
                sm += __shfl_xor_sync(0xffffffffu, sm, 2);
                if (t == 0) spm[warp][mb * 8 + g] = sm;
            }
            __syncthreads();
            if (tid < 64) {
                double sacc = spm[0][tid];
#pragma unroll
                for (int w = 1; w < 8; ++w) sacc += spm[w][tid];
                mu_part[((int64_t)p * (Np / LB_TILE) + ti) * Mp + j0 + h * 64 + tid] = sacc;
            }
            __syncthreads();
        }
    }
    } // tile loop
}

// one tile per CTA (or any grid): two CTAs per SM by registers
template <int KID, bool F16, bool EDGE, int DCH>
__global__ void __launch_bounds__(256, 2)
kstar_t32_kernel(const double* __restrict__ Xs, int64_t Np, int64_t N, const double* __restrict__ Qs, int64_t Mp, int64_t M,
    void* __restrict__ Kt_, int64_t ldk, KernParams kp, const double* __restrict__ alpha, int P,
    double* __restrict__ mu_part, int64_t i_first, int64_t j_first, int64_t ni, int64_t nj, const double* __restrict__ colw,
    void* __restrict__ Kt_lo)
{
    kstar_t32_body<KID, F16, EDGE, DCH>(Xs, Np, N, Qs, Mp, M, Kt_, ldk, kp, alpha, P, mu_part, i_first, j_first, ni, nj, colw, Kt_lo);
}
// mu[c*P + p] = sum over the training tiles of the partials written by kstar_t32_kernel (fixed order)
__global__ void __launch_bounds__(256)
mu_reduce_kernel(const double* __restrict__ part, int ntiles, int64_t Mp, int P, int64_t M, double* __restrict__ mu,
    double* __restrict__ bias)
{
    const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= M) return;
    for (int p = 0; p < P + (bias ? 1 : 0); ++p) {
        const double* q = part + (int64_t)p * ntiles * Mp + c;
        double s = 0.0;
        for (int t = 0; t < ntiles; ++t) s += q[(int64_t)t * Mp];
        if (p < P) mu[c * P + p] = s;
        else bias[c] = s;
    }
}

// w[k] = sum_n Linv[n, k]^2 (column k of the lower-triangular inverse, column-major): one block per column
__global__ void __launch_bounds__(256)
colnorm2_kernel(const double* __restrict__ Linv, int64_t ld, double* __restrict__ w)
{
    __shared__ double red[8];
    const int64_t k = blockIdx.x;
    const double* col = Linv + k * ld;
    double s = 0.0;
    for (int64_t n = k + threadIdx.x; n < ld; n += 256) s = fma(col[n], col[n], s);
    s = lb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += red[i];
        w[k] = t;
    }
}

// max |Linv| (for the fp16 scale): one value per block, reduced on the host (tiny)
__global__ void __launch_bounds__(256)
absmax_kernel(const double* __restrict__ A, int64_t n, double* __restrict__ out)
{
    __shared__ double red[8];
    double m = 0.0;
    for (int64_t i = blockIdx.x * (int64_t)256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) m = fmax(m, fabs(A[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmax(m, red[w]);
        out[blockIdx.x] = m;
    }
}

// LinvR[n * ldr + k] = (float) Linv[n + k * ld]  (column-major fp64 -> row-major fp32, 32 x 32 smem transpose)
template <bool F16>
__global__ void __launch_bounds__(256)
linv_to_rowmajor_kernel(const double* __restrict__ Linv, int64_t ld, void* __restrict__ R_, int64_t ldr, double scale, void* __restrict__ Rlo_)
{
    __shared__ double tile[32][33];
    const int64_t n0 = (int64_t)blockIdx.x * 32, k0 = (int64_t)blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int kk = ty; kk < 32; kk += 8) tile[kk][tx] = (k0 + kk <= n0 + tx) ? Linv[n0 + tx + (k0 + kk) * ld] * scale : 0.0;
    __syncthreads();
    for (int nn = ty; nn < 32; nn += 8) {
        const double v = tile[tx][nn];
        if (F16) {
            const __half hi = __float2half_rn((float)v);
            reinterpret_cast<__half*>(R_)[(n0 + nn) * ldr + k0 + tx] = hi;
            if (Rlo_) reinterpret_cast<__half*>(Rlo_)[(n0 + nn) * ldr + k0 + tx] = __float2half_rn((float)((v - (double)__half2float(hi)) * 2048.0));
        }
        else reinterpret_cast<float*>(R_)[(n0 + nn) * ldr + k0 + tx] = tf32_rna((float)v);
    }
}

// ---- inversion spread over G GPUs (query.cu: lb_launch_linv_columns): pack this rank's columns, adopt everybody's ----------------
// V: Np x ldr column-major, local column tile t = global tile c = rank + t * G.  Chunk of a rank (what the all_gather moves):
//   [ hi plane: Np x ldr row-major (fp16, or fp32 holding tf32) | lo plane (split mode only) | w: ldr doubles = |L^-1 e_k|^2 ]
template <bool F16>
__global__ void __launch_bounds__(256)
linv_cols_pack_kernel(const double* __restrict__ V, int64_t ld, int rank, int G, int T, void* __restrict__ R_, int64_t ldr, double scale,
    void* __restrict__ Rlo_)
{
    __shared__ double tile[32][33];
    const int64_t n0 = (int64_t)blockIdx.x * 32, l0 = (int64_t)blockIdx.y * 32; // rows, local columns
    const int64_t c = rank + (l0 / LB_TILE) * G;                                  // global column tile
    const int64_t k0 = c * LB_TILE + (l0 % LB_TILE);                              // global column of local column l0
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int kk = ty; kk < 32; kk += 8) tile[kk][tx] = (c < T && k0 + kk <= n0 + tx) ? V[n0 + tx + (l0 + kk) * ld] * scale : 0.0;
    __syncthreads();
    for (int nn = ty; nn < 32; nn += 8) {
        const double v = tile[tx][nn];
        if (F16) {
            const __half hi = __float2half_rn((float)v);
            reinterpret_cast<__half*>(R_)[(n0 + nn) * ldr + l0 + tx] = hi;
            if (Rlo_) reinterpret_cast<__half*>(Rlo_)[(n0 + nn) * ldr + l0 + tx] = __float2half_rn((float)((v - (double)__half2float(hi)) * 2048.0));
        }
        else reinterpret_cast<float*>(R_)[(n0 + nn) * ldr + l0 + tx] = tf32_rna((float)v);
    }
}

// w[l] = sum_n V[n, l]^2 (rows above the diagonal are zeros): one block per local column
__global__ void __launch_bounds__(256)
colnorm2_cols_kernel(const double* __restrict__ V, int64_t ld, double* __restrict__ w)
{
    __shared__ double red[8];
    const double* col = V + (int64_t)blockIdx.x * ld;
    double s = 0.0;
    for (int64_t n = threadIdx.x; n < ld; n += 256) s = fma(col[n], col[n], s);
    s = lb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += red[i];
        w[blockIdx.x] = t;
    }
}

// out[n, c * 128 + kk] = plane of rank (c mod G), row n, local column (c / G) * 128 + kk; 16-byte pieces, one block per row
__global__ void __launch_bounds__(256)
linv_unpermute_kernel(const char* __restrict__ all, size_t chunk_bytes, size_t plane_off, int G, int T, int64_t Np, int64_t ldr, int esz,
    char* __restrict__ out)
{
    const int64_t n = blockIdx.x;
    const int tile_bytes = LB_TILE * esz, per_tile = tile_bytes / 16;
    for (int idx = threadIdx.x; idx < T * per_tile; idx += 256) {
        const int c = idx / per_tile, q = idx - c * per_tile;
        const char* src = all + (size_t)(c % G) * chunk_bytes + plane_off + ((size_t)n * ldr + (size_t)(c / G) * LB_TILE) * esz + (size_t)q * 16;
        char* dst = out + ((size_t)n * Np + (size_t)c * LB_TILE) * esz + (size_t)q * 16;
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    }
}

__global__ void __launch_bounds__(256)
linvw_unpermute_kernel(const char* __restrict__ all, size_t chunk_bytes, size_t w_off, int G, int64_t Np, double* __restrict__ w)
{
    const int64_t k = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (k >= Np) return;
    const int64_t c = k / LB_TILE, kk = k % LB_TILE;
    w[k] = reinterpret_cast<const double*>(all + (size_t)(c % G) * chunk_bytes + w_off)[(c / G) * LB_TILE + kk];
}

// sigma^2 from fp64 norms (split-operand mode): no rounding-bias term
__global__ void __launch_bounds__(256)
sigma2_split_kernel(const double* __restrict__ norm2, int64_t M, double kvv, double noise, double norm_unscale, double* __restrict__ s2)
{
    const int64_t c = blockIdx.x * (int64_t)256 + threadIdx.x;
    if (c >= M) return;
    double res = kvv - norm2[c] * norm_unscale;
    res = (res <= 2.220446049250313e-16) ? 0.0 : res; // gp.hpp:623
    s2[c] = res + noise;                               // gp.hpp:166
}

__global__ void __launch_bounds__(256)
sigma2_t32_kernel(const float* __restrict__ norm2, int64_t M, double kvv, double noise, double norm_unscale,
    const double* __restrict__ bias, double bias_coeff, double* __restrict__ s2)
{
    const int64_t c = blockIdx.x * (int64_t)256 + threadIdx.x;
    if (c >= M) return;
    const double nrm = (double)norm2[c];
    // Rounding both operands to an 11-bit significand adds zero-mean noise e_n to every D[c, n]; sum_n D^2 then carries the
    // positive bias E sum e_n^2 = 2 u_r^2 sum_k k*_k^2 |L^-1 e_k|^2 (u_r^2 = E[relative rounding error^2]), which grows with
    // cond(K) while the zero-mean part does not (DESIGN.md §4.5): subtract its expectation.
    double res = kvv - (nrm * norm_unscale - (bias ? bias_coeff * bias[c] : 0.0));
    res = (res <= 2.220446049250313e-16) ? 0.0 : res; // gp.hpp:623
    s2[c] = res + noise;                               // gp.hpp:166
}

} // namespace tf32q

// Prepare the row-major reduced-precision copy of L^-1 (rows padded with zeros to a multiple of the 256-row n-tile).
// fp32 (tf32 MMA) stores L^-1 as is; fp16 stores L^-1 * 2^e with e chosen so that max |.| <= 2^14.
int lb_tf32_prepare(lb_gp* h)
{
    using namespace tf32q;
    if (h->linv32_valid) return LB_OK;
    const bool split = (h->precision == 3); // fp16 hi / lo planes (LB_PREC_FP16X3)
    const bool f16 = (h->precision == 2) || split;
    int rc;
    if (!h->linv_valid && (rc = lb_launch_linv(h))) return rc;
    const int64_t Np = h->Np, Nr = (Np + BN - 1) / BN * BN;
    const size_t esz = split ? 4 : (f16 ? 2 : 4); // split: two fp16 planes of Nr x Np
    if ((rc = h->dLinv32.resize(h, esz * Nr * Np))) return rc;
    double scale = 1.0;
    if (f16) {
        if ((rc = lb_ensure_scratch(h, sizeof(double) * 1024))) return rc;
        absmax_kernel<<<1024, 256, 0, h->stream>>>(h->dLinv.get(), Np * Np, h->dScratch.get());
        h->launches++;
        double part[1024];
        LB_CUDA(cudaMemcpyAsync(part, h->dScratch.get(), sizeof(part), cudaMemcpyDeviceToHost, h->stream));
        LB_CUDA(cudaStreamSynchronize(h->stream));
        double mx = 0.0;
        for (double v : part) mx = v > mx ? v : mx;
        if (!(mx > 0.0) || !std::isfinite(mx)) return LB_ERR_STATE;
        scale = std::ldexp(1.0, 14 - (int)std::ceil(std::log2(mx)));
    }
    h->linv32_scale = scale;
    __half* lo_plane = split ? reinterpret_cast<__half*>(h->dLinv32.get()) + Nr * Np : nullptr;
    if (split) LB_CUDA(cudaMemsetAsync(h->dLinv32.get(), 0, esz * Nr * Np, h->stream)); // both planes incl. the padding rows
    else if (Nr > Np) LB_CUDA(cudaMemsetAsync((char*)h->dLinv32.get() + esz * Np * Np, 0, esz * (Nr - Np) * Np, h->stream));
    dim3 grid((unsigned)(Np / 32), (unsigned)(Np / 32));
    LbProfScope ps(h, h->stream, LB_PC_OTHER);
    if (f16) linv_to_rowmajor_kernel<true><<<grid, 256, 0, h->stream>>>(h->dLinv.get(), Np, h->dLinv32.get(), Np, scale, lo_plane);
    else linv_to_rowmajor_kernel<false><<<grid, 256, 0, h->stream>>>(h->dLinv.get(), Np, h->dLinv32.get(), Np, 1.0, nullptr);
    h->launches++;
    if ((rc = h->dLinvW.resize(h, sizeof(double) * Np))) return rc;
    colnorm2_kernel<<<(unsigned)Np, 256, 0, h->stream>>>(h->dLinv.get(), Np, h->dLinvW.get()); // weights of the rounding-bias correction
    h->launches++;
    LB_CUDA(cudaGetLastError());
    h->linv32_valid = true;
    return LB_OK;
}

// ---- the same copy assembled from the column chunks of G ranks (lb_dinv_* in abi.cu; limbo_b200/dist_inv.py) --------------------
static size_t dinv_plane_bytes(const lb_gp* h, int G)
{
    const bool f16 = (h->precision == 2) || (h->precision == 3);
    return (size_t)h->Np * (size_t)lb_linv_columns_width(h, G) * (f16 ? 2 : 4);
}

size_t lb_dinv_chunk_bytes_impl(const lb_gp* h, int G)
{
    return dinv_plane_bytes(h, G) * (h->precision == 3 ? 2 : 1) + sizeof(double) * (size_t)lb_linv_columns_width(h, G);
}

// max |V| over this rank's columns (host value; synchronises the handle's stream)
int lb_dinv_absmax(lb_gp* h, const double* dV, int G, double* out)
{
    using namespace tf32q;
    int rc;
    if ((rc = lb_ensure_scratch(h, sizeof(double) * 1024))) return rc;
    absmax_kernel<<<1024, 256, 0, h->stream>>>(dV, h->Np * lb_linv_columns_width(h, G), h->dScratch.get());
    h->launches++;
    double part[1024];
    LB_CUDA(cudaMemcpyAsync(part, h->dScratch.get(), sizeof(part), cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    double mx = 0.0;
    for (double v : part) mx = v > mx ? v : mx;
    *out = mx;
    return LB_OK;
}

// the fp16 scale lb_tf32_prepare derives from max |L^-1| (1 for tf32)
static int dinv_scale(const lb_gp* h, double absmax, double* scale)
{
    *scale = 1.0;
    if (h->precision == 2 || h->precision == 3) {
        if (!(absmax > 0.0) || !std::isfinite(absmax)) return LB_ERR_STATE;
        *scale = std::ldexp(1.0, 14 - (int)std::ceil(std::log2(absmax)));
    }
    return LB_OK;
}

int lb_dinv_pack_impl(lb_gp* h, const double* dV, int rank, int G, double absmax_all, void* dChunk)
{
    using namespace tf32q;
    const bool split = (h->precision == 3), f16 = (h->precision == 2) || split;
    const int64_t Np = h->Np, ldr = lb_linv_columns_width(h, G);
    const int T = (int)(Np / LB_TILE);
    double scale;
    int rc = dinv_scale(h, absmax_all, &scale);
    if (rc) return rc;
    char* base = reinterpret_cast<char*>(dChunk);
    const size_t plane = dinv_plane_bytes(h, G);
    dim3 grid((unsigned)(Np / 32), (unsigned)(ldr / 32));
    LbProfScope ps(h, h->stream, LB_PC_OTHER);
    if (f16) linv_cols_pack_kernel<true><<<grid, 256, 0, h->stream>>>(dV, Np, rank, G, T, base, ldr, scale, split ? base + plane : nullptr);
    else linv_cols_pack_kernel<false><<<grid, 256, 0, h->stream>>>(dV, Np, rank, G, T, base, ldr, 1.0, nullptr);
    colnorm2_cols_kernel<<<(unsigned)ldr, 256, 0, h->stream>>>(dV, Np, reinterpret_cast<double*>(base + plane * (split ? 2 : 1)));
    h->launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_dinv_adopt_impl(lb_gp* h, int G, const void* dAll, double absmax_all)
{
    using namespace tf32q;
    const bool split = (h->precision == 3), f16 = (h->precision == 2) || split;
    const int64_t Np = h->Np, Nr = (Np + BN - 1) / BN * BN, ldr = lb_linv_columns_width(h, G);
    const int T = (int)(Np / LB_TILE);
    const size_t esz = split ? 4 : (f16 ? 2 : 4), el = f16 ? 2 : 4;
    double scale;
    int rc = dinv_scale(h, absmax_all, &scale);
    if (rc) return rc;
    if ((rc = h->dLinv32.resize(h, esz * Nr * Np))) return rc;
    if ((rc = h->dLinvW.resize(h, sizeof(double) * Np))) return rc;
    h->linv32_scale = scale;
    const size_t chunk = lb_dinv_chunk_bytes_impl(h, G), plane = dinv_plane_bytes(h, G);
    const char* all = reinterpret_cast<const char*>(dAll);
    char* out = reinterpret_cast<char*>(h->dLinv32.get());
    LbProfScope ps(h, h->stream, LB_PC_OTHER);
    if (Nr > Np) { // padding rows of both planes
        LB_CUDA(cudaMemsetAsync(out + el * Np * Np, 0, el * (Nr - Np) * Np, h->stream));
        if (split) LB_CUDA(cudaMemsetAsync(out + el * Nr * Np + el * Np * Np, 0, el * (Nr - Np) * Np, h->stream));
    }
    linv_unpermute_kernel<<<(unsigned)Np, 256, 0, h->stream>>>(all, chunk, 0, G, T, Np, ldr, (int)el, out);
    if (split) linv_unpermute_kernel<<<(unsigned)Np, 256, 0, h->stream>>>(all, chunk, plane, G, T, Np, ldr, (int)el, out + el * Nr * Np);
    linvw_unpermute_kernel<<<(unsigned)((Np + 255) / 256), 256, 0, h->stream>>>(all, chunk, plane * (split ? 2 : 1), G, Np, h->dLinvW.get());
    h->launches += split ? 3 : 2;
    LB_CUDA(cudaGetLastError());
    h->linv32_valid = true;
    return LB_OK;
}

// K*^T chunk (reduced precision, K-major) and mu (M x P, fp64) for Mc candidates.
int lb_launch_kstar_tf32(const lb_gp* h, cudaStream_t st, int64_t Mc, const double* dQs, int64_t Mcp, float* dKt, double* dMuPart,
    double* dMu, double* dBias, long long* launches)
{
    using namespace tf32q;
    const bool split = (h->precision == 3);
    const bool f16 = (h->precision == 2) || split;
    const int64_t Np = h->Np;
    void* dKtLo = split ? (void*)(reinterpret_cast<__half*>(dKt) + Mcp * Np) : nullptr; // lo plane behind the hi plane of this chunk
    {
        LbProfScope ps(h, st, LB_PC_KSTAR);
        // interior tiles without bounds checks; the last tile row / column (when N or Mc is not a multiple of 128) with
        const int64_t nti = Np / LB_TILE, ntj = Mcp / LB_TILE;
        const int64_t fi = h->N / LB_TILE, fj = Mc / LB_TILE; // number of full tiles
        auto go = [&](auto kid, auto f16c, auto edgec, int64_t ia, int64_t ib, int64_t ja, int64_t jb) {
            if (ib <= ia || jb <= ja) return;
            const int64_t tiles = (ib - ia) * (jb - ja);
            kstar_t32_kernel<decltype(kid)::value, decltype(f16c)::value, decltype(edgec)::value, DCH_WIDE><<<(unsigned)tiles, 256, 0, st>>>(h->dXs, Np,
                h->N, dQs, Mcp, Mc, dKt, Np, h->kp, h->dAlpha, h->P, dMuPart, ia, ja, ib - ia, jb - ja, dBias ? h->dLinvW.get() : nullptr, dKtLo);
            if (launches) ++*launches;
        };
        auto go_prec = [&](auto kid) {
            auto run = [&](auto f16c) {
                go(kid, f16c, std::false_type{}, 0, fi, 0, fj);
                go(kid, f16c, std::true_type{}, fi, nti, 0, ntj);
                go(kid, f16c, std::true_type{}, 0, fi, fj, ntj);
            };
            if (f16) run(std::true_type{});
            else run(std::false_type{});
        };
        switch (h->kp.id) {
        case LB_K_SE_ARD: go_prec(std::integral_constant<int, LB_K_SE_ARD>{}); break;
        case LB_K_MATERN52: go_prec(std::integral_constant<int, LB_K_MATERN52>{}); break;
        case LB_K_MATERN32: go_prec(std::integral_constant<int, LB_K_MATERN32>{}); break;
        default: go_prec(std::integral_constant<int, LB_K_EXP>{}); break;
        }
    }
    {
        LbProfScope ps(h, st, LB_PC_QREDUCE);
        mu_reduce_kernel<<<(unsigned)((Mc + 255) / 256), 256, 0, st>>>(dMuPart, (int)(Np / LB_TILE), Mcp, h->P, Mc, dMu, dBias);
    }
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// sigma2 (M, fp64 container of a reduced-precision value) from a K*^T chunk: wgmma GEMM + row norms, then the clamp / noise of gp.hpp:618-624
int lb_launch_sigma_tf32(const lb_gp* h, cudaStream_t st, int64_t Mc, int64_t Mcp, const float* dKt, float* dNorm2, int* dErr,
    const double* dBias, double* dS2, long long* launches)
{
    using namespace tf32q;
    const bool split = (h->precision == 3);
    const bool f16 = (h->precision == 2) || split;
    const int64_t Np = h->Np, Nr = (Np + BN - 1) / BN * BN; // rows of the copy (lb_tf32_prepare)
    const double kscale = f16 ? 1.0 / h->kp.sf2 : 1.0;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    // D was computed from (K* kscale) and (L^-1 scale): |V|^2 = norm / (kscale scale)^2
    const double unscale = 1.0 / ((kscale * h->linv32_scale) * (kscale * h->linv32_scale));
    int rc;
    if (split) { // hi / lo planes, three MMAs per k-step, fp64 combination and norm (dNorm2 holds Mcp doubles)
        const __half* Ah = reinterpret_cast<const __half*>(dKt);
        const __half* Bh = reinterpret_cast<const __half*>(h->dLinv32.get());
        {
            LbProfScope ps(h, st, LB_PC_QSTEP);
            rc = lb_launch_split_gemm_norm(st, Ah, Ah + Mcp * Np, Np, Bh, Bh + Nr * Np, Np, Mcp, Nr, Np, 1,
                reinterpret_cast<double*>(dNorm2), dErr, sms);
        }
        if (rc) return rc;
        sigma2_split_kernel<<<(unsigned)((Mc + 255) / 256), 256, 0, st>>>(reinterpret_cast<const double*>(dNorm2), Mc, h->kp.sf2, h->kp.noise, unscale, dS2);
        if (launches) *launches += 2;
        LB_CUDA(cudaGetLastError());
        return LB_OK;
    }
    {
        LbProfScope ps(h, st, LB_PC_QSTEP);
        rc = lb_launch_tf32_gemm_norm(st, dKt, Np, h->dLinv32.get(), Np, Mcp, Nr, Np, 1, dNorm2, nullptr, dErr, sms, f16);
    }
    if (rc) return rc;
    // u_r^2 for round-to-nearest with an 11-bit significand and log-uniform mantissas: (2^-22 / 3) * 0.541; both operands: x 2
    const double bias_coeff = 2.0 * (1.0 / 4194304.0 / 3.0) * 0.541;
    sigma2_t32_kernel<<<(unsigned)((Mc + 255) / 256), 256, 0, st>>>(dNorm2, Mc, h->kp.sf2, h->kp.noise, unscale, dBias, bias_coeff, dS2);
    if (launches) *launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
