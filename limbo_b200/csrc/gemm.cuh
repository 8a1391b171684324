// limbo_b200/csrc/gemm.cuh — fp64 tensor-core (DMMA) tile GEMM building block.
//
// A CTA accumulates a 128 x BN tile  acc (+/-)= A(128 x K) * B(K x BN)  with a 3-stage cp.async
// pipeline.  Configurations (Cfg<BN, WN, BK>):
//   * warps: 4 along M x WN along N  (THREADS = 128 * WN); warp tile 32 x (BN / WN);
//     both configurations keep >= 2 DMMA-issuing warps per SM sub-partition, so that the dependent
//     DMMAs of one warp do not leave the pipe idle:
//       Cfg<128, 4, 32>: 512 threads, one CTA per SM, 4 warps per sub-partition;
//       Cfg< 64, 2, 16>: 256 threads, TWO CTAs per SM (77 KB smem, <= 128 regs): while one CTA
//                        is in its C-tile prologue / store epilogue the other one computes.
//   * operands "outer-contiguous" (the m / n index is the unit-stride one, i.e. a column-major
//     block) or "K-contiguous"; shared tiles are padded by 4 doubles so every 64-bit fragment
//     load is bank-conflict free (DESIGN.md §4.1).
//   * NEG_A: acc -= A*B, so a tile update C - A*B preloads C into the accumulators and those loads
//     overlap the pipeline prologue instead of a dependent load-subtract-store epilogue.
//
// This replaces the arithmetic the reference delegates to Eigen:
//   LLT trailing update / panel solve            model/gp.hpp:565
//   triangular solves for alpha, sigma^2, K^-1   model/gp.hpp:260-261,608-610,620
#pragma once
#include "common.cuh"

namespace lbg {

constexpr int BM = 128;
constexpr int STAGES = 3;

// DF_ = number of n8-tiles per warp (0 or 1, the last ones) whose 32 x 8 strip is computed with plain DFMA instead of DMMA
// (the LB_SYRK_DF=1 experiment: part of the tile on the fp64 ALU pipe beside DMMA; off by default).
template <int BN_, int WN_, int BK_, int DF_ = 0>
struct Cfg {
    static constexpr int BN = BN_, WN = WN_, BK = BK_, DF = DF_;
    static constexpr int THREADS = 128 * WN;
    static constexpr int NT = BN / (8 * WN);      // n8 tiles per warp
    static constexpr int PITCH_A_OC = BM + 4;     // [BK][128+4]
    static constexpr int PITCH_B_OC = BN + 4;     // [BK][BN+4]
    static constexpr int PITCH_KC = BK + 4;       // [outer][BK+4]
    static constexpr int A_STAGE = (BM * PITCH_KC > BK * PITCH_A_OC) ? BM * PITCH_KC : BK * PITCH_A_OC;
    static constexpr int B_STAGE = (BN * PITCH_KC > BK * PITCH_B_OC) ? BN * PITCH_KC : BK * PITCH_B_OC;
    static constexpr size_t PIPE_BYTES = (size_t)STAGES * (A_STAGE + B_STAGE) * sizeof(double);
    static constexpr int A_PIPE_DOUBLES = STAGES * A_STAGE; // offset of the B stages
    static_assert(BN % (8 * WN) == 0 && BK % 8 == 0, "tile shape");
    static_assert(PITCH_KC % 16 == 4 && PITCH_A_OC % 16 == 4 && PITCH_B_OC % 16 == 4, "conflict-free pitches");
};
using CfgWide = Cfg<128, 4, 32>;  // 512 threads, 1 CTA / SM
using CfgDual = Cfg<64, 2, 16>;   // 256 threads, 2 CTAs / SM
using CfgDualDF = Cfg<64, 2, 16, 1>; // same, one n8-tile of every warp on the fp64 ALU pipe (experiment: DESIGN.md §4.1)
using CfgStep = Cfg<64, 4, 32>;   // 512 threads, 64-wide right-hand sides (multi-launch TRSM path)

// Per-thread copy plan for one operand: which 16-byte chunks of a (NOUTER x BK) slab this thread moves.  The
// chunk -> (global offset, shared offset) mapping is the same for every k-slab, so it is computed once; per
// pipeline stage only a base pointer advances (the per-stage index arithmetic used to sit between the CTA
// barrier and the first DMMA of every stage).
template <typename C, bool KC, int NOUTER, int PITCH_OC>
struct TilePlan {
    static constexpr int CHUNKS = NOUTER * C::BK / 2;
    static constexpr int PER_THREAD = (CHUNKS + C::THREADS - 1) / C::THREADS;
    int64_t goff[PER_THREAD];
    int soff[PER_THREAD];
    __device__ __forceinline__ void init(int64_t ld)
    {
#pragma unroll
        for (int q = 0; q < PER_THREAD; ++q) {
            const int c = threadIdx.x + q * C::THREADS;
            if (KC) { // element (o, k) at g[k + o*ld]; smem [o][k]
                constexpr int CPR = C::BK / 2;
                const int o = c / CPR, kc = c - o * CPR;
                goff[q] = (int64_t)o * ld + 2 * kc;
                soff[q] = o * C::PITCH_KC + 2 * kc;
            }
            else { // element (o, k) at g[o + k*ld]; smem [k][o]
                constexpr int CPR = NOUTER / 2;
                const int k = c / CPR, oc = c - k * CPR;
                goff[q] = (int64_t)k * ld + 2 * oc;
                soff[q] = k * PITCH_OC + 2 * oc;
            }
        }
    }
    __device__ __forceinline__ void issue(double* s, const double* __restrict__ g) const
    {
#pragma unroll
        for (int q = 0; q < PER_THREAD; ++q)
            if (CHUNKS % C::THREADS == 0 || (int)threadIdx.x + q * C::THREADS < CHUNKS) lb_cp_async16(s + soff[q], g + goff[q]);
    }
};

// Accumulators of one warp: 2 m16-tiles x NT n8-tiles.
template <typename C>
struct Acc {
    double v[2][C::NT][4];
    __device__ __forceinline__ void zero()
    {
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < C::NT; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) v[a][b][c] = 0.0;
    }
};

template <typename C, bool A_KC, bool B_KC, bool NEG_A>
__device__ __forceinline__ void compute_stage(Acc<C>& acc, const double* sA, const double* sB)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int m_base = wm * 32, n_base = wn * (C::BN / C::WN);
    constexpr int NTM = C::NT - C::DF; // n8-tiles on the tensor pipe
#pragma unroll
    for (int k0 = 0; k0 < C::BK; k0 += 4) {
        // one k4 step: 4 A values (rows g, g+8 of both m16 tiles), NTM B values, then 4*NTM independent DMMA.8x8x4
        double a[2][2], b[NTM > 0 ? NTM : 1];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                int m = m_base + mt * 16 + g + 8 * i;
                int k = k0 + t;
                a[mt][i] = A_KC ? sA[m * C::PITCH_KC + k] : sA[k * C::PITCH_A_OC + m];
                if (NEG_A) a[mt][i] = -a[mt][i];
            }
#pragma unroll
        for (int nt = 0; nt < NTM; ++nt) {
            int n = n_base + nt * 8 + g;
            int k = k0 + t;
            b[nt] = B_KC ? sB[n * C::PITCH_KC + k] : sB[k * C::PITCH_B_OC + n];
        }
#pragma unroll
        for (int nt = 0; nt < NTM; ++nt)
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                lb_dmma_8x8x4(acc.v[mt][nt][0], acc.v[mt][nt][1], a[mt][0], b[nt]);
                lb_dmma_8x8x4(acc.v[mt][nt][2], acc.v[mt][nt][3], a[mt][1], b[nt]);
            }
        if (C::DF > 0) {
            // the last n8-tile on the fp64 ALU pipe, same accumulator layout as a DMMA C fragment: rows g, g+8 (per m16 tile),
            // columns 2t, 2t+1; every lane needs all four k of the step (the 4 lanes of a row / the 8 lanes of a column pair
            // read the same words: broadcast)
            constexpr int nt = C::NT - 1;
            const int n = n_base + nt * 8 + 2 * t;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const int k = k0 + kk;
                const double bx = B_KC ? sB[n * C::PITCH_KC + k] : sB[k * C::PITCH_B_OC + n];
                const double by = B_KC ? sB[(n + 1) * C::PITCH_KC + k] : sB[k * C::PITCH_B_OC + n + 1];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int m = m_base + mt * 16 + g + 8 * i;
                        double av = A_KC ? sA[m * C::PITCH_KC + k] : sA[k * C::PITCH_A_OC + m];
                        if (NEG_A) av = -av;
                        acc.v[mt][nt][2 * i] = fma(av, bx, acc.v[mt][nt][2 * i]);
                        acc.v[mt][nt][2 * i + 1] = fma(av, by, acc.v[mt][nt][2 * i + 1]);
                    }
            }
        }
    }
}

// acc += A * B (acc -= A * B with NEG_A) over K (multiple of BK).  gA/gB point at the (0,0) element of
// the operand tile for k = 0; stepping k by BK advances an outer-contiguous operand by BK*ld and a
// K-contiguous one by BK.  All threads must call.  smem: C::PIPE_BYTES.  On return all cp.async groups
// are drained and the CTA is synchronised (smem may be reused).
template <typename C, bool A_KC, bool B_KC, bool NEG_A = false>
__device__ __forceinline__ void mainloop(Acc<C>& acc, const double* __restrict__ gA, int64_t lda,
    const double* __restrict__ gB, int64_t ldb, int K, double* smem)
{
    double* sA = smem;
    double* sB = smem + C::A_PIPE_DOUBLES;
    const int nk = K / C::BK;
    const int64_t stepA = A_KC ? C::BK : (int64_t)C::BK * lda;
    const int64_t stepB = B_KC ? C::BK : (int64_t)C::BK * ldb;
    TilePlan<C, A_KC, BM, C::PITCH_A_OC> pa;
    TilePlan<C, B_KC, C::BN, C::PITCH_B_OC> pb;
    pa.init(lda);
    pb.init(ldb);
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        if (s < nk) {
            pa.issue(sA + s * C::A_STAGE, gA + s * stepA);
            pb.issue(sB + s * C::B_STAGE, gB + s * stepB);
        }
        lb_cp_async_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
        lb_cp_async_wait<STAGES - 2>();
        __syncthreads();
        // compute first: the DMMA stream restarts right after the barrier; the prefetch of slab kt+2 (whose slot
        // was last read in iteration kt-1, i.e. before this barrier) is issued behind it
        const int s = kt % STAGES;
        compute_stage<C, A_KC, B_KC, NEG_A>(acc, sA + s * C::A_STAGE, sB + s * C::B_STAGE);
        const int nx = kt + STAGES - 1;
        if (nx < nk) {
            const int sn = nx % STAGES;
            pa.issue(sA + sn * C::A_STAGE, gA + nx * stepA);
            pb.issue(sB + sn * C::B_STAGE, gB + nx * stepB);
        }
        lb_cp_async_commit();
    }
    lb_cp_async_wait<0>();
    __syncthreads();
}

// Apply f(row, col, value&) to every accumulator element of this thread (row in [0,128), col in [0,BN)).
template <typename C, typename F>
__device__ __forceinline__ void for_each_acc(Acc<C>& acc, F&& f)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < C::NT; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int row = wm * 32 + mt * 16 + g + 8 * (i >> 1);
                int col = wn * (C::BN / C::WN) + nt * 8 + 2 * t + (i & 1);
                f(row, col, acc.v[mt][nt][i]);
            }
}

// acc <- C tile (column-major, ld): plain loads, no arithmetic, so they stay in flight while the
// cp.async prologue is issued.
template <typename C>
__device__ __forceinline__ void load_acc(Acc<C>& acc, const double* __restrict__ Cg, int64_t ld)
{
    for_each_acc<C>(acc, [&](int r, int c, double& v) { v = __ldcs(Cg + r + (int64_t)c * ld); });
}
template <typename C>
__device__ __forceinline__ void store_acc(Acc<C>& acc, double* __restrict__ Cg, int64_t ld)
{
    for_each_acc<C>(acc, [&](int r, int c, double& v) { Cg[r + (int64_t)c * ld] = v; });
}

// Second-phase product with a resident B operand: acc2 += A(128 x 128) * Bres where Bres is in shared
// memory as [n][k] with pitch BM+4 (k-contiguous) and A (outer-contiguous, ld = lda) streams through the
// A pipeline stages.  smem_pipe: the A stage area.
template <typename C>
__device__ __forceinline__ void mainloop_resB(Acc<C>& acc, const double* __restrict__ gA, int64_t lda,
    const double* sBres, double* smem_pipe)
{
    constexpr int PB = BM + 4;
    constexpr int nk = BM / C::BK;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    const int m_base = wm * 32, n_base = wn * (C::BN / C::WN);
    TilePlan<C, false, BM, C::PITCH_A_OC> pa;
    pa.init(lda);
#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) {
        pa.issue(smem_pipe + s * C::A_STAGE, gA + (int64_t)s * C::BK * lda);
        lb_cp_async_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
        lb_cp_async_wait<STAGES - 2>();
        __syncthreads();
        const int nx = kt + STAGES - 1;
        if (nx < nk) pa.issue(smem_pipe + (nx % STAGES) * C::A_STAGE, gA + (int64_t)nx * C::BK * lda);
        lb_cp_async_commit();
        const double* sA = smem_pipe + (kt % STAGES) * C::A_STAGE;
#pragma unroll
        for (int k0 = 0; k0 < C::BK; k0 += 4) {
            double a[2][2], b[C::NT];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int i = 0; i < 2; ++i) a[mt][i] = sA[(k0 + t) * C::PITCH_A_OC + m_base + mt * 16 + g + 8 * i];
#pragma unroll
            for (int nt = 0; nt < C::NT; ++nt) b[nt] = sBres[(n_base + nt * 8 + g) * PB + kt * C::BK + k0 + t];
#pragma unroll
            for (int nt = 0; nt < C::NT; ++nt)
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    lb_dmma_8x8x4(acc.v[mt][nt][0], acc.v[mt][nt][1], a[mt][0], b[nt]);
                    lb_dmma_8x8x4(acc.v[mt][nt][2], acc.v[mt][nt][3], a[mt][1], b[nt]);
                }
        }
    }
    lb_cp_async_wait<0>();
    __syncthreads();
}

} // namespace lbg
