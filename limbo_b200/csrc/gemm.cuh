// limbo_b200/csrc/gemm.cuh — fp64 tensor-core (DMMA) tile GEMM building block.
//
// A CTA accumulates a 128 x BN tile  acc (+/-)= A(128 x K) * B(K x BN)  with a 3-stage cp.async
// pipeline.  Configurations (Cfg<BN, WN, BK, WM, CTAS>):
//   * warps: WM along M x WN along N  (THREADS = 32 * WM * WN); warp tile (128 / WM) x (BN / WN), i.e.
//     MT = 8 / WM m16 tiles by NT n8 tiles, MT * NT independent DMMA chains per warp; CTAS CTAs per SM:
//       Cfg<128, 4, 32, 4, 1>: 512 threads, one CTA per SM, 4 warps per sub-partition, 32 x 32 warp tiles;
//       Cfg< 64, 2, 16, 2, 2>: 128 threads, TWO CTAs per SM (90 KB smem, <= 255 regs), 64 x 32 warp tiles:
//                              2 warps per sub-partition with 16 chains each (the m16n8k4 rate of 8 warps
//                              per SM, DESIGN.md §4.1), and while one CTA is in its C-tile prologue / store
//                              epilogue the other one computes.
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
// k extent of one DMMA: every product of the core is a chain of m16n8k<MMA_K> steps (DESIGN.md §4.1).  All callers
// share it, so a tile's accumulator sees the same sequence of DMMAs whatever the launch scheme (the bit-identity of
// the pair / quad / distributed factorisations rests on that).
constexpr int MMA_K = 4;

template <int BN_, int WN_, int BK_, int WM_ = 4, int CTAS_ = 1>
struct Cfg {
    static constexpr int BN = BN_, WN = WN_, BK = BK_, WM = WM_;
    static constexpr int CTAS_PER_SM = CTAS_;     // __launch_bounds__ minimum blocks per SM
    static constexpr int THREADS = 32 * WM * WN;
    static constexpr int MT = BM / (16 * WM);     // m16 tiles per warp
    static constexpr int NT = BN / (8 * WN);      // n8 tiles per warp
    static constexpr int WTM = 16 * MT, WTN = 8 * NT; // warp tile
    static constexpr int PITCH_A_OC = BM + 4;     // [BK][128+4]
    static constexpr int PITCH_B_OC = BN + 4;     // [BK][BN+4]
    static constexpr int PITCH_KC = BK + 4;       // [outer][BK+4]
    static constexpr int A_STAGE = (BM * PITCH_KC > BK * PITCH_A_OC) ? BM * PITCH_KC : BK * PITCH_A_OC;
    static constexpr int B_STAGE = (BN * PITCH_KC > BK * PITCH_B_OC) ? BN * PITCH_KC : BK * PITCH_B_OC;
    static constexpr size_t PIPE_BYTES = (size_t)STAGES * (A_STAGE + B_STAGE) * sizeof(double);
    static constexpr int A_PIPE_DOUBLES = STAGES * A_STAGE; // offset of the B stages
    static_assert(BN % (8 * WN) == 0 && BM % (32 * WM) == 0 && (WM & (WM - 1)) == 0 && BK % MMA_K == 0, "tile shape");
    static_assert(PITCH_KC % 16 == 4 && PITCH_A_OC % 16 == 4 && PITCH_B_OC % 16 == 4, "conflict-free pitches");
};
using CfgWide = Cfg<128, 4, 32>;       // 512 threads, 1 CTA / SM, 32 x 32 warp tiles
using CfgDual = Cfg<64, 2, 16, 2, 2>;  // 128 threads, 2 CTAs / SM, 64 x 32 warp tiles
using CfgStep = Cfg<64, 4, 32>;        // 512 threads, 64-wide right-hand sides (multi-launch TRSM path)

// Per-thread copy plan for one operand: which 16-byte chunks of a (NOUTER x BK) slab this thread moves.  The
// chunk -> (global offset, shared offset) mapping is the same for every k-slab, so it is computed once; per
// pipeline stage only a base pointer advances (the per-stage index arithmetic used to sit between the CTA
// barrier and the first DMMA of every stage).  Chunk q of a thread is chunk 0 moved by q * THREADS / CPR
// outer rows (KC) or k rows (outer-contiguous), so the plan is one offset pair and one global stride: three
// registers instead of three per chunk, which the k loop of the 128-register configurations needs.
template <typename C, bool KC, int NOUTER, int PITCH_OC>
struct TilePlan {
    static constexpr int CHUNKS = NOUTER * C::BK / 2;
    static constexpr int PER_THREAD = (CHUNKS + C::THREADS - 1) / C::THREADS;
    static constexpr int CPR = KC ? C::BK / 2 : NOUTER / 2; // chunks per row of the slab
    static constexpr int ROWS_PER_Q = C::THREADS / CPR;
    static constexpr int SSTEP = ROWS_PER_Q * (KC ? C::PITCH_KC : PITCH_OC);
    static_assert(C::THREADS % CPR == 0, "every chunk of a thread sits in the same column of the slab");
    int64_t goff, gstep;
    int soff;
    __device__ __forceinline__ void init(int64_t ld)
    {
        const int row = threadIdx.x / CPR, cc = threadIdx.x - row * CPR;
        // KC: element (o, k) at g[k + o*ld], smem [o][k]; otherwise element (o, k) at g[o + k*ld], smem [k][o]
        goff = (int64_t)row * ld + 2 * cc;
        gstep = (int64_t)ROWS_PER_Q * ld;
        soff = row * (KC ? C::PITCH_KC : PITCH_OC) + 2 * cc;
    }
    __device__ __forceinline__ void issue(double* s, const double* __restrict__ g) const
    {
        s += soff;
        g += goff;
#pragma unroll
        for (int q = 0; q < PER_THREAD; ++q)
            if (CHUNKS % C::THREADS == 0 || (int)threadIdx.x + q * C::THREADS < CHUNKS) lb_cp_async16(s + q * SSTEP, g + q * gstep);
    }
};

// Accumulators of one warp: MT m16-tiles x NT n8-tiles.
template <typename C>
struct Acc {
    double v[C::MT][C::NT][4];
    __device__ __forceinline__ void zero()
    {
#pragma unroll
        for (int a = 0; a < C::MT; ++a)
#pragma unroll
            for (int b = 0; b < C::NT; ++b)
#pragma unroll
                for (int c = 0; c < 4; ++c) v[a][b][c] = 0.0;
    }
};

// Origin of this warp's tile in the CTA tile; warps are numbered M-fastest.
template <typename C>
__device__ __forceinline__ int warp_row0() { return ((int)(threadIdx.x >> 5) & (C::WM - 1)) * C::WTM; }
template <typename C>
__device__ __forceinline__ int warp_col0() { return ((int)(threadIdx.x >> 5) / C::WM) * C::WTN; }

// One k-step of MMA_K for the warp tile: the A fragments of the MT m16 tiles, the B fragments of the NT n8 tiles, then
// MT*NT independent DMMA.16x8xMMA_K.  fa(dm, dk) / fb(dn, dk) read the operand at row / column (base + dm / dn) and
// k (k0 + t + dk) of this thread, base including g: a[mt][i] is row 16 mt + g + 8 (i&1), k t + 4 (i>>1); b[nt][i] is
// k t + 4 i, column 8 nt + g.  Those are the words MMA_K/4 steps of k4 fragment loads read, so the padded pitches
// stay bank-conflict free.
template <typename C, bool NEG_A, typename FA, typename FB>
__device__ __forceinline__ void mma_kstep(Acc<C>& acc, FA fa, FB fb)
{
    double a[C::MT][MMA_K / 2], b[C::NT][MMA_K / 4];
#pragma unroll
    for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
        for (int i = 0; i < MMA_K / 2; ++i) {
            a[mt][i] = fa(mt * 16 + 8 * (i & 1), 4 * (i >> 1));
            if (NEG_A) a[mt][i] = -a[mt][i];
        }
#pragma unroll
    for (int nt = 0; nt < C::NT; ++nt)
#pragma unroll
        for (int i = 0; i < MMA_K / 4; ++i) b[nt][i] = fb(nt * 8, 4 * i);
#pragma unroll
    for (int nt = 0; nt < C::NT; ++nt)
#pragma unroll
        for (int mt = 0; mt < C::MT; ++mt) lb_dmma_16x8<MMA_K>(acc.v[mt][nt], a[mt], b[nt]);
}

template <typename C, bool A_KC, bool B_KC, bool NEG_A>
__device__ __forceinline__ void compute_stage(Acc<C>& acc, const double* sA, const double* sB)
{
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int m_base = warp_row0<C>() + g, n_base = warp_col0<C>() + g;
    // two k-steps per trip: fully unrolled, ptxas hoists the fragment loads of the whole stage and the 128-register
    // configurations spill inside the k loop (the m16n8k4 operands sit in aligned register pairs / quads); CfgDual
    // (255 registers) fits either way, and measured faster by two (DESIGN.md §4.1)
#pragma unroll 2
    for (int k0 = 0; k0 < C::BK; k0 += MMA_K) {
        const int k = k0 + t;
        mma_kstep<C, NEG_A>(
            acc,
            [&](int dm, int dk) { return A_KC ? sA[(m_base + dm) * C::PITCH_KC + k + dk] : sA[(k + dk) * C::PITCH_A_OC + m_base + dm]; },
            [&](int dn, int dk) { return B_KC ? sB[(n_base + dn) * C::PITCH_KC + k + dk] : sB[(k + dk) * C::PITCH_B_OC + n_base + dn]; });
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
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int row0 = warp_row0<C>(), col0 = warp_col0<C>();
#pragma unroll
    for (int mt = 0; mt < C::MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < C::NT; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int row = row0 + mt * 16 + g + 8 * (i >> 1);
                int col = col0 + nt * 8 + 2 * t + (i & 1);
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
    const int lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int m_base = warp_row0<C>() + g, n_base = warp_col0<C>() + g;
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
        for (int k0 = 0; k0 < C::BK; k0 += MMA_K) {
            const int k = k0 + t;
            mma_kstep<C, false>(
                acc, [&](int dm, int dk) { return sA[(k + dk) * C::PITCH_A_OC + m_base + dm]; },
                [&](int dn, int dk) { return sBres[(n_base + dn) * PB + kt * C::BK + k + dk]; });
        }
    }
    lb_cp_async_wait<0>();
    __syncthreads();
}

} // namespace lbg
