// limbo_b200/csrc/potrf.cu — blocked right-looking Cholesky, trailing update on
// fp64 tensor cores (DMMA).
//
// Replaces `_matrixL = Eigen::LLT<Eigen::MatrixXd>(_kernel).matrixL()`
// (model/gp.hpp:565).  Per 128-column panel k:
//   1. potf2_inv_kernel : factor the 128x128 diagonal block in one CTA
//                         (32x32 sub-blocks in registers via warp shuffles) and
//                         form its inverse (kept in invD for every later
//                         triangular solve);
//   2. trsm_panel_kernel: L[i,k] = A[i,k] * inv(L[k,k])^T   (DMMA GEMM)
//   3. syrk_kernel      : A[i,j] -= L[i,k] * L[j,k]^T, k < j <= i (DMMA GEMM)
// A non-positive pivot is reported LAPACK-style through info (the reference
// never checks Eigen's info(), SURVEY.md §5).
#include "gemm.cuh"
#include <cstdlib>

namespace {

constexpr int PS = LB_TILE + 4;   // pitch of the diagonal block in smem (== 4 mod 16: conflict-free DMMA fragment loads)
constexpr int XP = 36;            // pitch of a 32x32 inverse block
constexpr int XB = 32 * XP;
constexpr size_t POTF2_SMEM = (size_t)(LB_TILE * PS + 10 * XB + LB_TILE) * sizeof(double);

__device__ __forceinline__ int blk(int ib, int jb) { return ib * (ib + 1) / 2 + jb; }

// One warp: c(16x8) += sum_k A(m,k) B(k,n), K a multiple of lbg::MMA_K; fa(m,k), fb(k,n) read shared memory.
// The same DMMA shape as the tile GEMM core (gemm.cuh).
template <typename FA, typename FB>
__device__ __forceinline__ void warp_mma(double (&c)[4], int K, FA fa, FB fb)
{
    constexpr int KS = lbg::MMA_K;
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    for (int k0 = 0; k0 < K; k0 += KS) {
        double a[KS / 2], b[KS / 4];
#pragma unroll
        for (int i = 0; i < KS / 2; ++i) a[i] = fa(g + 8 * (i & 1), k0 + t + 4 * (i >> 1));
#pragma unroll
        for (int i = 0; i < KS / 4; ++i) b[i] = fb(k0 + t + 4 * i, g);
        lb_dmma_16x8<KS>(c, a, b);
    }
}

__device__ __forceinline__ double rsqrt_nr(double x)
{
    // branch-free reciprocal square root: MUFU.RSQ64H seed + two Newton steps (<= 1 ulp for normal x)
    double r;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    double h = 0.5 * x;
    r = fma(r, fma(-h * r, r, 0.5), r);
    r = fma(r, fma(-h * r, r, 0.5), r);
    return r;
}

// Factor the 128x128 diagonal block k of L in place and form its inverse (invD[k]).
// Panel work is latency bound (a chain of 128 dependent pivots), so everything that is
// not on that chain runs on the tensor cores from shared memory (block kept COLUMN-major,
// S[c*PS + r], so global <-> shared copies are 16-byte vectors and every DMMA fragment
// load is bank-conflict free):
//   per 32-column sub-block jb:
//     warp 0   : 32x32 Cholesky in registers (row per lane, warp shuffles, branch-free
//                rsqrt) and its inverse by column-oriented substitution;
//     all warps: rows below  X = A * inv(Ld)^T      (DMMA, in place)
//                trailing    A22 -= X X^T           (DMMA, lower tiles)
//   then the off-diagonal blocks of inv(L_kk) block row by block row (DMMA).
__global__ void __launch_bounds__(256, 1)
potf2_inv_kernel(double* __restrict__ L, int64_t ld, int k, double* __restrict__ invD, int* __restrict__ info, int do_factor,
    long long* __restrict__ clk = nullptr)
{
    int clk_n = 0;
#define LB_TICK() do { if (clk && threadIdx.x == 0) clk[clk_n++] = clock64(); } while (0)
    LB_TICK();
    extern __shared__ __align__(16) double smem[];
    double* S = smem;                         // [128 cols][PS]   S[c*PS + r]
    double* Xb = smem + LB_TILE * PS;         // 10 blocks [32 cols][XP]  X[c*XP + r]
    double* sInv = Xb + 10 * XB;              // [128] reciprocal diagonal
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int64_t k0 = (int64_t)k * LB_TILE;
    double* Lkk = L + k0 + k0 * ld;

    for (int idx = tid; idx < LB_TILE * (LB_TILE / 2); idx += 256) { // 16-byte chunks, coalesced along rows
        const int c = idx >> 6, r = (idx & 63) * 2;
        lb_cp_async16(&S[c * PS + r], Lkk + r + (int64_t)c * ld);
    }
    lb_cp_async_commit();
    lb_cp_async_wait<0>();
    __syncthreads();
    LB_TICK();
    int bad = 0;

    for (int jb = 0; jb < 4; ++jb) {
        const int c0 = 32 * jb;
        if (warp == 0) {
            double a[32];
            if (do_factor) {
                // ---- 32x32 Cholesky, one row per lane, right-looking ----
#pragma unroll
                for (int c = 0; c < 32; ++c) a[c] = S[(c0 + c) * PS + c0 + lane];
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const double ajj = __shfl_sync(0xffffffffu, a[j], j);
                    if (!(ajj > 0.0) && bad == 0) bad = c0 + j + 1;
                    const double inv = rsqrt_nr(ajj);
                    const double d = ajj * inv;
                    const double lij = (lane > j) ? a[j] * inv : ((lane == j) ? d : 0.0);
                    a[j] = lij;
                    if (lane == j) sInv[c0 + j] = inv;
#pragma unroll
                    for (int kk = j + 1; kk < 32; ++kk) {
                        const double lkj = __shfl_sync(0xffffffffu, lij, kk);
                        a[kk] = fma(-lij, lkj, a[kk]);
                    }
                }
#pragma unroll
                for (int c = 0; c < 32; ++c) S[(c0 + c) * PS + c0 + lane] = (c <= lane) ? a[c] : 0.0;
            }
            else {
                sInv[c0 + lane] = 1.0 / S[(c0 + lane) * PS + c0 + lane];
            }
            __syncwarp();
            if (jb == 0) LB_TICK();
            // ---- inverse of the 32x32 diagonal sub-block: lane = column of X, column-oriented ----
            double x[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) x[i] = (i == lane) ? 1.0 : 0.0;
#pragma unroll
            for (int kk = 0; kk < 32; ++kk) {
                const double xk = x[kk] * sInv[c0 + kk];
                x[kk] = xk;
#pragma unroll
                for (int i = kk + 1; i < 32; ++i) x[i] = fma(-S[(c0 + kk) * PS + c0 + i], xk, x[i]);
            }
            double* X = Xb + blk(jb, jb) * XB;
#pragma unroll
            for (int i = 0; i < 32; ++i) X[lane * XP + i] = (i >= lane) ? x[i] : 0.0;
        }
        __syncthreads();
        if (jb == 0) LB_TICK();
        if (!do_factor) continue;
        const int nrem = LB_TILE - c0 - 32;
        const int r0 = c0 + 32;
        // ---- rows below: X = A * inv(Ld)^T, in place; one m16 row tile (all 4 n8 tiles) per warp ----
        const double* Wd = Xb + blk(jb, jb) * XB;
        for (int mt = warp; mt < nrem / 16; mt += 8) {
            const int rb = r0 + 16 * mt;
            double acc[4][4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[nt][e] = 0.0;
                warp_mma(acc[nt], 32, [&](int m, int kk) { return S[(c0 + kk) * PS + rb + m]; },
                    [&](int kk, int n) { return Wd[kk * XP + 8 * nt + n]; }); // (Wd^T)(kk, n) = Wd[n][kk]
            }
            __syncwarp();
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) S[(c0 + 8 * nt + 2 * t + (e & 1)) * PS + rb + g + 8 * (e >> 1)] = acc[nt][e];
        }
        __syncthreads();
        if (jb == 0) LB_TICK();
        // ---- trailing update of the block: A22 -= X X^T (tiles touching the lower triangle) ----
        {
            const int mts = nrem / 16, nts = nrem / 8;
            int w = 0;
            for (int mt = 0; mt < mts; ++mt)
                for (int nt = 0; nt < nts && nt <= 2 * mt + 1; ++nt, ++w) {
                    if ((w & 7) != warp) continue;
                    const int rb = r0 + 16 * mt, cb = r0 + 8 * nt;
                    double c[4];
#pragma unroll
                    for (int e = 0; e < 4; ++e) c[e] = 0.0;
                    warp_mma(c, 32, [&](int m, int kk) { return S[(c0 + kk) * PS + rb + m]; },
                        [&](int kk, int n) { return S[(c0 + kk) * PS + cb + n]; });
#pragma unroll
                    for (int e = 0; e < 4; ++e) S[(cb + 2 * t + (e & 1)) * PS + rb + g + 8 * (e >> 1)] -= c[e];
                }
        }
        __syncthreads();
    }
    if (bad && tid == 0) atomicCAS(info, 0, (int)(k0 + bad));

    LB_TICK();
    // ---- off-diagonal blocks of the inverse, block row by block row:
    //      X[ib,jb] = -X[ib,ib] * sum_{kb=jb}^{ib-1} L[ib,kb] X[kb,jb]
    for (int ib = 1; ib < 4; ++ib) {
        // T[jb] (32x32) -> free upper block (rows of jb, cols of ib) of S; 8 mma tiles per jb
        for (int w = warp; w < 8 * ib; w += 8) {
            const int jb = w >> 3, mt = (w >> 2) & 1, nt = w & 3;
            double c[4] = {0.0, 0.0, 0.0, 0.0};
            for (int kb = jb; kb < ib; ++kb) {
                const double* Xk = Xb + blk(kb, jb) * XB;
                warp_mma(c, 32, [&](int m, int kk) { return S[(32 * kb + kk) * PS + 32 * ib + 16 * mt + m]; },
                    [&](int kk, int n) { return Xk[(8 * nt + n) * XP + kk]; });
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) S[(32 * ib + 8 * nt + 2 * t + (e & 1)) * PS + 32 * jb + 16 * mt + g + 8 * (e >> 1)] = c[e];
        }
        __syncthreads();
        const double* Xd = Xb + blk(ib, ib) * XB;
        for (int w = warp; w < 8 * ib; w += 8) {
            const int jb = w >> 3, mt = (w >> 2) & 1, nt = w & 3;
            double c[4] = {0.0, 0.0, 0.0, 0.0};
            warp_mma(c, 32, [&](int m, int kk) { return Xd[kk * XP + 16 * mt + m]; },
                [&](int kk, int n) { return S[(32 * ib + 8 * nt + n) * PS + 32 * jb + kk]; });
            double* Xo = Xb + blk(ib, jb) * XB;
#pragma unroll
            for (int e = 0; e < 4; ++e) Xo[(8 * nt + 2 * t + (e & 1)) * XP + 16 * mt + g + 8 * (e >> 1)] = -c[e];
        }
        __syncthreads();
    }
    LB_TICK();
    // ---- write back L[k,k] (clean lower) and inv(L[k,k]): two consecutive rows per 16-byte store ----
    double* inv_out = invD + (int64_t)k * LB_TILE * LB_TILE;
    for (int idx = tid; idx < LB_TILE * (LB_TILE / 2); idx += 256) {
        const int c = idx >> 6, r = (idx & 63) * 2;
        if (c > r + 1) continue; // strictly upper part: never read by any consumer (invD is zero-initialised)
        if (do_factor) {
            double2 v = *reinterpret_cast<const double2*>(&S[c * PS + r]);
            if (c > r) v.x = 0.0;
            if (c > r + 1) v.y = 0.0;
            *reinterpret_cast<double2*>(Lkk + r + (int64_t)c * ld) = v;
        }
        double2 x = make_double2(0.0, 0.0);
        if (c <= r + 1) {
            const double* Xs_ = Xb + blk(r >> 5, c >> 5) * XB + (c & 31) * XP + (r & 31);
            x = *reinterpret_cast<const double2*>(Xs_);
            if (c > r) x.x = 0.0;
        }
        *reinterpret_cast<double2*>(inv_out + r + c * LB_TILE) = x;
    }
    __syncthreads();
    LB_TICK();
#undef LB_TICK
}

// L[i,k] <- A[i,k] * inv(L[k,k])^T for i = k+1 .. T-1
__global__ void __launch_bounds__(lbg::CfgWide::THREADS, 1)
trsm_panel_kernel(double* __restrict__ L, int64_t ld, int k, const double* __restrict__ invD)
{
    using C = lbg::CfgWide;
    extern __shared__ __align__(16) double smem[];
    const int i = k + 1 + blockIdx.x;
    double* A = L + (int64_t)i * LB_TILE + (int64_t)k * LB_TILE * ld;
    const double* B = invD + (int64_t)k * LB_TILE * LB_TILE; // B(kk,n) = inv[n + kk*128]
    lbg::Acc<C> acc;
    acc.zero();
    lbg::mainloop<C, false, false>(acc, A, ld, B, LB_TILE, LB_TILE, smem);
    lbg::store_acc<C>(acc, A, ld);
}

// Trailing update with the panel block columns [kb, kb + kd):
//   A[i,j] -= L[i, kb:kb+kd] L[j, kb:kb+kd]^T   for j in [j0, j0 + nc), j <= i < T
// (kd = 1: one 128-column panel, K = 128; kd = 2: two panels at once, K = 256 —
// half the C traffic and half the tile prologues per flop).  C is preloaded into
// the accumulators so its latency overlaps the operand pipeline's prologue.
// Cfg = CfgDual: 128 x 64 tiles, 128 threads, two CTAs per SM (one CTA's C-tile prologue / store epilogue
// hides under the other's DMMA stream).
template <typename C>
__global__ void __launch_bounds__(C::THREADS, C::CTAS_PER_SM)
syrk_kernel(double* __restrict__ L, int64_t ld, int kb, int kd, int j0, int nc, int T)
{
    extern __shared__ __align__(16) double smem[];
    constexpr int SPLIT = LB_TILE / C::BN; // column sub-tiles per 128-block
    int idx = blockIdx.x / SPLIT, c = 0;
    const int h = blockIdx.x - idx * SPLIT;
    while (c < nc && idx >= T - j0 - c) { idx -= T - j0 - c; ++c; }
    const int j = j0 + c, i = j + idx;
    const double* A = L + (int64_t)i * LB_TILE + (int64_t)kb * LB_TILE * ld;
    const double* B = L + (int64_t)j * LB_TILE + h * C::BN + (int64_t)kb * LB_TILE * ld;
    double* Cg = L + (int64_t)i * LB_TILE + ((int64_t)j * LB_TILE + h * C::BN) * ld;
    lbg::Acc<C> acc;
    lbg::load_acc<C>(acc, Cg, ld);
    lbg::mainloop<C, false, false, true>(acc, A, ld, B, ld, kd * LB_TILE, smem);
    lbg::store_acc<C>(acc, Cg, ld);
}

using SyrkCfg = lbg::CfgDual;
constexpr int SYRK_SPLIT = LB_TILE / SyrkCfg::BN;

LbOncePerDevice g_attr_once;
int set_attrs()
{
    if (!g_attr_once.need()) return LB_OK;
    LB_CUDA(cudaFuncSetAttribute(potf2_inv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)POTF2_SMEM));
    LB_CUDA(cudaFuncSetAttribute(trsm_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbg::CfgWide::PIPE_BYTES));
    LB_CUDA(cudaFuncSetAttribute(syrk_kernel<SyrkCfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SyrkCfg::PIPE_BYTES));
    return LB_OK;
}

} // namespace

// debug: cycle stamps of the phases of one panel factorisation (thread 0): start, loaded, [jb=0: factored,
// inverted, panel solved], all sub-blocks done, inverse assembled, written back
int lb_debug_potf2_clocks(lb_gp* h, int k, long long* out_host, int n)
{
    int rc = set_attrs();
    if (rc) return rc;
    long long* d = nullptr;
    LB_CUDA(cudaMalloc(&d, sizeof(long long) * 16));
    LB_CUDA(cudaMemset(d, 0, sizeof(long long) * 16));
    potf2_inv_kernel<<<1, 256, POTF2_SMEM, h->stream>>>(h->dL, h->Np, k, h->dInvD, h->dInfo, 1, d);
    LB_CUDA(cudaStreamSynchronize(h->stream));
    LB_CUDA(cudaMemcpy(out_host, d, sizeof(long long) * (n < 16 ? n : 16), cudaMemcpyDeviceToHost));
    cudaFree(d);
    return LB_OK;
}

int lb_launch_potf2_block(lb_gp* h, int k, int do_factor)
{
    int rc = set_attrs();
    if (rc) return rc;
    potf2_inv_kernel<<<1, 256, POTF2_SMEM, h->stream>>>(h->dL, h->Np, k, h->dInvD, h->dInfo, do_factor);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

static inline int syrk_tiles(int T, int j0, int nc)
{
    int n = 0;
    for (int c = 0; c < nc; ++c) n += T - j0 - c;
    return n;
}

// Right-looking factorisation with look-ahead, panels in QUADS of 128-column block columns (two pairs):
//   side stream : pair(k)  = potf2(k) trsm(k) syrk[k -> col k+1] potf2(k+1) trsm(k+1)
//                 a_in     = K=256 update of block columns k+2, k+3 with pair(k)            (inside the quad)
//                 pair(k+2)
//   main stream : a(q)     = K=512 update of the NEXT quad's four block columns with all four panels of this quad
//                 b(q)     = K=512 update of everything right of them
// quad(q+1) only needs a(q), so the latency-bound panel chain runs under b(q).  K=512 instead of the K=256 of round 1: every
// trailing tile is loaded / stored half as often per flop (the C-tile prologue and store epilogue are what keeps a short-K GEMM
// below the long-K kernels of this library: 0.76-0.84 against 0.90-0.92).  A tile's accumulator runs through the same sequence
// of DMMAs as with two K=256 passes (the store / load in between does not round), so the factor is bit-identical to the
// pair-wise distributed factorisation below (tests/test_gpu_dist_fit.py, tests/test_gpu_multirank.py).
// LB_POTRF_QUAD=0 restores the pair scheme.
static int launch_pair_panel(lb_gp* h, cudaStream_t side, int k, int T, int64_t ld)
{
    {
        LbProfScope ps(h, side, LB_PC_POTF2);
        potf2_inv_kernel<<<1, 256, POTF2_SMEM, side>>>(h->dL, ld, k, h->dInvD, h->dInfo, 1);
    }
    h->launches++;
    if (k + 1 < T) {
        {
            LbProfScope ps(h, side, LB_PC_TRSM_PANEL);
            trsm_panel_kernel<<<T - k - 1, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, side>>>(h->dL, ld, k, h->dInvD);
        }
        {
            LbProfScope ps(h, side, LB_PC_SYRK_COL);
            syrk_kernel<SyrkCfg><<<(T - k - 1) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, side>>>(h->dL, ld, k, 1, k + 1, 1, T);
        }
        {
            LbProfScope ps(h, side, LB_PC_POTF2);
            potf2_inv_kernel<<<1, 256, POTF2_SMEM, side>>>(h->dL, ld, k + 1, h->dInvD, h->dInfo, 1);
        }
        h->launches += 3;
        if (k + 2 < T) {
            LbProfScope ps(h, side, LB_PC_TRSM_PANEL);
            trsm_panel_kernel<<<T - k - 2, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, side>>>(h->dL, ld, k + 1, h->dInvD);
            h->launches++;
        }
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

static int launch_potrf_quads(lb_gp* h)
{
    const int T = (int)(h->Np / LB_TILE);
    const int64_t ld = h->Np;
    cudaStream_t main = h->stream, side = h->side ? h->side : h->stream;
    LB_CUDA(cudaMemsetAsync(h->dInfo, 0, 2 * sizeof(int), main));
    if (side != main) {
        LB_CUDA(cudaEventRecord(h->ev[0], main)); // inputs (K) ready
        LB_CUDA(cudaStreamWaitEvent(side, h->ev[0], 0));
    }
    int rc, q = 0;
    for (int k = 0; k < T; k += 4, ++q) {
        // ---- quad(q) on the side stream ----
        if ((rc = launch_pair_panel(h, side, k, T, ld))) return rc;
        if (k + 2 < T) {
            const int nc2 = (T - (k + 2) < 2) ? (T - (k + 2)) : 2;
            {
                LbProfScope ps(h, side, LB_PC_SYRK_COL);
                syrk_kernel<SyrkCfg><<<syrk_tiles(T, k + 2, nc2) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, side>>>(h->dL, ld, k, 2, k + 2, nc2, T);
            }
            h->launches++;
            if ((rc = launch_pair_panel(h, side, k + 2, T, ld))) return rc;
        }
        if (k + 4 >= T) break;
        if (side != main) {
            LB_CUDA(cudaEventRecord(h->ev[1 + (q & 1)], side));
            LB_CUDA(cudaStreamWaitEvent(main, h->ev[1 + (q & 1)], 0));
        }
        // ---- a(q): the next quad's block columns, K = 512 ----
        const int j0 = k + 4;
        const int nca = (T - j0 < 4) ? (T - j0) : 4;
        {
            LbProfScope ps(h, main, LB_PC_SYRK);
            syrk_kernel<SyrkCfg><<<syrk_tiles(T, j0, nca) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, main>>>(h->dL, ld, k, 4, j0, nca, T);
        }
        h->launches++;
        if (side != main) {
            LB_CUDA(cudaEventRecord(h->ev[3 + (q & 1)], main));
            LB_CUDA(cudaStreamWaitEvent(side, h->ev[3 + (q & 1)], 0));
        }
        // ---- b(q): the rest of the trailing matrix, K = 512 ----
        const int ncb = T - j0 - nca;
        if (ncb > 0) {
            LbProfScope ps(h, main, LB_PC_SYRK);
            syrk_kernel<SyrkCfg><<<syrk_tiles(T, j0 + nca, ncb) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, main>>>(h->dL, ld, k, 4, j0 + nca, ncb, T);
            h->launches++;
        }
    }
    if (side != main) { // join
        LB_CUDA(cudaEventRecord(h->ev[5], side));
        LB_CUDA(cudaStreamWaitEvent(main, h->ev[5], 0));
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Pair scheme of round 1 (K = 256 trailing updates), kept behind LB_POTRF_QUAD=0:
//   side stream : panel(p)  = potf2(k) trsm(k) syrk[k -> col k+1] potf2(k+1) trsm(k+1)
//   main stream : a(p)      = K=256 update of the next pair's two block columns (k+2, k+3)
//                 b(p)      = K=256 update of everything right of them
// panel(p+1) only needs a(p), so the latency-bound panel work runs under b(p).
int lb_launch_potrf(lb_gp* h)
{
    int rc = set_attrs();
    if (rc) return rc;
    static int quad = -1;
    if (quad < 0) { const char* e = getenv("LB_POTRF_QUAD"); quad = (e && atoi(e) == 0) ? 0 : 1; }
    if (quad) return launch_potrf_quads(h);
    const int T = (int)(h->Np / LB_TILE);
    const int64_t ld = h->Np;
    cudaStream_t main = h->stream, side = h->side ? h->side : h->stream;
    // b(p) is split at a FIXED block column cstar into a left group (main stream) and a right group (second, normal-priority
    // stream): a tile never changes group, so each group's stream order carries its tile dependencies, and the tail of one
    // group's launch (partial last wave, plus SMs handed to the side-stream panel kernels) is filled by the other group's CTAs.
    // Here the side-stream panel kernels already fill most of the tails, and the per-class launch timers would double count
    // concurrent launches - so it is an experiment, OFF unless LB_POTRF_SPLIT=1.
    static int split_on = -1;
    if (split_on < 0) { const char* e = getenv("LB_POTRF_SPLIT"); split_on = (e && atoi(e) != 0) ? 1 : 0; }
    cudaStream_t second = main;
    if (split_on && T >= 24 && side != main) {
        if (!h->aux && cudaStreamCreateWithFlags(&h->aux, cudaStreamNonBlocking) != cudaSuccess) h->aux = nullptr;
        if (h->aux) second = h->aux;
    }
    const int cstar = (second != main) ? (((int)(0.38 * T)) & ~1) : T; // even: a pair (k, k + 1) never straddles the boundary // left group: columns < cstar (long columns), right: >= cstar; ~equal tile counts at the start
    LB_CUDA(cudaMemsetAsync(h->dInfo, 0, 2 * sizeof(int), main));
    if (side != main) {
        LB_CUDA(cudaEventRecord(h->ev[0], main)); // inputs (K) ready
        LB_CUDA(cudaStreamWaitEvent(side, h->ev[0], 0));
        if (second != main) LB_CUDA(cudaStreamWaitEvent(second, h->ev[0], 0));
    }
    int p = 0;
    for (int k = 0; k < T; k += 2, ++p) {
        const bool pair = (k + 1 < T);
        // ---- panel(p) on the side stream ----
        {
            LbProfScope ps(h, side, LB_PC_POTF2);
            potf2_inv_kernel<<<1, 256, POTF2_SMEM, side>>>(h->dL, ld, k, h->dInvD, h->dInfo, 1);
        }
        h->launches++;
        if (pair) {
            {
                LbProfScope ps(h, side, LB_PC_TRSM_PANEL);
                trsm_panel_kernel<<<T - k - 1, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, side>>>(h->dL, ld, k, h->dInvD);
            }
            {
                LbProfScope ps(h, side, LB_PC_SYRK_COL);
                syrk_kernel<SyrkCfg><<<(T - k - 1) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, side>>>(h->dL, ld, k, 1, k + 1, 1, T);
            }
            {
                LbProfScope ps(h, side, LB_PC_POTF2);
                potf2_inv_kernel<<<1, 256, POTF2_SMEM, side>>>(h->dL, ld, k + 1, h->dInvD, h->dInfo, 1);
            }
            h->launches += 3;
            if (k + 2 < T) {
                LbProfScope ps(h, side, LB_PC_TRSM_PANEL);
                trsm_panel_kernel<<<T - k - 2, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, side>>>(h->dL, ld, k + 1, h->dInvD);
                h->launches++;
            }
        }
        if (k + 2 >= T) break;
        if (side != main) {
            LB_CUDA(cudaEventRecord(h->ev[1 + (p & 1)], side));
            LB_CUDA(cudaStreamWaitEvent(main, h->ev[1 + (p & 1)], 0));
        }
        // ---- a(p): the next pair's block columns ----
        const int j0 = k + 2;
        const int nca = (T - j0 < 2) ? (T - j0) : 2;
        // once the factorisation has passed cstar the look-ahead columns belong to the right group: hand over to the second stream
        // for good (its earlier updates of these tiles precede in stream order; main has nothing left)
        cudaStream_t sa = (second != main && j0 >= cstar) ? second : main;
        if (sa != main && side != main) LB_CUDA(cudaStreamWaitEvent(sa, h->ev[1 + (p & 1)], 0));
        {
            LbProfScope ps(h, sa, LB_PC_SYRK);
            syrk_kernel<SyrkCfg><<<syrk_tiles(T, j0, nca) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, sa>>>(h->dL, ld, k, 2, j0, nca, T);
        }
        h->launches++;
        if (side != main) {
            LB_CUDA(cudaEventRecord(h->ev[3 + (p & 1)], sa));
            LB_CUDA(cudaStreamWaitEvent(side, h->ev[3 + (p & 1)], 0));
        }
        // ---- b(p): the rest of the trailing matrix ----
        const int jb = j0 + nca;
        if (sa == main && second != main) {
            const int left_end = cstar < jb ? jb : cstar; // columns [jb, left_end) on main, [left_end, T) on the second stream
            if (left_end > jb) {
                LbProfScope ps(h, main, LB_PC_SYRK);
                syrk_kernel<SyrkCfg><<<syrk_tiles(T, jb, left_end - jb) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, main>>>(h->dL, ld, k, 2, jb, left_end - jb, T);
                h->launches++;
            }
            if (T - left_end > 0) {
                if (side != main) LB_CUDA(cudaStreamWaitEvent(second, h->ev[1 + (p & 1)], 0)); // the panel it multiplies with
                LbProfScope ps(h, second, LB_PC_SYRK);
                syrk_kernel<SyrkCfg><<<syrk_tiles(T, left_end, T - left_end) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, second>>>(h->dL, ld, k, 2, left_end, T - left_end, T);
                h->launches++;
            }
        }
        else {
            const int ncb = T - jb;
            if (ncb > 0) {
                LbProfScope ps(h, sa, LB_PC_SYRK);
                syrk_kernel<SyrkCfg><<<syrk_tiles(T, jb, ncb) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, sa>>>(h->dL, ld, k, 2, jb, ncb, T);
                h->launches++;
            }
        }
    }
    if (side != main) { // join
        LB_CUDA(cudaEventRecord(h->ev[5], side));
        LB_CUDA(cudaStreamWaitEvent(main, h->ev[5], 0));
    }
    if (second != main) {
        LB_CUDA(cudaEventRecord(h->ev[6], second));
        LB_CUDA(cudaStreamWaitEvent(main, h->ev[6], 0));
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// =====================================================================================================================
// Multi-GPU Cholesky (BASELINE.json config 5, SURVEY.md §8e "stretch"): building blocks for a 1-D block-cyclic
// right-looking factorisation over 256-column panels ("pairs" of 128-blocks, the same pair structure as lb_launch_potrf).
// Pair p (global 128-block columns 2p, 2p+1) lives on rank p mod G; a rank stores its pairs side by side, full height:
//   local 128-block column l  <->  global block column  j(l) = 2 * (G * (l / 2) + rank) + (l & 1)
// One step = owner factors its pair (potf2, trsm, K=128 column update, potf2, trsm: the kernels above on its local
// columns), packs the rows below the pair into a contiguous panel, the host broadcasts the panel (NCCL, the only
// exchange step of the path), and every rank applies the K = 256 update to the local columns right of the pair.  The host
// side (limbo_b200/dist_chol.py) owns the streams, the double-buffered panel and the look-ahead.
// =====================================================================================================================
namespace {

__device__ __forceinline__ int dchol_global_block(int l, int rank, int G) { return 2 * (G * (l >> 1) + rank) + (l & 1); }

// K[:, local columns] for this rank: dLoc[i + c*ld], c = local column; noise + 1e-8 on the diagonal (kernel.hpp:83);
// identity in the padding (i or global column >= N).
__global__ void __launch_bounds__(256)
dchol_build_kernel(const double* __restrict__ Xs, int64_t xs_ld, int64_t N, int64_t Nd, KernParams kp, int rank, int G, int64_t ncols_local,
    double* __restrict__ dLoc)
{
    const int64_t i = (int64_t)blockIdx.y * 256 + threadIdx.x; // columns on grid.x (no 65535 limit), 256-row slabs on grid.y
    const int64_t c = blockIdx.x;
    if (i >= Nd || c >= ncols_local) return;
    const int64_t j = (int64_t)dchol_global_block((int)(c / LB_TILE), rank, G) * LB_TILE + (c % LB_TILE);
    double v;
    if (i >= N || j >= N) v = (i == j) ? 1.0 : 0.0;
    else {
        double z = 0.0;
        for (int d = 0; d < kp.D; ++d) {
            const double q = Xs[(int64_t)d * xs_ld + i] - Xs[(int64_t)d * xs_ld + j];
            z = fma(q, q, z);
        }
        v = lb_kernel_from_z(kp.id, z, kp) + ((i == j) ? kp.noise + 1e-8 : 0.0);
    }
    dLoc[i + c * Nd] = v;
}

// panel[r + c*ldp] = cols[(row0 + r) + c*ld], r < ldp, c < 256
__global__ void __launch_bounds__(256)
dchol_pack_kernel(const double* __restrict__ cols, int64_t ld, int64_t row0, double* __restrict__ panel, int64_t ldp)
{
    const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int c = blockIdx.y;
    if (r < ldp) panel[r + c * ldp] = cols[row0 + r + c * ld];
}

// C[i, j(l)] -= P[i,:] P[j(l),:]^T for the local block columns l in [l0, l1) whose global index j(l) > kpair+1, i >= j(l).
// P is the packed panel: row block b of the global matrix sits at panel row (b - (kpair + 2)) * 128, ld = ldp, K = 256.
template <typename C>
__global__ void __launch_bounds__(C::THREADS, C::CTAS_PER_SM)
dchol_update_kernel(double* __restrict__ Lloc, int64_t ld, const double* __restrict__ P, int64_t ldp, int kpair, int l0, int l1, int rank,
    int G, int T)
{
    extern __shared__ __align__(16) double smem[];
    constexpr int SPLIT = LB_TILE / C::BN;
    int idx = blockIdx.x / SPLIT;
    const int h = blockIdx.x - idx * SPLIT;
    int l = l0;
    for (; l < l1; ++l) {
        const int nt = T - dchol_global_block(l, rank, G);
        if (idx < nt) break;
        idx -= nt;
    }
    if (l >= l1) return;
    const int j = dchol_global_block(l, rank, G), i = j + idx;
    const int b0 = kpair + 2;
    const double* A = P + (int64_t)(i - b0) * LB_TILE;
    const double* B = P + (int64_t)(j - b0) * LB_TILE + h * C::BN;
    double* Cg = Lloc + (int64_t)i * LB_TILE + ((int64_t)l * LB_TILE + h * C::BN) * ld;
    lbg::Acc<C> acc;
    lbg::load_acc<C>(acc, Cg, ld);
    lbg::mainloop<C, false, false, true>(acc, A, ldp, B, ldp, 2 * LB_TILE, smem);
    lbg::store_acc<C>(acc, Cg, ld);
}

// zero the strictly upper part of the local columns (matrixL has a zero upper triangle, gp.hpp:565) and return
// sum log L_jj over the local columns with global index < N in out[0]
__global__ void __launch_bounds__(256)
dchol_finish_kernel(double* __restrict__ Lloc, int64_t ld, int64_t N, int rank, int G, int64_t ncols_local, double* __restrict__ part)
{
    __shared__ double red[8];
    double s = 0.0;
    for (int64_t c = blockIdx.x; c < ncols_local; c += gridDim.x) {
        const int64_t j = (int64_t)dchol_global_block((int)(c / LB_TILE), rank, G) * LB_TILE + (c % LB_TILE);
        double* col = Lloc + c * ld;
        for (int64_t i = threadIdx.x; i < j && i < ld; i += 256) col[i] = 0.0;
        if (threadIdx.x == 0 && j < N) s += log(col[j]);
    }
    s = lb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        part[blockIdx.x] = t;
    }
}
__global__ void dchol_sum_kernel(const double* __restrict__ part, int n, double* __restrict__ out)
{
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += part[i];
    *out = s;
}

LbOncePerDevice g_dchol_once;

} // namespace

extern "C" {

// K columns of this rank.  h supplies the staged samples and the kernel (lb_set_data + lb_set_kernel, no fit needed);
// Nd = padded order (multiple of 256), dLoc = Nd x ncols_local, column-major.
int lb_dchol_build(lb_gp* h, int64_t Nd, int rank, int G, int64_t ncols_local, double* dLoc)
{
    if (!h || !dLoc || Nd % (2 * LB_TILE) || !h->kernel_set || h->N <= 0) return LB_ERR_ARG;
    int rc = lb_launch_scale_x(h);
    if (rc) return rc;
    dim3 grid((unsigned)ncols_local, (unsigned)((Nd + 255) / 256));
    dchol_build_kernel<<<grid, 256, 0, h->stream>>>(h->dXs, h->Np, h->N, Nd, h->kp, rank, G, ncols_local, dLoc);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Owner step for pair `kpair` (global 128-block index of its first column, even): dCols = the pair's 256 local columns
// (Nd x 256, ld = Nd).  Factors them in place and packs rows [(kpair+2)*128, Nd) into dPanel (ld = Nd - (kpair+2)*128).
// dInvD: 2 x 128 x 128 scratch; dInfo: 2 ints (first failing pivot, 1-based local to the pair's diagonal block, or 0).
int lb_dchol_panel(lb_gp* h, double* dCols, int64_t Nd, int kpair, double* dInvD, int* dInfo, double* dPanel)
{
    if (!h || !dCols || !dInvD || !dInfo) return LB_ERR_ARG;
    int rc = set_attrs();
    if (rc) return rc;
    const int T = (int)(Nd / LB_TILE);
    cudaStream_t st = h->stream;
    // the kernels above address block (i, k) as L + i*128 + k*128*ld: shift the bases so that block column kpair is dCols
    double* Lb = dCols - (int64_t)kpair * LB_TILE * Nd;
    double* Ib = dInvD - (int64_t)kpair * LB_TILE * LB_TILE;
    potf2_inv_kernel<<<1, 256, POTF2_SMEM, st>>>(Lb, Nd, kpair, Ib, dInfo, 1);
    trsm_panel_kernel<<<T - kpair - 1, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, st>>>(Lb, Nd, kpair, Ib);
    syrk_kernel<SyrkCfg><<<(T - kpair - 1) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, st>>>(Lb, Nd, kpair, 1, kpair + 1, 1, T);
    potf2_inv_kernel<<<1, 256, POTF2_SMEM, st>>>(Lb, Nd, kpair + 1, Ib, dInfo, 1);
    h->launches += 4;
    if (kpair + 2 < T) {
        trsm_panel_kernel<<<T - kpair - 2, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, st>>>(Lb, Nd, kpair + 1, Ib);
        const int64_t ldp = Nd - (int64_t)(kpair + 2) * LB_TILE;
        dim3 grid((unsigned)((ldp + 255) / 256), 2 * LB_TILE);
        dchol_pack_kernel<<<grid, 256, 0, st>>>(dCols, Nd, (int64_t)(kpair + 2) * LB_TILE, dPanel, ldp);
        h->launches += 2;
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Trailing update of the local block columns [l0, l1) with the packed panel of pair kpair (on h's stream).
int lb_dchol_update(lb_gp* h, double* dLoc, int64_t Nd, const double* dPanel, int kpair, int l0, int l1, int rank, int G)
{
    if (!h || !dLoc || !dPanel) return LB_ERR_ARG;
    if (g_dchol_once.need()) {
        LB_CUDA(cudaFuncSetAttribute(dchol_update_kernel<SyrkCfg>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SyrkCfg::PIPE_BYTES));
    }
    const int T = (int)(Nd / LB_TILE);
    int64_t tiles = 0;
    int lfirst = l1;
    for (int l = l0; l < l1; ++l) {
        const int j = 2 * (G * (l >> 1) + rank) + (l & 1);
        if (j <= kpair + 1) continue; // left of / inside the panel: nothing to update
        if (l < lfirst) lfirst = l;
        tiles += T - j;
    }
    if (tiles == 0) return LB_OK;
    const int64_t ldp = Nd - (int64_t)(kpair + 2) * LB_TILE;
    LbProfScope ps(h, h->stream, LB_PC_SYRK);
    dchol_update_kernel<SyrkCfg><<<(unsigned)(tiles * SYRK_SPLIT), SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, h->stream>>>(dLoc, Nd, dPanel, ldp, kpair,
        lfirst, l1, rank, G, T);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// zero the upper triangle of the local columns; *dLogdetPart (device) = sum over local columns of log L_jj
int lb_dchol_finish(lb_gp* h, double* dLoc, int64_t Nd, int64_t N, int rank, int G, int64_t ncols_local, double* dLogdetPart)
{
    if (!h || !dLoc || !dLogdetPart) return LB_ERR_ARG;
    int rc = lb_ensure_scratch(h, sizeof(double) * 1024);
    if (rc) return rc;
    dchol_finish_kernel<<<1024, 256, 0, h->stream>>>(dLoc, Nd, N, rank, G, ncols_local, h->dScratch);
    dchol_sum_kernel<<<1, 1, 0, h->stream>>>(h->dScratch, 1024, dLogdetPart);
    h->launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

} // extern "C"
