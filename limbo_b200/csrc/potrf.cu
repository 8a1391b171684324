// limbo_b200/csrc/potrf.cu — blocked Cholesky with deferred trailing updates, trailing
// update on fp64 tensor cores (DMMA).
//
// Replaces `_matrixL = Eigen::LLT<Eigen::MatrixXd>(_kernel).matrixL()`
// (model/gp.hpp:565).  Per 128-column panel k:
//   1. potf2_inv_kernel : factor the 128x128 diagonal block in one CTA
//                         (32x32 sub-blocks in registers via warp shuffles) and
//                         form its inverse (kept in invD for every later
//                         triangular solve);
//   2. trsm_panel_kernel: L[i,k] = A[i,k] * inv(L[k,k])^T   (DMMA GEMM)
//   3. syrk_kernel      : A[i,j] -= L[i,k] * L[j,k]^T, k < j <= i (DMMA GEMM), several
//                         panels per pass (potrf_plan below decides which and when)
// A non-positive pivot is reported LAPACK-style through info (the reference
// never checks Eigen's info(), SURVEY.md §5).
#include "gemm.cuh"

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

// The block columns of one trailing-update pass: column j0 + c takes the panel block columns [kb[c], kend), c < nc.
constexpr int SYRK_MAX_COLS = 64;
struct SyrkCols {
    int j0, nc, kend;
    int kb[SYRK_MAX_COLS];
};

// Trailing update of block column j = j0 + c with its panel block columns [kb[c], kend):
//   A[i,j] -= L[i, kb[c]:kend] L[j, kb[c]:kend]^T   for c < nc, j <= i < T
// C is preloaded into the accumulators so its latency overlaps the operand pipeline's prologue.  The grid walks the columns
// from the right: the planner never gives a column a later kb than the columns left of it, so the longest-K tiles start first
// and the short ones fill the last wave.  Cfg = CfgDual: 128 x 64 tiles, 128 threads, two CTAs per SM (one CTA's C-tile
// prologue / store epilogue hides under the other's DMMA stream).
template <typename C>
__global__ void __launch_bounds__(C::THREADS, C::CTAS_PER_SM)
syrk_kernel(double* __restrict__ L, int64_t ld, const __grid_constant__ SyrkCols cols, int T)
{
    extern __shared__ __align__(16) double smem[];
    constexpr int SPLIT = LB_TILE / C::BN; // column sub-tiles per 128-block
    int idx = blockIdx.x / SPLIT, c = cols.nc - 1;
    const int h = blockIdx.x - idx * SPLIT;
    while (c > 0 && idx >= T - cols.j0 - c) { idx -= T - cols.j0 - c; --c; }
    const int j = cols.j0 + c, i = j + idx, kb = cols.kb[c];
    const double* A = L + (int64_t)i * LB_TILE + (int64_t)kb * LB_TILE * ld;
    const double* B = L + (int64_t)j * LB_TILE + h * C::BN + (int64_t)kb * LB_TILE * ld;
    double* Cg = L + (int64_t)i * LB_TILE + ((int64_t)j * LB_TILE + h * C::BN) * ld;
    lbg::Acc<C> acc;
    lbg::load_acc<C>(acc, Cg, ld);
    lbg::mainloop<C, false, false, true>(acc, A, ld, B, ld, (cols.kend - kb) * LB_TILE, smem);
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
    potf2_inv_kernel<<<1, 256, POTF2_SMEM, h->stream>>>(h->dL, h->Np, k, h->dInvD, h->dInfo.get(), 1, d);
    LB_CUDA(cudaStreamSynchronize(h->stream));
    LB_CUDA(cudaMemcpy(out_host, d, sizeof(long long) * (n < 16 ? n : 16), cudaMemcpyDeviceToHost));
    cudaFree(d);
    return LB_OK;
}

int lb_launch_potf2_block(lb_gp* h, int k, int do_factor)
{
    int rc = set_attrs();
    if (rc) return rc;
    potf2_inv_kernel<<<1, 256, POTF2_SMEM, h->stream>>>(h->dL, h->Np, k, h->dInvD, h->dInfo.get(), do_factor);
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

static void launch_syrk(cudaStream_t st, double* L, int64_t ld, const SyrkCols& cols, int T)
{
    syrk_kernel<SyrkCfg><<<syrk_tiles(T, cols.j0, cols.nc) * SYRK_SPLIT, SyrkCfg::THREADS, SyrkCfg::PIPE_BYTES, st>>>(L, ld, cols, T);
}

// syrk_kernel over the block columns [j0, j0 + nc), each with the panel block columns [kb, kb + kd)
static void launch_syrk(cudaStream_t st, double* L, int64_t ld, int kb, int kd, int j0, int nc, int T)
{
    SyrkCols cols{j0, nc, kb + kd, {}};
    for (int c = 0; c < nc; ++c) cols.kb[c] = kb;
    launch_syrk(st, L, ld, cols, T);
}

// Pair panel (k, k + 1): potf2(k) trsm(k) syrk[k -> col k+1] (K = 128) potf2(k+1), and trsm(k+1) when k + 2 < T.  L, invD and
// info are the bases from which the kernels address block (i, k) and the diagonal-block inverse k.
static int launch_pair_panel(lb_gp* h, cudaStream_t st, double* L, double* invD, int* info, int64_t ld, int k, int T)
{
    {
        LbProfScope ps(h, st, LB_PC_POTF2);
        potf2_inv_kernel<<<1, 256, POTF2_SMEM, st>>>(L, ld, k, invD, info, 1);
    }
    h->launches++;
    if (k + 1 < T) {
        {
            LbProfScope ps(h, st, LB_PC_TRSM_PANEL);
            trsm_panel_kernel<<<T - k - 1, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, st>>>(L, ld, k, invD);
        }
        {
            LbProfScope ps(h, st, LB_PC_SYRK_COL);
            launch_syrk(st, L, ld, k, 1, k + 1, 1, T);
        }
        {
            LbProfScope ps(h, st, LB_PC_POTF2);
            potf2_inv_kernel<<<1, 256, POTF2_SMEM, st>>>(L, ld, k + 1, invD, info, 1);
        }
        h->launches += 3;
        if (k + 2 < T) {
            LbProfScope ps(h, st, LB_PC_TRSM_PANEL);
            trsm_panel_kernel<<<T - k - 2, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, st>>>(L, ld, k + 1, invD);
            h->launches++;
        }
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Blocked factorisation with look-ahead, panels in QUADS of four 128-column block columns (two pairs), and trailing updates
// deferred into long-K passes.  applied[j] counts the panels already subtracted from block column j; every update of column j
// takes the panels [applied[j], kend) in one pass, so each tile's accumulator runs through the same ascending sequence of DMMAs
// whatever the passes are (a store and a reload in between do not round), and the factor is bit-identical to the right-looking
// and the pair-wise distributed factorisations (tests/test_gpu_dist_fit.py, tests/test_gpu_multirank.py).  Per quad q (k = 4q):
//   side stream : pair(k)  = potf2(k) trsm(k) syrk[k -> col k+1] potf2(k+1) trsm(k+1)
//                 K = 256 update of block columns k+2, k+3 with pair(k)                    (inside the quad)
//                 pair(k+2)
//   main stream : a(q)     = K = 512 update of the next quad's four block columns with this quad's panels
//                 LL(q)    = quad q+2's block columns with every panel not yet applied to them (up to k+4), then further
//                            columns to the right, each with its own [applied, k+4), until the pass holds POTRF_FILL_WAVES
//                            waves of CTAs
// quad q+1's chain only needs a(q), so it runs under LL(q).  A column is loaded and stored once per pass instead of once per
// quad, and most trailing flops run at K in the thousands.  The fill bound keeps the late passes, whose deferred columns hold
// few tiles of long K, from ending in a sliver wave (DESIGN.md §4.2).
namespace {

constexpr int POTRF_FILL_WAVES = 8;

enum { PLAN_MAIN = 0, PLAN_SIDE = 1 };
enum { POP_PAIR = 0, POP_UPDATE, POP_RECORD, POP_WAIT };

struct PotrfOp {
    int op;        // POP_*
    int stream;    // PLAN_MAIN / PLAN_SIDE
    int arg;       // POP_PAIR: first block column of the pair; POP_RECORD / POP_WAIT: index into lb_gp::ev
    SyrkCols cols; // POP_UPDATE
};

// The factorisation of a T x T block matrix as one list of operations in issue order, for `sms` SMs.  Streams order their own
// operations; POP_WAIT orders its stream behind the latest POP_RECORD of the same event issued before it.
std::vector<PotrfOp> potrf_plan(int T, int sms)
{
    std::vector<PotrfOp> ops;
    std::vector<int> applied(T > 0 ? T : 0, 0);
    const int64_t fill = (int64_t)POTRF_FILL_WAVES * sms * SyrkCfg::CTAS_PER_SM;
    auto sync = [&](int from, int to, int ev) {
        ops.push_back({POP_RECORD, from, ev, {}});
        ops.push_back({POP_WAIT, to, ev, {}});
    };
    auto pair = [&](int k) {
        ops.push_back({POP_PAIR, PLAN_SIDE, k, {}});
        if (k + 1 < T) applied[k + 1] = k + 1;
    };
    // the columns [j0, j1) up to panel kend, then more columns while the pass is short of `want` CTAs
    auto update = [&](int st, int j0, int j1, int kend, int64_t want) {
        PotrfOp o{POP_UPDATE, st, 0, {j0, 0, kend, {}}};
        int64_t ctas = 0;
        for (int j = j0; j < T && o.cols.nc < SYRK_MAX_COLS && (j < j1 || ctas < want); ++j) {
            o.cols.kb[o.cols.nc++] = applied[j];
            applied[j] = kend;
            ctas += (int64_t)(T - j) * SYRK_SPLIT;
        }
        if (o.cols.nc > 0) ops.push_back(o);
    };
    sync(PLAN_MAIN, PLAN_SIDE, 0); // inputs (K) ready
    for (int k = 0, q = 0; k < T; k += 4, ++q) {
        pair(k);
        if (k + 2 < T) {
            update(PLAN_SIDE, k + 2, k + 4, k + 2, 0);
            pair(k + 2);
        }
        if (k + 4 >= T) break;
        sync(PLAN_SIDE, PLAN_MAIN, 1 + (q & 1));
        update(PLAN_MAIN, k + 4, k + 8, k + 4, 0); // a(q)
        sync(PLAN_MAIN, PLAN_SIDE, 3 + (q & 1));
        update(PLAN_MAIN, k + 8, k + 12, k + 4, fill); // LL(q)
    }
    sync(PLAN_SIDE, PLAN_MAIN, 5); // join
    return ops;
}

} // namespace

int lb_launch_potrf(lb_gp* h)
{
    int rc = set_attrs();
    if (rc) return rc;
    const int T = (int)(h->Np / LB_TILE);
    const int64_t ld = h->Np;
    cudaStream_t main = h->stream, side = h->side ? h->side : h->stream;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device);
    LB_CUDA(cudaMemsetAsync(h->dInfo.get(), 0, 2 * sizeof(int), main));
    for (const PotrfOp& o : potrf_plan(T, sms)) {
        cudaStream_t st = o.stream == PLAN_SIDE ? side : main;
        switch (o.op) {
        case POP_PAIR:
            if ((rc = launch_pair_panel(h, st, h->dL, h->dInvD, h->dInfo.get(), ld, o.arg, T))) return rc;
            break;
        case POP_UPDATE: {
            LbProfScope ps(h, st, o.stream == PLAN_SIDE ? LB_PC_SYRK_COL : LB_PC_SYRK);
            launch_syrk(st, h->dL, ld, o.cols, T);
            h->launches++;
            break;
        }
        case POP_RECORD:
            if (side != main) LB_CUDA(cudaEventRecord(h->ev[o.arg], st));
            break;
        case POP_WAIT:
            if (side != main) LB_CUDA(cudaStreamWaitEvent(st, h->ev[o.arg], 0));
            break;
        }
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// The plan lb_launch_potrf walks, for host-side checks: one record of 6 + SYRK_MAX_COLS ints per operation, {op, stream, arg,
// j0, nc, kend, kb[0 .. SYRK_MAX_COLS)}, at most `cap` records written.  Returns the number of operations.
extern "C" int lb_debug_potrf_plan(int T, int sms, int* out, int cap)
{
    if (T < 1 || sms < 1) return LB_ERR_ARG;
    const std::vector<PotrfOp> ops = potrf_plan(T, sms);
    constexpr int W = 6 + SYRK_MAX_COLS;
    for (int n = 0; n < (int)ops.size() && n < cap; ++n) {
        const PotrfOp& o = ops[n];
        int* r = out + (int64_t)n * W;
        r[0] = o.op; r[1] = o.stream; r[2] = o.arg;
        r[3] = o.cols.j0; r[4] = o.cols.nc; r[5] = o.cols.kend;
        for (int c = 0; c < SYRK_MAX_COLS; ++c) r[6 + c] = o.cols.kb[c];
    }
    return (int)ops.size();
}

// =====================================================================================================================
// Multi-GPU Cholesky (BASELINE.json config 5, SURVEY.md §8e "stretch"): building blocks for a 1-D block-cyclic
// right-looking factorisation over 256-column panels ("pairs" of 128-blocks, the pairs lb_launch_potrf's quads are made of).
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
    if ((rc = launch_pair_panel(h, st, Lb, Ib, dInfo, Nd, kpair, T))) return rc;
    if (kpair + 2 < T) {
        const int64_t ldp = Nd - (int64_t)(kpair + 2) * LB_TILE;
        dim3 grid((unsigned)((ldp + 255) / 256), 2 * LB_TILE);
        dchol_pack_kernel<<<grid, 256, 0, st>>>(dCols, Nd, (int64_t)(kpair + 2) * LB_TILE, dPanel, ldp);
        h->launches++;
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
    dchol_finish_kernel<<<1024, 256, 0, h->stream>>>(dLoc, Nd, N, rank, G, ncols_local, h->dScratch.get());
    dchol_sum_kernel<<<1, 1, 0, h->stream>>>(h->dScratch.get(), 1024, dLogdetPart);
    h->launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

} // extern "C"
