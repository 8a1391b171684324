// limbo_b200/csrc/lml.cu — log marginal likelihood, K^-1 and the kernel
// hyper-parameter gradient (what model::gp::KernelLFOpt evaluates per Rprop step,
// model/gp/kernel_lf_opt.hpp:77-92).
//
//   GP::compute_log_lik             model/gp.hpp:267-282  -> loglik_kernel
//   GP::compute_inv_kernel          model/gp.hpp:254-264  -> trtri (block rows, DMMA) + lauum_kernel (DMMA)
//                                   2N^3/3 flops instead of the reference's 2N^3
//   GP::compute_kernel_grad_log_lik model/gp.hpp:285-311  -> grad_kernel: one streaming pass over the
//                                   lower tiles of K^-1, k_ij and d k_ij / d theta recomputed from X
//                                   (W = alpha alpha^T - K^-1 is never materialised)
#include "gemm.cuh"
#include "pair_tile.cuh"

namespace {

__global__ void __launch_bounds__(1024)
loglik_kernel(const double* __restrict__ L, int64_t ld, int64_t N, const double* __restrict__ Y,
    const double* __restrict__ alpha, int P, double* __restrict__ out)
{
    __shared__ double r1[32], r2[32];
    double s_log = 0.0, s_a = 0.0;
    for (int64_t i = threadIdx.x; i < N; i += 1024) {
        s_log += log(L[i + i * ld]);
        for (int p = 0; p < P; ++p) s_a = fma(Y[i + (int64_t)p * ld], alpha[i + (int64_t)p * ld], s_a);
    }
    s_log = lb_warp_sum(s_log);
    s_a = lb_warp_sum(s_a);
    if ((threadIdx.x & 31) == 0) { r1[threadIdx.x >> 5] = s_log; r2[threadIdx.x >> 5] = s_a; }
    __syncthreads();
    if (threadIdx.x < 32) {
        double v1 = lb_warp_sum(r1[threadIdx.x]);
        double v2 = lb_warp_sum(r2[threadIdx.x]);
        if (threadIdx.x == 0) {
            double logdet = 2.0 * v1; // gp.hpp:274
            out[0] = v2;
            out[1] = logdet;
            out[2] = -0.5 * v2 - 0.5 * logdet - 0.5 * (double)N * log(2.0 * M_PI); // gp.hpp:279
        }
    }
}

__global__ void set_identity_kernel(double* __restrict__ A, int64_t n)
{
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t tot = n * n;
    for (; idx < tot; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx % n, c = idx / n;
        A[idx] = (r == c) ? 1.0 : 0.0;
    }
}

// ---- recursive (divide and conquer) triangular inverse ----------------------------------
// inv [[A,0],[B,C]] = [[A^-1, 0], [-C^-1 B A^-1, C^-1]].  Level with half-size sb (in 128-blocks): the matrix is cut
// into problems of 2*sb block rows; problem q has A = X[a0:a0+sb, a0:a0+sb] and C = X[c0:c0+sb, c0:c0+sb] already
// inverted by the previous level (a0 = 2*q*sb, c0 = a0 + sb) and B = L[c0:c0+sb, a0:a0+sb].
//   step 1:  W = B * A^-1            W[i,j] = sum_{k >= j} B[i,k] Ainv[k,j]
//   step 2:  X[C rows, A cols] = -C^-1 * W   [i,j] = -sum_{k <= i} Cinv[i,k] W[k,j]
// All tiles of a level are independent (one launch per step), unlike the block-row recurrence whose j = 0
// tile serialises T^2/2 K-chunks on one SM.
__global__ void __launch_bounds__(lbg::CfgWide::THREADS, 1)
trtri_level_kernel(const double* __restrict__ L, double* __restrict__ X, double* __restrict__ W, int64_t ld, int sb, int step,
    int T)
{
    extern __shared__ __align__(16) double smem[];
    const int per = sb * sb;
    const int q = blockIdx.x / per;
    int rem = blockIdx.x - q * per;
    const int a0 = 2 * q * sb, c0 = a0 + sb;
    int nC = sb;                       // block rows available in the C part (last problem may be short)
    if (c0 >= T) return;
    if (c0 + nC > T) nC = T - c0;
    lbg::Acc<lbg::CfgWide> acc;
    acc.zero();
    if (step == 1) {
        const int j = rem / sb, i = rem - j * sb; // heavy tiles (small j) first
        if (i >= nC) return;
        // A = B[i, j..sb-1] = L[(c0+i), (a0+j)...] (outer-contiguous); Bop(k,n) = Ainv[(a0+j)+k, (a0+j)*128+n] (k-contiguous)
        lbg::mainloop<lbg::CfgWide, false, true>(acc, L + (int64_t)(c0 + i) * LB_TILE + (int64_t)(a0 + j) * LB_TILE * ld, ld,
            X + (int64_t)(a0 + j) * LB_TILE + (int64_t)(a0 + j) * LB_TILE * ld, ld, (sb - j) * LB_TILE, smem);
        lbg::store_acc<lbg::CfgWide>(acc, W + (int64_t)(c0 + i) * LB_TILE + (int64_t)(a0 + j) * LB_TILE * ld, ld);
    }
    else {
        const int ii = rem / sb, j = rem - ii * sb;
        const int i = sb - 1 - ii; // heavy tiles (large i) first
        if (i >= nC) return;
        // A = Cinv[i, 0..i] = X[(c0+i), c0...] (outer-contiguous); Bop(k,n) = W[c0*128 + k, (a0+j)*128 + n] (k-contiguous)
        lbg::mainloop<lbg::CfgWide, false, true, true>(acc, X + (int64_t)(c0 + i) * LB_TILE + (int64_t)c0 * LB_TILE * ld, ld,
            W + (int64_t)c0 * LB_TILE + (int64_t)(a0 + j) * LB_TILE * ld, ld, (i + 1) * LB_TILE, smem);
        lbg::store_acc<lbg::CfgWide>(acc, X + (int64_t)(c0 + i) * LB_TILE + (int64_t)(a0 + j) * LB_TILE * ld, ld);
    }
}

__global__ void __launch_bounds__(256)
trtri_diag_copy_kernel(const double* __restrict__ invD, double* __restrict__ X, int64_t ld)
{
    const int d = blockIdx.x;
    const double* src = invD + (int64_t)d * LB_TILE * LB_TILE;
    double* dst = X + (int64_t)d * LB_TILE + (int64_t)d * LB_TILE * ld;
    for (int idx = threadIdx.x; idx < LB_TILE * LB_TILE; idx += 256) {
        int r = idx & 127, c = idx >> 7;
        dst[r + (int64_t)c * ld] = src[idx];
    }
}

// Kinv[i,j] = sum_{k >= i} X[k,i]^T X[k,j]  for i >= j (lower tiles only)
__global__ void __launch_bounds__(lbg::CfgWide::THREADS, 1)
lauum_kernel(const double* __restrict__ X, int64_t ld, double* __restrict__ Kinv, int T)
{
    extern __shared__ __align__(16) double smem[];
    // longest K ranges (small i) first: enumerate tiles so that i ascends
    int i, j;
    tile_from_index(blockIdx.x, i, j);
    lbg::Acc<lbg::CfgWide> acc;
    acc.zero();
    const int64_t k0 = (int64_t)i * LB_TILE;
    lbg::mainloop<lbg::CfgWide, true, true>(acc, X + k0 + (int64_t)i * LB_TILE * ld, ld, X + k0 + (int64_t)j * LB_TILE * ld, ld,
        (T - i) * LB_TILE, smem);
    double* C = Kinv + (int64_t)i * LB_TILE + (int64_t)j * LB_TILE * ld;
    lbg::store_acc<lbg::CfgWide>(acc, C, ld);
}

// mirror lower -> upper (export only)
__global__ void symmetrize_kernel(double* __restrict__ A, int64_t n)
{
    __shared__ double tile[32][33];
    int bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    int64_t r = (int64_t)bi * 32 + threadIdx.x, c0 = (int64_t)bj * 32;
    for (int cc = threadIdx.y; cc < 32; cc += 8) tile[cc][threadIdx.x] = A[r + (c0 + cc) * n];
    __syncthreads();
    // write A[c0+x, bi*32 + y] = tile[x][y]  (upper counterpart)
    for (int cc = threadIdx.y; cc < 32; cc += 8) {
        int64_t rr = c0 + threadIdx.x, col = (int64_t)bi * 32 + cc;
        if (rr < col) A[rr + col * n] = tile[threadIdx.x][cc];
    }
}

// grad partials: part[tile][q], q < nh.
//   sum_{i>=j} w_ij * dK_ij/dtheta_q * (1/2 if i==j)        gp.hpp:299-308
//   w = alpha alpha^T - K^-1                                  gp.hpp:293-296
// One pass over the lower tiles of K^-1 (HBM floor 4 N^2 bytes).  The kernel id and the edge handling
// are template parameters (interior tiles carry no predicates), alpha_i / alpha_j are staged in shared memory, and the
// exponentials use the branch-free lb_exp_nonpos (<= 3e-16 relative, inside the 1e-9 bar of the gradient).
constexpr int GRAD_PMAX = 4; // outputs staged in shared memory (more: global loads)

// columns per pass: 4 chunks of 8 (four passes over the 128 columns of a tile) keep the live accumulators small enough for three
// CTAs per SM (the kernel is bound by latency / instruction issue rather than by the fp64 pipe)
constexpr int GNC = 2, GNH = 16 / GNC, GHW = 8 * GNC;

template <int KID, bool EDGE>
__device__ __forceinline__ void grad_tile(const double* __restrict__ Xs, const double* __restrict__ Kinv, const double* __restrict__ alpha, int P,
    int64_t N, int64_t Np, const KernParams& kp, int optimize_noise, int nh, double* __restrict__ part, int bi, int bj,
    double (*sxi)[LB_TILE], double (*sxj)[LB_TILE], double (*sai)[LB_TILE], double (*saj)[LB_TILE], double (*sred)[DCH + 4], double* stot,
    uint64_t* bar)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int li = lane & 7, lj = lane >> 3;
    const int D = kp.D;
    const int64_t i0 = (int64_t)bi * LB_TILE, j0 = (int64_t)bj * LB_TILE;
    const int r0 = warp * 16 + 2 * li;
    constexpr bool ard = (KID == LB_K_SE_ARD);
    if (tid == 0) {
        lb_mbar_init(bar, 1);
        lb_fence_barrier_init();
    }
    for (int q = tid; q < LB_MAX_D + 2; q += 256) stot[q] = 0.0;
    const int Ps = P < GRAD_PMAX ? P : GRAD_PMAX;
    for (int idx = tid; idx < Ps * LB_TILE; idx += 256) {
        const int p = idx >> 7, c = idx & 127;
        sai[p][c] = alpha[i0 + c + (int64_t)p * Np];
        saj[p][c] = alpha[j0 + c + (int64_t)p * Np];
    }
    __syncthreads();
    uint32_t phase = 0;
    const int npass = (D + DCH - 1) / DCH;

    double g_sf = 0.0, g_l = 0.0, g_noise = 0.0;
    for (int h = 0; h < GNH; ++h) { // GNH passes of GHW columns
        // the K^-1 values of this half: issued before the distance sweep so that their latency hides under it
        const int64_t gi = i0 + r0;
        double2 kv[GNC][2];
#pragma unroll
        for (int c = 0; c < GNC; ++c) {
            const int64_t gj = j0 + h * GHW + c * 8 + 2 * lj;
            kv[c][0] = __ldcs(reinterpret_cast<const double2*>(&Kinv[gi + gj * Np]));
            kv[c][1] = __ldcs(reinterpret_cast<const double2*>(&Kinv[gi + (gj + 1) * Np]));
        }
        double z[GNC][4];
        pair_distances<GNC>(Xs, Np, i0, Xs, Np, j0, D, sxi, sxj, bar, phase, h, z);
        // weights w_ij * f_ij and the parameter-independent factors
        double wk[GNC][4]; // SE-ARD: w * f * k
#pragma unroll
        for (int c = 0; c < GNC; ++c) {
            const int cl = h * GHW + c * 8 + 2 * lj; // local column
            const int64_t gj = j0 + cl;
            const double kin[4] = {kv[c][0].x, kv[c][0].y, kv[c][1].x, kv[c][1].y};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int rl = r0 + (e & 1), cc = cl + (e >> 1);
                double w = -kin[e];
                for (int p = 0; p < Ps; ++p) w = fma(sai[p][rl], saj[p][cc], w);
                for (int p = Ps; p < P; ++p) w = fma(alpha[i0 + rl + (int64_t)p * Np], alpha[j0 + cc + (int64_t)p * Np], w);
                if (EDGE) { // diagonal tile (strictly upper part does not count, the diagonal counts half) or padding
                    const int64_t ii = gi + (e & 1), jj = gj + (e >> 1);
                    double f = (ii == jj) ? 0.5 : ((ii > jj) ? 1.0 : 0.0);
                    if (ii >= N || jj >= N) f = 0.0;
                    w *= f;
                    if (ii == jj) g_noise = fma(w, 2.0 * kp.noise, g_noise); // kernel.hpp:90-93
                }
                double g0, g1; // common.cuh lb_kernel_grad_pair
                lb_kernel_grad_pair<KID>(z[c][e], kp, g0, g1);
                if (ard) {
                    wk[c][e] = w * g0;
                    g_sf = fma(w, g1, g_sf);
                }
                else {
                    wk[c][e] = 0.0;
                    g_l = fma(w, g0, g_l);
                    g_sf = fma(w, g1, g_sf);
                }
            }
        }
        if (ard) {
            // second sweep over the input dimensions: g_d += w k q_d^2
            for (int pass = 0; pass < npass; ++pass) {
                int dc;
                if (npass > 1) dc = pair_stage(Xs, Np, i0, Xs, Np, j0, D, pass, sxi, sxj, bar, phase);
                else dc = D;
                const int d0 = pass * DCH;
                double gd[DCH];
#pragma unroll
                for (int d = 0; d < DCH; ++d) gd[d] = 0.0;
#pragma unroll
                for (int d = 0; d < DCH; ++d) {
                    if (d < dc) {
                        const double2 xi = *reinterpret_cast<const double2*>(&sxi[d][r0]);
                        double s = 0.0;
#pragma unroll
                        for (int c = 0; c < GNC; ++c) {
                            const double2 xj = *reinterpret_cast<const double2*>(&sxj[d][h * GHW + c * 8 + 2 * lj]);
                            double q;
                            q = xi.x - xj.x; s = fma(wk[c][0], q * q, s);
                            q = xi.y - xj.x; s = fma(wk[c][1], q * q, s);
                            q = xi.x - xj.y; s = fma(wk[c][2], q * q, s);
                            q = xi.y - xj.y; s = fma(wk[c][3], q * q, s);
                        }
                        gd[d] = s;
                    }
                }
#pragma unroll
                for (int d = 0; d < DCH; ++d) {
                    if (d < dc) { // dc is uniform over the CTA
                        double s = lb_warp_sum(gd[d]);
                        if (lane == 0) sred[warp][d] = s;
                    }
                }
                __syncthreads();
                if (tid < dc) {
                    double s = 0.0;
                    for (int w = 0; w < 8; ++w) s += sred[w][tid];
                    stot[d0 + tid] += s;
                }
                __syncthreads();
            }
        }
    }
    // scalar parts
    g_sf = lb_warp_sum(g_sf);
    g_l = lb_warp_sum(g_l);
    g_noise = lb_warp_sum(g_noise);
    __syncthreads();
    if (lane == 0) { sred[warp][0] = g_sf; sred[warp][1] = g_l; sred[warp][2] = g_noise; }
    __syncthreads();
    if (tid == 0) {
        double a = 0, b = 0, c = 0;
        for (int w = 0; w < 8; ++w) { a += sred[w][0]; b += sred[w][1]; c += sred[w][2]; }
        double* out = part + (int64_t)blockIdx.x * nh;
        if (ard) { // [ell (Draw), Lambda entries (filled by lb_launch_grad_lambda), sigma_f, (noise)]
            const int nk = nh - (optimize_noise ? 1 : 0);
            for (int d = 0; d < kp.Draw; ++d) out[d] = stot[d];
            for (int d = kp.Draw; d < nk - 1; ++d) out[d] = 0.0;
            out[nk - 1] = a;
            if (optimize_noise) out[nk] = c;
        }
        else {
            out[0] = b;
            out[1] = a;
            if (optimize_noise) out[2] = c;
        }
    }
}

template <int KID>
__global__ void __launch_bounds__(256, 3)
grad_kernel(const double* __restrict__ Xs, const double* __restrict__ Kinv, const double* __restrict__ alpha, int P,
    int64_t N, int64_t Np, KernParams kp, int optimize_noise, int nh, double* __restrict__ part)
{
    __shared__ __align__(128) double sxi[DCH][LB_TILE];
    __shared__ __align__(128) double sxj[DCH][LB_TILE];
    __shared__ double sai[GRAD_PMAX][LB_TILE];
    __shared__ double saj[GRAD_PMAX][LB_TILE];
    __shared__ double sred[8][DCH + 4];
    __shared__ double stot[LB_MAX_D + 2];
    __shared__ __align__(8) uint64_t bar;
    int bi, bj;
    tile_from_index(blockIdx.x, bi, bj);
    const bool edge = (bi == bj) || ((int64_t)(bi + 1) * LB_TILE > N);
    if (edge) grad_tile<KID, true>(Xs, Kinv, alpha, P, N, Np, kp, optimize_noise, nh, part, bi, bj, sxi, sxj, sai, saj, sred, stot, &bar);
    else grad_tile<KID, false>(Xs, Kinv, alpha, P, N, Np, kp, optimize_noise, nh, part, bi, bj, sxi, sxj, sai, saj, sred, stot, &bar);
}

__global__ void __launch_bounds__(256)
grad_reduce_kernel(const double* __restrict__ part, int ntiles, int nh, double* __restrict__ grad)
{
    __shared__ double red[8];
    const int q = blockIdx.x;
    double s = 0.0;
    for (int t = threadIdx.x; t < ntiles; t += 256) s += part[(int64_t)t * nh + q];
    s = lb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        grad[q] = t;
    }
}


LbOncePerDevice g_attr_once;
int set_attrs()
{
    if (!g_attr_once.need()) return LB_OK;
    LB_CUDA(cudaFuncSetAttribute(lauum_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbg::CfgWide::PIPE_BYTES));
    LB_CUDA(cudaFuncSetAttribute(trtri_level_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lbg::CfgWide::PIPE_BYTES));
    return LB_OK;
}

} // namespace

int lb_launch_loglik(lb_gp* h, double* dOut)
{
    loglik_kernel<<<1, 1024, 0, h->stream>>>(h->dL, h->Np, h->N, h->dY, h->dAlpha, h->P, dOut);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Inverse of the diagonal blocks of L made of `want_tiles` 128-tiles (a power of two; >= T: all of L^-1), by the levels of
// the recursion above; levels already present are kept (the batched query wants 16-tile blocks, the likelihood gradient
// all of L^-1 - the second continues where the first stopped).  dKinv is the W workspace of the recursion.
int lb_launch_linv_levels(lb_gp* h, int want_tiles)
{
    int rc = set_attrs();
    if (rc) return rc;
    const int T = (int)(h->Np / LB_TILE);
    const size_t bytes = sizeof(double) * h->Np * h->Np;
    if (!h->dLinv) {
        if ((rc = h->dLinv.reserve(h, bytes))) return rc;
        LB_CUDA(cudaMemsetAsync(h->dLinv.get(), 0, bytes, h->stream)); // strict upper part stays zero
        h->linv_levels = 0;
    }
    if ((rc = h->dKinv.reserve(h, bytes))) return rc; // doubles as the W workspace of the recursion
    LbProfScope ps(h, h->stream, LB_PC_TRTRI);
    if (h->linv_levels == 0) {
        trtri_diag_copy_kernel<<<T, 256, 0, h->stream>>>(h->dInvD, h->dLinv.get(), h->Np);
        h->launches++;
        h->linv_levels = 1;
    }
    for (int sb = h->linv_levels; sb < want_tiles && sb < T; sb *= 2) {
        const int nprob = (T + 2 * sb - 1) / (2 * sb);
        h->kinv_valid = false; // W overwrites dKinv
        for (int step = 1; step <= 2; ++step) {
            trtri_level_kernel<<<nprob * sb * sb, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, h->stream>>>(h->dL, h->dLinv.get(), h->dKinv.get(), h->Np, sb,
                step, T);
            h->launches++;
        }
        h->linv_levels = 2 * sb;
    }
    LB_CUDA(cudaGetLastError());
    if (h->linv_levels >= T) h->linv_valid = true;
    return LB_OK;
}

int lb_launch_linv(lb_gp* h)
{
    const int T = (int)(h->Np / LB_TILE);
    int want = 1;
    while (want < T) want *= 2;
    return lb_launch_linv_levels(h, want);
}

int lb_launch_kinv(lb_gp* h)
{
    int rc = set_attrs();
    if (rc) return rc;
    if (!h->linv_valid) {
        rc = lb_launch_linv(h);
        if (rc) return rc;
    }
    const int T = (int)(h->Np / LB_TILE);
    if ((rc = h->dKinv.reserve(h, sizeof(double) * h->Np * h->Np))) return rc;
    LbProfScope ps(h, h->stream, LB_PC_LAUUM);
    lauum_kernel<<<T * (T + 1) / 2, lbg::CfgWide::THREADS, lbg::CfgWide::PIPE_BYTES, h->stream>>>(h->dLinv.get(), h->Np, h->dKinv.get(), T);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    h->kinv_valid = true;
    h->kinv_sym = false;
    return LB_OK;
}

int lb_launch_symmetrize(lb_gp* h, double* dA)
{
    dim3 grid((unsigned)(h->Np / 32), (unsigned)(h->Np / 32));
    symmetrize_kernel<<<grid, dim3(32, 8), 0, h->stream>>>(dA, h->Np);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_grad(lb_gp* h, int optimize_noise, double* dGrad)
{
    const int T = (int)(h->Np / LB_TILE);
    const int ntiles = T * (T + 1) / 2;
    const int nh = h->n_hparams + (optimize_noise ? 1 : 0);
    int rc = lb_ensure_scratch(h, sizeof(double) * (size_t)ntiles * nh);
    if (rc) return rc;
    LbProfScope ps(h, h->stream, LB_PC_GRAD);
    switch (h->kp.id) {
    case LB_K_SE_ARD: grad_kernel<LB_K_SE_ARD><<<ntiles, 256, 0, h->stream>>>(h->dXs, h->dKinv.get(), h->dAlpha, h->P, h->N, h->Np, h->kp, optimize_noise, nh, h->dScratch.get()); break;
    case LB_K_MATERN52: grad_kernel<LB_K_MATERN52><<<ntiles, 256, 0, h->stream>>>(h->dXs, h->dKinv.get(), h->dAlpha, h->P, h->N, h->Np, h->kp, optimize_noise, nh, h->dScratch.get()); break;
    case LB_K_MATERN32: grad_kernel<LB_K_MATERN32><<<ntiles, 256, 0, h->stream>>>(h->dXs, h->dKinv.get(), h->dAlpha, h->P, h->N, h->Np, h->kp, optimize_noise, nh, h->dScratch.get()); break;
    default: grad_kernel<LB_K_EXP><<<ntiles, 256, 0, h->stream>>>(h->dXs, h->dKinv.get(), h->dAlpha, h->P, h->N, h->Np, h->kp, optimize_noise, nh, h->dScratch.get()); break;
    }
    grad_reduce_kernel<<<nh, 256, 0, h->stream>>>(h->dScratch.get(), ntiles, nh, dGrad);
    h->launches += 2;
    LB_CUDA(cudaGetLastError());
    if (h->kp.id == LB_K_SE_ARD && h->kp.klam > 0) return lb_launch_grad_lambda(h, dGrad);
    return LB_OK;
}
