// limbo_b200/csrc/query_grad.cu — batched candidate gradients of mu, sigma^2 and the UCB / GP_UCB / EI acquisitions.
//
// The reference's acquisitions assert(!gradient) (acqui/ucb.hpp:83-90, gp_ucb.hpp:96-103, ei.hpp:85-116); its gradient
// optimisers (opt/gradient_ascent.hpp, opt/adam.hpp, opt/rprop.hpp) take f(x, gradient).  For M candidates at once:
//   forward   lb_launch_query_panel (query.cu, unchanged): K*, mu = K*^T alpha, V = L^-1 K*, sigma^2
//   backward  W = L^-T V in place over V, 2048-row super-blocks from the last to the first (panel_bwd_update_kernel,
//             panel_bwd_solve_kernel: the forward panel solve's tiles with the transposed factor as a K-contiguous A operand)
//   gradient  query_grad_kernel: the kernel values of the N x M pairs again (K* is gone once the solve has run), then
//             grad mu = sum_n g_n alpha_n0,  grad sigma^2 = -2 sum_n g_n W_nc   (g_n = dk(u, u_n)/du, k(v, v) is constant)
//             mapped back from the staged coordinates u to x, and the acquisition's value and gradient.
#include "gemm.cuh"
#include <cfloat>

namespace {

namespace panel_bwd {

constexpr int SB = 16;

// Tbuf[i, ct] = V[s0 + i, ct] - L[s1:, s0 + i]^T W[s1:, ct]     (s1 = s0 + nrows: the rows below the super-block, already W)
// A = L^T is read down the columns of the column-major factor: a K-contiguous operand.   grid = nrows * ncols, row tile fastest
template <typename C>
__global__ void __launch_bounds__(C::THREADS, C::CTAS_PER_SM)
panel_bwd_update_kernel(const double* __restrict__ L, int64_t ld, const double* __restrict__ V, double* __restrict__ Tbuf, int64_t ldt,
    int s0, int nrows, int T, int ct0)
{
    extern __shared__ __align__(16) double smem[];
    const int i = blockIdx.x % nrows, ct = ct0 + blockIdx.x / nrows;
    const int s1 = s0 + nrows;
    const double* Vc = V + (int64_t)ct * C::BN * ld;
    lbg::Acc<C> acc;
    lbg::load_acc<C>(acc, Vc + (int64_t)(s0 + i) * LB_TILE, ld);
    if (s1 < T)
        lbg::mainloop<C, true, true, true>(acc, L + (int64_t)s1 * LB_TILE + (int64_t)(s0 + i) * LB_TILE * ld, ld, Vc + (int64_t)s1 * LB_TILE, ld,
            (T - s1) * LB_TILE, smem);
    lbg::store_acc<C>(acc, Tbuf + (int64_t)i * LB_TILE + (int64_t)ct * C::BN * ldt, ldt);
}

// W[s0 + i, ct] = sum_{k >= i} inv(L_ss)[s0 + k, s0 + i] Tbuf[k, ct]   (inv(L_ss)^T is upper triangular; the diagonal tiles of
// the cached inverse have a zero upper part)
template <typename C>
__global__ void __launch_bounds__(C::THREADS, C::CTAS_PER_SM)
panel_bwd_solve_kernel(const double* __restrict__ Linv, int64_t ld, const double* __restrict__ Tbuf, int64_t ldt, double* __restrict__ W,
    int s0, int nrows, int ct0)
{
    extern __shared__ __align__(16) double smem[];
    const int i = (int)(blockIdx.x % nrows), ct = ct0 + blockIdx.x / nrows; // i = 0 has the longest K range: first
    lbg::Acc<C> acc;
    acc.zero();
    lbg::mainloop<C, true, true>(acc, Linv + (int64_t)(s0 + i) * LB_TILE + (int64_t)(s0 + i) * LB_TILE * ld, ld,
        Tbuf + (int64_t)i * LB_TILE + (int64_t)ct * C::BN * ldt, ldt, (nrows - i) * LB_TILE, smem);
    lbg::store_acc<C>(acc, W + (int64_t)(s0 + i) * LB_TILE + (int64_t)ct * C::BN * ld, ld);
}

LbOncePerDevice g_once;

} // namespace panel_bwd

constexpr int GTHREADS = 256;
constexpr int GCH = 16; // staged coordinates per accumulation pass

// dk(u, u_n)/du = c(z) (u - u_n) for the four stationary kernels (z = |u - u_n|^2 in staged coordinates)
template <int KID>
__device__ __forceinline__ double grad_coef(double z, const KernParams& kp)
{
    if (KID == LB_K_SE_ARD) return -lb_kernel_from_z(LB_K_SE_ARD, z, kp); // -k
    if (KID == LB_K_EXP) return -lb_kernel_from_z(LB_K_EXP, z, kp) * kp.c1; // -k / l^2
    const double d = lb_dist_from_z(z);
    const double e = lb_exp_nonpos(-kp.c1 * d);
    if (KID == LB_K_MATERN52) return -kp.sf2 * kp.c2 * fma(kp.c1, d, 1.0) * e; // -(5 sf2 / 3 l^2)(1 + sqrt5 d / l) e^(-sqrt5 d / l)
    return -kp.sf2 * (kp.c1 * kp.c1) * e;                                        // -(3 sf2 / l^2) e^(-sqrt3 d / l)
}

// One CTA per candidate.  Every thread takes the training points n = tid + 256 j in a fixed order; the per-thread sums are
// reduced over the lanes and then over the warps in a fixed order, so a candidate's result is run-to-run identical and does
// not depend on the other candidates of the batch.  mu0 / s2 / norms: the forward pass's outputs for this chunk.
template <int KID>
__global__ void __launch_bounds__(GTHREADS)
query_grad_kernel(const double* __restrict__ Xs, int64_t Np, int64_t N, const double* __restrict__ Qs, int64_t Mp,
    const double* __restrict__ alpha, const double* __restrict__ W, const double* __restrict__ mu0, int P, const double* __restrict__ s2,
    const double* __restrict__ norms, int T, const KernParams kp, const LbGradOut out)
{
    __shared__ double su[LB_MAX_D];
    __shared__ double red[2][GTHREADS / 32][GCH];
    __shared__ double gu[2][LB_MAX_D];
    __shared__ int clamped;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t m = blockIdx.x;
    const int De = kp.D, Draw = kp.Draw;
    for (int d = tid; d < De; d += GTHREADS) su[d] = Qs[(int64_t)d * Mp + m];
    if (tid == 0) { // the clamp of gp.hpp:623, from the same partial sums in the same order as panel_finish_kernel
        double s = 0.0;
        for (int tt = 0; tt < T; ++tt) s += norms[(int64_t)tt * Mp + m];
        clamped = (kp.sf2 - s) <= DBL_EPSILON;
    }
    __syncthreads();
    const double* Wc = W + m * Np;
    for (int d0 = 0; d0 < De; d0 += GCH) {
        const int dc = min(GCH, De - d0);
        double am[GCH], aw[GCH];
#pragma unroll
        for (int j = 0; j < GCH; ++j) am[j] = aw[j] = 0.0;
        for (int64_t n = tid; n < N; n += GTHREADS) {
            double z = 0.0;
            for (int d = 0; d < De; ++d) {
                const double q = su[d] - Xs[(int64_t)d * Np + n];
                z = fma(q, q, z);
            }
            const double c = grad_coef<KID>(z, kp);
            const double ca = c * alpha[n], cw = c * Wc[n];
#pragma unroll
            for (int j = 0; j < GCH; ++j)
                if (j < dc) {
                    const double q = su[d0 + j] - Xs[(int64_t)(d0 + j) * Np + n];
                    am[j] = fma(ca, q, am[j]);
                    aw[j] = fma(cw, q, aw[j]);
                }
        }
#pragma unroll
        for (int j = 0; j < GCH; ++j) {
            const double a = lb_warp_sum(am[j]), b = lb_warp_sum(aw[j]);
            if (lane == 0) {
                red[0][warp][j] = a;
                red[1][warp][j] = b;
            }
        }
        __syncthreads();
        if (tid < 2 * GCH) {
            const int k = tid / GCH, j = tid % GCH;
            double s = 0.0;
            for (int w = 0; w < GTHREADS / 32; ++w) s += red[k][w][j];
            if (j < dc) gu[k][d0 + j] = (k == 0) ? s : -2.0 * s;
        }
        __syncthreads();
    }
    if (tid >= Draw) return;
    // back to the caller's coordinates: u_r = x_r / ell_r (r < Draw), u_{Draw + j} = sum_r A[r, j] x_r (SE-ARD); u = x otherwise
    const int r = tid;
    double gmu = gu[0][r], gs2 = gu[1][r];
    if (KID == LB_K_SE_ARD) {
        gmu *= kp.inv_ell[r];
        gs2 *= kp.inv_ell[r];
        for (int j = 0; j < kp.klam; ++j) {
            const double a = kp.lambda[(int64_t)j * Draw + r];
            gmu = fma(a, gu[0][Draw + j], gmu);
            gs2 = fma(a, gu[1][Draw + j], gs2);
        }
    }
    if (clamped) gs2 = 0.0;
    const int64_t o = m * Draw + r;
    if (out.dmu) out.dmu[o] = gmu;
    if (out.ds2) out.ds2[o] = gs2;
    if (out.acq_id < 0) return;
    const double s = s2[m];
    const double mu = mu0[m * P] + (out.mean ? out.mean[m] : out.mean_const);
    if (out.mean_grad) gmu += out.mean_grad[o];
    const double g = lb_acq_grad_value(out.acq_id, mu, s, gmu, gs2, out.p0, out.p1);
    if (out.grad) out.grad[o] = g;
    if (r == 0 && out.acq) out.acq[m] = lb_acq_value(out.acq_id, mu, s, out.p0, out.p1);
}

// The prior (no samples, gp.hpp:161-163): mu = 0 (the caller's mean is added by the caller), sigma^2 = k(v, v) + noise, zero
// gradients of both; the acquisition from the mean alone, with acq_kernel's value formula.
__global__ void __launch_bounds__(256)
prior_grad_kernel(int64_t M, int D, int P, double s, const LbGradOut out, double* __restrict__ mu, double* __restrict__ s2)
{
    const int64_t m = blockIdx.x * (int64_t)256 + threadIdx.x;
    if (m >= M) return;
    for (int p = 0; p < P; ++p) mu[m * P + p] = 0.0;
    s2[m] = s;
    for (int d = 0; d < D; ++d) {
        if (out.dmu) out.dmu[m * D + d] = 0.0;
        if (out.ds2) out.ds2[m * D + d] = 0.0;
    }
    if (out.acq_id < 0) return;
    const double mean = out.mean ? out.mean[m] : out.mean_const;
    if (out.acq) out.acq[m] = lb_acq_value(out.acq_id, mean, s, out.p0, out.p1);
    double w = 1.0; // UCB: d(mu + p0 sqrt(s)) = d mean
    if (out.acq_id != 0) { // EI: Phi(Z) d mean, 0 below sigma = 1e-10
        const double sigma = sqrt(s);
        w = (sigma < 1e-10) ? 0.0 : 0.5 * erfc(-((mean - out.p0 - out.p1) / sigma) / sqrt(2.0));
    }
    if (out.grad)
        for (int d = 0; d < D; ++d) out.grad[m * D + d] = out.mean_grad ? w * out.mean_grad[m * D + d] : 0.0;
}

} // namespace

int lb_launch_prior_grad(cudaStream_t st, int64_t M, int D, int P, double s2, const LbGradOut& out, double* dMu, double* dS2)
{
    prior_grad_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(M, D, P, s2, out, dMu, dS2);
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// W = L^-T V in place over the panel workspace's V (Np x Mp), after lb_launch_query_panel has left V = L^-1 K* there.
int lb_launch_query_bwd(lb_gp* h, cudaStream_t st, int64_t Mp, double* dWork, long long* launches)
{
    using namespace panel_bwd;
    using CD = lbg::CfgDual;
    if (g_once.need()) {
        LB_CUDA(cudaFuncSetAttribute(panel_bwd_update_kernel<CD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CD::PIPE_BYTES));
        LB_CUDA(cudaFuncSetAttribute(panel_bwd_solve_kernel<CD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CD::PIPE_BYTES));
    }
    const int T = (int)(h->Np / LB_TILE);
    const int64_t ld = h->Np, ldt = (int64_t)SB * LB_TILE;
    double* dV = dWork;
    double* dT = lb_query_panel_tbuf(h, dWork, Mp);
    constexpr int wmul = LB_TILE / CD::BN;
    cudaStream_t sts[4];
    int gbeg[5];
    const int ngroups = lb_query_panel_groups(h, st, (int)(Mp / LB_TILE), sts, gbeg);
    LbProfScope ps(h, st, LB_PC_QSTEP);
    if (ngroups >= 2) {
        LB_CUDA(cudaEventRecord(h->ev[0], st));
        for (int g = 1; g < ngroups; ++g) LB_CUDA(cudaStreamWaitEvent(sts[g], h->ev[0], 0));
    }
    for (int s0 = (T - 1) / SB * SB; s0 >= 0; s0 -= SB) {
        const int nrows = (T - s0 < SB) ? (T - s0) : SB;
        for (int g = 0; g < ngroups; ++g) {
            const int c0 = gbeg[g] * wmul, nc = (gbeg[g + 1] - gbeg[g]) * wmul;
            if (nc <= 0) continue;
            panel_bwd_update_kernel<CD><<<nrows * nc, CD::THREADS, CD::PIPE_BYTES, sts[g]>>>(h->dL, ld, dV, dT, ldt, s0, nrows, T, c0);
            panel_bwd_solve_kernel<CD><<<nrows * nc, CD::THREADS, CD::PIPE_BYTES, sts[g]>>>(h->dLinv.get(), ld, dT, ldt, dV, s0, nrows, c0);
            if (launches) *launches += 2;
        }
    }
    for (int g = 1; g < ngroups; ++g) {
        LB_CUDA(cudaEventRecord(h->ev[g], sts[g]));
        LB_CUDA(cudaStreamWaitEvent(st, h->ev[g], 0));
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Forward pass, backward solve and gradient pass for M (<= Mp) staged candidates dQs (De x Mp): mu (M x P) and sigma^2 (M) as
// lb_launch_query_panel leaves them, and the gradient outputs of `out`, whose pointers start at this chunk.
int lb_launch_query_grad(lb_gp* h, cudaStream_t st, int64_t M, const double* dQs, int64_t Mp, double* dWork, double* dMu, double* dS2,
    const LbGradOut& out, long long* launches)
{
    int rc = lb_launch_query_panel(h, st, M, dQs, Mp, dWork, dMu, dS2, launches);
    if (rc) return rc;
    if ((rc = lb_launch_query_bwd(h, st, Mp, dWork, launches))) return rc;
    const int T = (int)(h->Np / LB_TILE);
    const double* norms = lb_query_panel_norms(h, dWork, Mp); // the forward pass's |V_c|^2 partials, for the clamp test
    const int P = h->P > 0 ? h->P : 1;
    {
        LbProfScope ps(h, st, LB_PC_QREDUCE);
        switch (h->kp.id) {
#define LB_GRAD_LAUNCH(KID)                                                                                                      \
    case KID:                                                                                                                    \
        query_grad_kernel<KID><<<(unsigned)M, GTHREADS, 0, st>>>(h->dXs, h->Np, h->N, dQs, Mp, h->dAlpha, dWork, dMu, P, dS2, norms, T, \
            h->kp, out);                                                                                                         \
        break;
            LB_GRAD_LAUNCH(LB_K_SE_ARD)
            LB_GRAD_LAUNCH(LB_K_MATERN52)
            LB_GRAD_LAUNCH(LB_K_MATERN32)
            LB_GRAD_LAUNCH(LB_K_EXP)
#undef LB_GRAD_LAUNCH
        default: return LB_ERR_UNSUPPORTED;
        }
    }
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
