// limbo_b200/csrc/loo.cu — leave-one-out cross-validation objective of the GP and its kernel gradient
// (the objective of model::gp::KernelLooOpt, model/gp/kernel_loo_opt.hpp:57-97), and the K^-1 * obs_mean product
// the mean-parameter gradient is built from.
//
//   GP::compute_log_loo_cv              model/gp.hpp:339-351 -> loo_value_kernel (diag(K^-1), alpha; O(N))
//   GP::compute_kernel_grad_log_loo_cv  model/gp.hpp:353-399 -> per hyper-parameter q:
//        dk_build_kernel   dK/dtheta_q, N x N, generated from X (the reference assembles it from N(N+1)/2 functor calls)
//        loo_zeta_kernel   Z = K^-1 dK on the fp64 tensor cores (DMMA); Z is never stored: the epilogue reduces
//                          (Z alpha)_i and (Z K^-1)_ii = sum_l Z_il K^-1_li per row and 128-column tile
//        loo_grad_reduce_kernel   sum_i,p [alpha Zalpha - 1/2 (1 + alpha^2 / K^-1_ii) (Z K^-1)_ii] / K^-1_ii  (fixed order)
//      The reference forms Z, Z alpha and Z K^-1 as three dense products per parameter (6 N^3 flops); here 2 N^3.
//   GP::compute_mean_grad_log_lik       model/gp.hpp:313-330 -> kinv_obs_kernel: obs_mean^T K^-1 (the mean functor's own
//                                       gradient stays on the host, mean/mean.hpp:72-76)
#include "gemm.cuh"

namespace {

using Cfg = lbg::CfgWide;

// dK[i + j*ld] = d k(x_i, x_j) / d theta_q for i, j < N, 0 in the padding.
//   SE-ARD   (squared_exp_ard.hpp:107-136): q < D: k * ((x_q - y_q)/ell_q)^2 ; Lambda entry A(i,j): -k (d^T A(:,j)) d_i ;
//            last: 2k
//   Matern52 (matern_five_halves.hpp:115-133), Matern32 (matern_three_halves.hpp:110-124), Exp (exp.hpp:101-110):
//            q == 0: d/d log l ; q == 1: 2k
//   q == n_hparams (optimize_noise): 2 * noise on the diagonal (kernel.hpp:90-93)
__global__ void __launch_bounds__(256)
dk_build_kernel(const double* __restrict__ Xs, int64_t Np, int64_t N, KernParams kp, int q, int n_hparams, double* __restrict__ dK)
{
    const int64_t i = (int64_t)blockIdx.y * 256 + threadIdx.x; // columns on grid.x (no 65535 limit), 256-row slabs on grid.y
    const int64_t j = blockIdx.x;
    if (i >= Np) return;
    double out = 0.0;
    if (i < N && j < N) {
        if (q >= n_hparams)
            out = (i == j) ? 2.0 * kp.noise : 0.0;
        else {
            // SE-ARD parameter layout: [ell (Draw), A(:,0) .. A(:,klam-1) (Draw each), sigma_f]
            const bool is_lam = (kp.id == LB_K_SE_ARD) && q >= kp.Draw && q < n_hparams - 1;
            const int lam_j = is_lam ? (q - kp.Draw) / kp.Draw : 0, lam_i = is_lam ? (q - kp.Draw) % kp.Draw : 0;
            double z = 0.0, qd2 = 0.0, proj = 0.0, raw = 0.0;
            for (int d = 0; d < kp.D; ++d) {
                const double df = Xs[(int64_t)d * Np + i] - Xs[(int64_t)d * Np + j];
                z = fma(df, df, z);
                if (d == q) qd2 = df * df;
                if (is_lam && d == kp.Draw + lam_j) proj = df;          // (x1 - x2)^T A(:,j)
                if (is_lam && d == lam_i) raw = df / kp.inv_ell[lam_i];  // (x1 - x2)_i (the staged one is divided by ell_i)
            }
            if (kp.id == LB_K_SE_ARD) {
                const double k = kp.sf2 * exp(-0.5 * z);
                if (q < kp.Draw) out = k * qd2;             // squared_exp_ard.hpp:117 / :131
                else if (is_lam) out = -proj * raw * k;     // squared_exp_ard.hpp:119-122
                else out = 2.0 * k;
            }
            else if (kp.id == LB_K_MATERN52) {
                const double d = sqrt(z), d_sq = d * d, l_sq = kp.l * kp.l;
                const double term1 = sqrt(5.0) * d / kp.l;
                const double term2 = 5. * d_sq / (3. * l_sq);
                const double r = exp(-term1);
                out = (q == 0) ? kp.sf2 * (r * term1 * (1 + term1 + term2) + (-term1 - 2. * term2) * r) : 2 * kp.sf2 * (1 + term1 + term2) * r;
            }
            else if (kp.id == LB_K_MATERN32) {
                const double d = sqrt(z);
                const double term = sqrt(3.0) * d / kp.l;
                const double r = exp(-term);
                out = (q == 0) ? kp.sf2 * (-term * r + (1 + term) * term * r) : 2 * kp.sf2 * (1 + term) * r;
            }
            else {
                const double r = z / (kp.l * kp.l);
                const double k = kp.sf2 * exp(-0.5 * r);
                out = (q == 0) ? r * k : 2 * k;
            }
        }
    }
    dK[i + j * Np] = out;
}

// One 128 x 128 tile of Z = Kinv * dK (both symmetric, full storage, column-major):
//   Z[i0+m, j0+n] = sum_k Kinv[i0+m, k] dK[k, j0+n]
// A operand = Kinv rows (outer-contiguous), B operand = dK columns (K-contiguous).  Epilogue per row m:
//   part_zk[bj][i0+m]    = sum_n Z[m,n] Kinv[i0+m, j0+n]        (Kinv symmetric: = Kinv[j0+n, i0+m])
//   part_za[p][bj][i0+m] = sum_n Z[m,n] alpha[j0+n, p]
__global__ void __launch_bounds__(Cfg::THREADS, 1)
loo_zeta_kernel(const double* __restrict__ Kinv, const double* __restrict__ dK, int64_t ld, const double* __restrict__ alpha, int P, int T,
    double* __restrict__ part_zk, double* __restrict__ part_za)
{
    extern __shared__ __align__(16) double smem[];
    const int bi = blockIdx.x % T, bj = blockIdx.x / T;
    const int64_t i0 = (int64_t)bi * LB_TILE, j0 = (int64_t)bj * LB_TILE;
    lbg::Acc<Cfg> acc;
    acc.zero();
    lbg::mainloop<Cfg, false, true>(acc, Kinv + i0, ld, dK + j0 * ld, ld, T * LB_TILE, smem);
    // after the main loop the pipeline memory is free: red[wn][row]
    double* red = smem;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp & 3, wn = warp >> 2;
    constexpr int WCOLS = Cfg::BN / Cfg::WN;
    for (int pass = 0; pass <= P; ++pass) { // pass 0: Kinv weights; pass p+1: alpha column p
        double s[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < Cfg::NT; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int row = wm * 32 + mt * 16 + g + 8 * (i >> 1);
                    const int col = wn * WCOLS + nt * 8 + 2 * t + (i & 1);
                    const double w = (pass == 0) ? Kinv[i0 + row + (j0 + col) * ld] : alpha[j0 + col + (int64_t)(pass - 1) * ld];
                    s[mt][i >> 1] = fma(acc.v[mt][nt][i], w, s[mt][i >> 1]);
                }
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                double v = s[mt][hf];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                if (t == 0) red[wn * LB_TILE + wm * 32 + mt * 16 + g + 8 * hf] = v;
            }
        __syncthreads();
        if (threadIdx.x < LB_TILE) {
            double v = red[threadIdx.x];
#pragma unroll
            for (int w = 1; w < Cfg::WN; ++w) v += red[w * LB_TILE + threadIdx.x];
            double* dst = (pass == 0) ? part_zk : part_za + (int64_t)(pass - 1) * T * ld;
            dst[(int64_t)bj * ld + i0 + threadIdx.x] = v;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ double block_sum_1024(double v, double* sh)
{
    v = lb_warp_sum(v);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = 0.0;
    if (threadIdx.x < 32) r = lb_warp_sum(sh[threadIdx.x]);
    __syncthreads();
    return r;
}

// gp.hpp:391: sum over i, p of (alpha Zalpha - 0.5 (1 + alpha^2 inv_diag) diag(Z Kinv)) inv_diag
__global__ void __launch_bounds__(1024)
loo_grad_reduce_kernel(const double* __restrict__ Kinv, int64_t ld, int64_t N, const double* __restrict__ alpha, int P, int T,
    const double* __restrict__ part_zk, const double* __restrict__ part_za, double* __restrict__ out)
{
    __shared__ double sh[32];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < N; i += 1024) {
        double zk = 0.0;
        for (int b = 0; b < T; ++b) zk += part_zk[(int64_t)b * ld + i];
        const double inv_diag = 1.0 / Kinv[i + i * ld];
        for (int p = 0; p < P; ++p) {
            double za = 0.0;
            const double* q = part_za + (int64_t)p * T * ld + i;
            for (int b = 0; b < T; ++b) za += q[(int64_t)b * ld];
            const double a = alpha[i + (int64_t)p * ld];
            s += (a * za - 0.5 * (1. + a * a * inv_diag) * zk) * inv_diag;
        }
    }
    s = block_sum_1024(s, sh);
    if (threadIdx.x == 0) *out = s;
}

// gp.hpp:347: sum over i, p of -0.5 alpha^2 inv_diag - 0.5 log(inv_diag) - 0.5 log(2 pi)
__global__ void __launch_bounds__(1024)
loo_value_kernel(const double* __restrict__ Kinv, int64_t ld, int64_t N, const double* __restrict__ alpha, int P, double* __restrict__ out)
{
    __shared__ double sh[32];
    double s = 0.0;
    for (int64_t i = threadIdx.x; i < N; i += 1024) {
        const double inv_diag = 1.0 / Kinv[i + i * ld];
        for (int p = 0; p < P; ++p) {
            const double a = alpha[i + (int64_t)p * ld];
            s += -0.5 * a * a * inv_diag - 0.5 * log(inv_diag) - 0.5 * log(2.0 * M_PI);
        }
    }
    s = block_sum_1024(s, sh);
    if (threadIdx.x == 0) *out = s;
}

// part[ks][i + p*ld] = sum over the ks-th slice of k of Kinv[i, k] Y[k, p]   (Kinv symmetric-full; coalesced over i)
constexpr int KSLICES = 32;
__global__ void __launch_bounds__(256)
kinv_obs_kernel(const double* __restrict__ Kinv, int64_t ld, int64_t N, const double* __restrict__ Y, int P, double* __restrict__ part)
{
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int ks = blockIdx.y;
    const int64_t per = (N + KSLICES - 1) / KSLICES;
    const int64_t k0 = ks * per, k1 = (k0 + per < N) ? k0 + per : N;
    if (i >= N) return;
    for (int p = 0; p < P; ++p) {
        double s = 0.0;
        const double* y = Y + (int64_t)p * ld;
        for (int64_t k = k0; k < k1; ++k) s = fma(Kinv[i + k * ld], y[k], s);
        part[((int64_t)ks * P + p) * ld + i] = s;
    }
}
__global__ void __launch_bounds__(256)
kinv_obs_reduce_kernel(const double* __restrict__ part, int64_t ld, int64_t N, int P, double* __restrict__ out)
{
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= N) return;
    for (int p = 0; p < P; ++p) {
        double s = 0.0;
        for (int ks = 0; ks < KSLICES; ++ks) s += part[((int64_t)ks * P + p) * ld + i];
        out[i + (int64_t)p * N] = s; // N x P column-major, unpadded
    }
}

// part[b] = sum over a fixed slice of the elements (i, j < N) of (sum_p alpha_ip alpha_jp - Kinv_ij) dK_ij
constexpr int WDOT_BLOCKS = 1024;
__global__ void __launch_bounds__(256)
wdot_kernel(const double* __restrict__ Kinv, const double* __restrict__ dK, int64_t ld, int64_t N, const double* __restrict__ alpha, int P,
    double* __restrict__ part)
{
    __shared__ double red[8];
    double s = 0.0;
    for (int64_t j = blockIdx.x; j < N; j += WDOT_BLOCKS)
        for (int64_t i = threadIdx.x; i < N; i += 256) {
            double w = -Kinv[i + j * ld];
            for (int p = 0; p < P; ++p) w = fma(alpha[i + (int64_t)p * ld], alpha[j + (int64_t)p * ld], w);
            s = fma(w, dK[i + j * ld], s);
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
__global__ void __launch_bounds__(256)
wdot_reduce_kernel(const double* __restrict__ part, double* __restrict__ out)
{
    __shared__ double red[8];
    double s = 0.0;
    for (int b = threadIdx.x; b < WDOT_BLOCKS; b += 256) s += part[b];
    s = lb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        *out = 0.5 * t;
    }
}

int ensure_sym_kinv(lb_gp* h)
{
    int rc;
    if (!h->kinv_valid && (rc = lb_launch_kinv(h))) return rc;
    if (!h->kinv_sym) {
        if ((rc = lb_launch_symmetrize(h, h->dKinv.get()))) return rc;
        h->kinv_sym = true;
    }
    return LB_OK;
}

} // namespace

int lb_launch_loo_value(lb_gp* h, double* dOut)
{
    int rc;
    if (!h->kinv_valid && (rc = lb_launch_kinv(h))) return rc;
    loo_value_kernel<<<1, 1024, 0, h->stream>>>(h->dKinv.get(), h->Np, h->N, h->dAlpha, h->P, dOut);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_loo_grad(lb_gp* h, int optimize_noise, double* dGrad)
{
    int rc = ensure_sym_kinv(h);
    if (rc) return rc;
    const int64_t Np = h->Np;
    const int T = (int)(Np / LB_TILE);
    const int nh = h->n_hparams + (optimize_noise ? 1 : 0);
    if ((rc = h->dWork.resize(h, sizeof(double) * Np * Np))) return rc;
    if ((rc = lb_ensure_scratch(h, sizeof(double) * (size_t)(h->P + 1) * T * Np))) return rc;
    LB_CUDA(cudaFuncSetAttribute(loo_zeta_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::PIPE_BYTES));
    double* part_zk = h->dScratch.get();
    double* part_za = h->dScratch.get() + (int64_t)T * Np;
    LbProfScope ps(h, h->stream, LB_PC_GRAD);
    for (int q = 0; q < nh; ++q) {
        dim3 g1((unsigned)Np, (unsigned)((Np + 255) / 256));
        dk_build_kernel<<<g1, 256, 0, h->stream>>>(h->dXs, Np, h->N, h->kp, q, h->n_hparams, h->dWork.get());
        loo_zeta_kernel<<<T * T, Cfg::THREADS, Cfg::PIPE_BYTES, h->stream>>>(h->dKinv.get(), h->dWork.get(), Np, h->dAlpha, h->P, T, part_zk,
            part_za);
        loo_grad_reduce_kernel<<<1, 1024, 0, h->stream>>>(h->dKinv.get(), Np, h->N, h->dAlpha, h->P, T, part_zk, part_za, dGrad + q);
        h->launches += 3;
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Likelihood gradient wrt the entries of the SE-ARD Lambda matrix (squared_exp_ard.hpp:119-122; gp.hpp:299-308):
//   g_q = sum_{i >= j} w_ij dK_q,ij (1/2 on the diagonal) = 1/2 sum_{all i,j} (alpha alpha^T - K^-1)_ij dK_q,ij
// one dK build + one weighted reduction per entry (k > 0 is a rarely used option; the ell / sigma_f / noise entries come
// from the fused grad_kernel).
int lb_launch_grad_lambda(lb_gp* h, double* dGrad)
{
    int rc = ensure_sym_kinv(h);
    if (rc) return rc;
    const int64_t Np = h->Np;
    if ((rc = h->dWork.resize(h, sizeof(double) * Np * Np))) return rc;
    if ((rc = lb_ensure_scratch(h, sizeof(double) * WDOT_BLOCKS))) return rc;
    const int Dr = h->kp.Draw;
    for (int q = Dr; q < Dr + Dr * h->kp.klam; ++q) {
        dim3 g1((unsigned)Np, (unsigned)((Np + 255) / 256));
        dk_build_kernel<<<g1, 256, 0, h->stream>>>(h->dXs, Np, h->N, h->kp, q, h->n_hparams, h->dWork.get());
        wdot_kernel<<<WDOT_BLOCKS, 256, 0, h->stream>>>(h->dKinv.get(), h->dWork.get(), Np, h->N, h->dAlpha, h->P, h->dScratch.get());
        wdot_reduce_kernel<<<1, 256, 0, h->stream>>>(h->dScratch.get(), dGrad + q);
        h->launches += 3;
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// dOut: N x P column-major (unpadded) = K^-1 * obs_mean
int lb_launch_kinv_obs(lb_gp* h, double* dOut)
{
    int rc = ensure_sym_kinv(h);
    if (rc) return rc;
    if ((rc = lb_ensure_scratch(h, sizeof(double) * (size_t)KSLICES * h->P * h->Np))) return rc;
    dim3 g((unsigned)((h->N + 255) / 256), KSLICES);
    kinv_obs_kernel<<<g, 256, 0, h->stream>>>(h->dKinv.get(), h->Np, h->N, h->dY, h->P, h->dScratch.get());
    kinv_obs_reduce_kernel<<<(unsigned)((h->N + 255) / 256), 256, 0, h->stream>>>(h->dScratch.get(), h->Np, h->N, h->P, dOut);
    h->launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
