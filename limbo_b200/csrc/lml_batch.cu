// limbo_b200/csrc/lml_batch.cu — the log marginal likelihood and its kernel hyper-parameter gradient at R kernel states in one
// launch (lb_lml_grad_batch): what model::gp::KernelLFOpt evaluates per Rprop step (model/gp/kernel_lf_opt.hpp:77-92), for
// every restart of opt::ParallelRepeater at once.
//
// At the sizes the reference's loop runs (N of a few hundred) the single path (kbuild, potrf, trsv, lml.cu) is a dozen launches
// of 128-row tiles that occupy a handful of SMs.  Here one CTA evaluates one vector end to end, and a persistent grid of
// min(R, resident CTAs) walks the vectors:
//   1. stage x / ell and A^T x (SE-ARD) resp. x from the handle's raw samples        lb_staged_coord (common.cuh)
//   2. lower triangle of K, noise + 1e-8 on the diagonal                              kbuild.cu's functor and jitter
//   3. right-looking Cholesky in place, first non-positive pivot recorded            gp.hpp:565
//   4. alpha = K^-1 obs_mean by forward / backward substitution, log det, likelihood  gp.hpp:267-282
//   5. L^-1 in place (dtrti2's column order), K^-1 = L^-T L^-1 in place (dlauu2's), one sweep over i >= j of
//      w_ij dk_ij / dtheta with the pair derivatives of grad_kernel (lml.cu), then one per 8 SE-ARD ell / Lambda entries
//      over w_ij k_ij kept in K^-1's place                                             gp.hpp:285-311
// The vector's matrix, staged coordinates and alpha live in shared memory up to N = 128 and otherwise in a pooled per-CTA
// workspace (at N = 200, D = 6 about 336 KB per CTA, 44 MB over 132 CTAs: of the order of the 50 MB L2; its hit rate is not
// measured); the code is the same, through generic pointers.  Every reduction runs in a fixed
// order over a thread assignment that depends on N only, so a vector's result does not depend on R or on its place in the batch.
#include "common.cuh"
#include <cstring>
#include <math_constants.h>

namespace {

constexpr int NT = 256, NW = NT / 32;
constexpr int GCH = 8;                  // SE-ARD ell / Lambda gradient entries per sweep
constexpr int SMEM_MAX_N = 128;         // largest N whose workspace goes to shared memory
constexpr int SMEM_BYTES_MAX = 200 * 1024;

struct LmlBatchArgs {
    const double* X;   // D x ldx raw samples (SoA)
    int64_t ldx;
    const double* Y;   // ldx x P obs_mean (column-major)
    int N, Draw, klam, De, P;
    const double* prm; // R x stride: sf2, l, c1, c2, noise, 0, 0, 0, 1/ell (Draw), Lambda (Draw x klam column-major)
    int stride;
    int R, nh, optimize_noise, want_grad;
    double* lik;       // R
    double* grad;      // R x nh, or NULL
    int* info;         // R, or NULL
    double* ws;        // per-CTA workspace of ws_stride doubles, or NULL (shared memory)
    int64_t ws_stride;
    int ld;            // leading dimension of the vector's matrix (odd: conflict-free row walks in shared memory)
};

__host__ __device__ inline int64_t ws_doubles(int N, int ld, int De, int P)
{
    return (int64_t)ld * N + (int64_t)De * N + 2 * (int64_t)P * N + N;
}

// fixed-order CTA sum of NV values per thread; the totals land in out[] (shared), visible to every thread on return
template <int NV>
__device__ __forceinline__ void block_sum(double (&v)[NV], double (*red)[GCH], double* out)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int f = 0; f < NV; ++f) {
        const double s = lb_warp_sum(v[f]);
        if (lane == 0) red[warp][f] = s;
    }
    __syncthreads();
    if (threadIdx.x < NV) {
        double s = 0.0;
        for (int w = 0; w < NW; ++w) s += red[w][threadIdx.x];
        out[threadIdx.x] = s;
    }
    __syncthreads();
}

template <int KID>
__global__ void __launch_bounds__(NT)
lml_batch_kernel(const LmlBatchArgs a)
{
    extern __shared__ __align__(16) double smem[];
    __shared__ KernParams skp;
    __shared__ double red[NW][GCH];
    __shared__ double tot[GCH];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = a.N, ld = a.ld, De = a.De, P = a.P;
    double* A = a.ws ? a.ws + (int64_t)blockIdx.x * a.ws_stride : smem;
    double* xs = A + (int64_t)ld * N;   // De x N staged coordinates
    double* yv = xs + (int64_t)De * N;  // P x N: obs_mean, then alpha
    double* zv = yv + (int64_t)P * N;   // P x N: forward solution
    double* tmp = zv + (int64_t)P * N;  // N
    constexpr bool ard = (KID == LB_K_SE_ARD);

    for (int r = blockIdx.x; r < a.R; r += gridDim.x) {
        const double* pr = a.prm + (int64_t)r * a.stride;
        __syncthreads(); // the previous vector's readers of skp / the workspace are done
        if (tid == 0) {
            skp.id = KID;
            skp.D = De;
            skp.Draw = a.Draw;
            skp.klam = a.klam;
            skp.sf2 = pr[0];
            skp.l = pr[1];
            skp.c1 = pr[2];
            skp.c2 = pr[3];
            skp.noise = pr[4];
            skp.lambda = a.klam > 0 ? pr + 8 + a.Draw : nullptr;
        }
        for (int d = tid; d < a.Draw; d += NT) skp.inv_ell[d] = ard ? pr[8 + d] : 1.0;
        __syncthreads();
        const KernParams& kp = skp;

        // 1. staged coordinates, obs_mean
        for (int idx = tid; idx < De * N; idx += NT) {
            const int d = idx / N, i = idx - d * N;
            xs[idx] = lb_staged_coord(kp, d, [&](int q) { return a.X[(int64_t)q * a.ldx + i]; });
        }
        for (int idx = tid; idx < P * N; idx += NT) {
            const int p = idx / N, i = idx - p * N;
            yv[idx] = a.Y[(int64_t)p * a.ldx + i];
        }
        __syncthreads();
        // 2. lower triangle of K (kbuild.cu's functor and diagonal)
        for (int j = warp; j < N; j += NW)
            for (int i = j + lane; i < N; i += 32) {
                double z = 0.0;
                for (int d = 0; d < De; ++d) {
                    const double q = xs[(int64_t)d * N + i] - xs[(int64_t)d * N + j];
                    z = fma(q, q, z);
                }
                double k = lb_kernel_from_z(KID, z, kp);
                if (i == j) k += kp.noise + 1e-8; // kernel.hpp:83
                A[i + (int64_t)j * ld] = k;
            }
        __syncthreads();
        // 3. Cholesky, column by column
        int fail = 0;
        for (int k = 0; k < N; ++k) {
            const double d = A[k + (int64_t)k * ld];
            if (!(d > 0.0)) { fail = k + 1; break; } // every thread reads the same value: a uniform exit
            const double lkk = sqrt(d);
            double* colk = A + (int64_t)k * ld;
            for (int i = k + 1 + tid; i < N; i += NT) colk[i] /= lkk;
            __syncthreads();
            if (tid == 0) colk[k] = lkk;
            for (int j = k + 1 + warp; j < N; j += NW) {
                const double ljk = colk[j];
                double* colj = A + (int64_t)j * ld;
                for (int i = j + lane; i < N; i += 32) colj[i] = fma(-colk[i], ljk, colj[i]);
            }
            __syncthreads();
        }
        if (fail) {
            if (tid == 0) {
                a.lik[r] = CUDART_NAN;
                if (a.info) a.info[r] = fail;
            }
            if (a.grad)
                for (int q = tid; q < a.nh; q += NT) a.grad[(int64_t)r * a.nh + q] = CUDART_NAN;
            continue;
        }
        // 4. alpha: L z = y, L^T alpha = z (alpha over y, the forward solution in zv); log det and y^T alpha
        for (int p = 0; p < P; ++p) {
            double* y = yv + (int64_t)p * N;
            double* z = zv + (int64_t)p * N;
            for (int k = 0; k < N; ++k) {
                const double t = y[k] / A[k + (int64_t)k * ld];
                if (tid == 0) z[k] = t;
                for (int i = k + 1 + tid; i < N; i += NT) y[i] = fma(-A[i + (int64_t)k * ld], t, y[i]);
                __syncthreads();
            }
            for (int k = N - 1; k >= 0; --k) {
                const double t = z[k] / A[k + (int64_t)k * ld];
                if (tid == 0) y[k] = t;
                for (int i = tid; i < k; i += NT) z[i] = fma(-A[k + (int64_t)i * ld], t, z[i]);
                __syncthreads();
            }
        }
        {
            double v[2] = {0.0, 0.0};
            for (int i = tid; i < N; i += NT) {
                v[0] += log(A[i + (int64_t)i * ld]);
                for (int p = 0; p < P; ++p) v[1] = fma(a.Y[(int64_t)p * a.ldx + i], yv[(int64_t)p * N + i], v[1]);
            }
            block_sum<2>(v, red, tot);
            if (tid == 0) {
                const double logdet = 2.0 * tot[0]; // gp.hpp:274
                a.lik[r] = -0.5 * tot[1] - 0.5 * logdet - 0.5 * (double)N * log(2.0 * M_PI); // gp.hpp:279
                if (a.info) a.info[r] = 0;
            }
        }
        if (!a.want_grad) continue;

        // 5a. L^-1 in place (dtrti2, lower, non-unit): column j from the inverted trailing block
        for (int j = N - 1; j >= 0; --j) {
            const double inv = 1.0 / A[j + (int64_t)j * ld];
            for (int i = j + 1 + tid; i < N; i += NT) tmp[i] = A[i + (int64_t)j * ld];
            __syncthreads();
            if (tid == 0) A[j + (int64_t)j * ld] = inv;
            for (int i = j + 1 + tid; i < N; i += NT) {
                double s = 0.0;
                for (int c = j + 1; c <= i; ++c) s = fma(A[i + (int64_t)c * ld], tmp[c], s);
                A[i + (int64_t)j * ld] = -inv * s;
            }
            __syncthreads();
        }
        // 5b. K^-1 = L^-T L^-1 in place (dlauu2): row i of the lower triangle from the rows k >= i of L^-1
        for (int i = 0; i < N; ++i) {
            const double* coli = A + (int64_t)i * ld;
            for (int j = warp; j <= i; j += NW) {
                const double* colj = A + (int64_t)j * ld;
                double s = 0.0;
                for (int k = i + lane; k < N; k += 32) s = fma(coli[k], colj[k], s);
                s = lb_warp_sum(s);
                if (lane == 0) tmp[j] = s;
            }
            __syncthreads();
            for (int j = tid; j <= i; j += NT) A[i + (int64_t)j * ld] = tmp[j];
            __syncthreads();
        }
        // 5c. sum_{i >= j} w_ij dk_ij / dtheta, w = alpha alpha^T - K^-1, half weight on the diagonal (gp.hpp:293-308)
        double g[3] = {0.0, 0.0, 0.0}; // sigma_f, length scale (isotropic kernels), noise
        for (int j = warp; j < N; j += NW)
            for (int i = j + lane; i < N; i += 32) {
                double* kij = A + i + (int64_t)j * ld;
                double w = -*kij;
                for (int p = 0; p < P; ++p) w = fma(yv[(int64_t)p * N + i], yv[(int64_t)p * N + j], w);
                if (i == j) {
                    w *= 0.5;
                    g[2] = fma(w, 2.0 * kp.noise, g[2]); // kernel.hpp:90-93
                }
                double z = 0.0;
                for (int d = 0; d < De; ++d) {
                    const double q = xs[(int64_t)d * N + i] - xs[(int64_t)d * N + j];
                    z = fma(q, q, z);
                }
                double g0, g1;
                lb_kernel_grad_pair<KID>(z, kp, g0, g1);
                if (ard) *kij = w * g0; // w k, for the ell / Lambda sweeps
                else g[1] = fma(w, g0, g[1]);
                g[0] = fma(w, g1, g[0]);
            }
        block_sum<3>(g, red, tot);
        double* gout = a.grad + (int64_t)r * a.nh;
        const int nk = a.nh - (a.optimize_noise ? 1 : 0);
        if (tid == 0) {
            gout[nk - 1] = tot[0];
            if (!ard) gout[0] = tot[1];
            if (a.optimize_noise) gout[nk] = tot[2];
        }
        if (ard) {
            // entry q < Draw: (x_i - x_j)_q^2 / ell_q^2 (squared_exp_ard.hpp:117); Lambda entry A(li, lj):
            // -(x_i - x_j)^T A(:, lj) (x_i - x_j)_li (squared_exp_ard.hpp:119-122)
            const int nent = nk - 1;
            for (int q0 = 0; q0 < nent; q0 += GCH) {
                double acc[GCH];
#pragma unroll
                for (int f = 0; f < GCH; ++f) acc[f] = 0.0;
                for (int j = warp; j < N; j += NW)
                    for (int i = j + 1 + lane; i < N; i += 32) {
                        const double wk = A[i + (int64_t)j * ld];
#pragma unroll
                        for (int f = 0; f < GCH; ++f) {
                            const int q = q0 + f;
                            if (q < nent) {
                                double feat;
                                if (q < a.Draw) {
                                    const double t = xs[(int64_t)q * N + i] - xs[(int64_t)q * N + j];
                                    feat = t * t;
                                }
                                else {
                                    const int e = q - a.Draw, lj = e / a.Draw, li = e - lj * a.Draw;
                                    const double proj = xs[(int64_t)(a.Draw + lj) * N + i] - xs[(int64_t)(a.Draw + lj) * N + j];
                                    const double raw = (xs[(int64_t)li * N + i] - xs[(int64_t)li * N + j]) / kp.inv_ell[li];
                                    feat = -proj * raw;
                                }
                                acc[f] = fma(wk, feat, acc[f]);
                            }
                        }
                    }
                block_sum<GCH>(acc, red, tot);
                if (tid < GCH && q0 + tid < nent) gout[q0 + tid] = tot[tid];
            }
        }
    }
}

LbOncePerDevice g_attr_once;
int set_attrs()
{
    if (!g_attr_once.need()) return LB_OK;
    LB_CUDA(cudaFuncSetAttribute(lml_batch_kernel<LB_K_SE_ARD>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES_MAX));
    LB_CUDA(cudaFuncSetAttribute(lml_batch_kernel<LB_K_MATERN52>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES_MAX));
    LB_CUDA(cudaFuncSetAttribute(lml_batch_kernel<LB_K_MATERN32>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES_MAX));
    LB_CUDA(cudaFuncSetAttribute(lml_batch_kernel<LB_K_EXP>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES_MAX));
    return LB_OK;
}

template <int KID>
int launch(const LmlBatchArgs& a0, StreamTemps& tmp, cudaStream_t st, long long* launches)
{
    LmlBatchArgs a = a0;
    a.ld = a.N | 1;
    const int64_t per = ws_doubles(a.N, a.ld, a.De, a.P);
    const size_t sbytes = sizeof(double) * (size_t)per;
    const bool in_smem = a.N <= SMEM_MAX_N && sbytes <= (size_t)SMEM_BYTES_MAX;
    int dev = 0, sms = 0, occ = 0;
    LB_CUDA(cudaGetDevice(&dev));
    LB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    LB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, lml_batch_kernel<KID>, NT, in_smem ? sbytes : 0));
    if (occ < 1) occ = 1;
    // the global workspace: one CTA per SM bounds it at SMs x per doubles
    const int64_t resident = (int64_t)sms * (in_smem ? occ : 1);
    const int grid = (int)std::min<int64_t>(a.R, resident);
    a.ws = nullptr;
    a.ws_stride = 0;
    if (!in_smem) {
        a.ws_stride = (per + 31) / 32 * 32;
        int rc = tmp.alloc(sizeof(double) * (size_t)a.ws_stride * grid, &a.ws);
        if (rc) return rc;
    }
    lml_batch_kernel<KID><<<grid, NT, in_smem ? sbytes : 0, st>>>(a);
    ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

} // namespace

int lb_launch_lml_batch(cudaStream_t st, StreamTemps& tmp, const KernParams* kps, const double* hparams, int n_hparams, int R,
    const double* dX, int64_t ldx, const double* dY, int N, int P, int nh, int optimize_noise, double* dLik, double* dGrad, int* dInfo,
    long long* launches)
{
    int rc = set_attrs();
    if (rc) return rc;
    const int kernel_id = kps[0].id, Draw = kps[0].Draw, klam = kps[0].klam;
    // the rows of LmlBatchArgs::prm
    const int stride = kernel_id == LB_K_SE_ARD ? 8 + Draw * (1 + klam) : 8;
    std::vector<double> prm((size_t)R * stride, 0.0);
    for (int r = 0; r < R; ++r) {
        const KernParams& kp = kps[r];
        double* o = prm.data() + (size_t)r * stride;
        o[0] = kp.sf2;
        o[1] = kp.l;
        o[2] = kp.c1;
        o[3] = kp.c2;
        o[4] = kp.noise;
        if (kernel_id == LB_K_SE_ARD) {
            std::memcpy(o + 8, kp.inv_ell, sizeof(double) * Draw);
            std::memcpy(o + 8 + Draw, hparams + (size_t)r * n_hparams + Draw, sizeof(double) * Draw * klam);
        }
    }
    double* dPrm = nullptr;
    if ((rc = tmp.alloc(sizeof(double) * prm.size(), &dPrm))) return rc;
    LB_CUDA(cudaMemcpyAsync(dPrm, prm.data(), sizeof(double) * prm.size(), cudaMemcpyHostToDevice, st));
    LmlBatchArgs a{};
    a.X = dX; a.ldx = ldx; a.Y = dY; a.N = N; a.Draw = Draw; a.klam = klam; a.De = Draw + klam; a.P = P;
    a.prm = dPrm; a.stride = stride; a.R = R; a.nh = nh; a.optimize_noise = optimize_noise; a.want_grad = dGrad != nullptr;
    a.lik = dLik; a.grad = dGrad; a.info = dInfo;
    switch (kernel_id) {
    case LB_K_SE_ARD: return launch<LB_K_SE_ARD>(a, tmp, st, launches);
    case LB_K_MATERN52: return launch<LB_K_MATERN52>(a, tmp, st, launches);
    case LB_K_MATERN32: return launch<LB_K_MATERN32>(a, tmp, st, launches);
    default: return launch<LB_K_EXP>(a, tmp, st, launches);
    }
}
