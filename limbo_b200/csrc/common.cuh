// limbo_b200/csrc/common.cuh — shared declarations for the sm_90a GP backend.
//
// Data layout in HBM (see DESIGN.md §3):
//   * every N-sized dimension is padded to Np = roundup(N, 128); the padded
//     part of K is the identity, so the Cholesky factor, the triangular
//     solves, K^-1 and log|K| of the padded system restrict exactly to those
//     of the N x N system and no kernel needs edge predication;
//   * X  : D x Np "SoA" (dimension-major) so 128-point blocks of one input
//     dimension are 1 KB contiguous runs (TMA bulk-copy friendly);
//   * K/L: Np x Np column-major (Eigen::MatrixXd's layout, gp.hpp:553), the
//     factor overwrites the lower triangle in place;
//   * invD: T blocks of 128 x 128 (column-major, lower) = inverses of the
//     diagonal blocks of L, produced by the panel factorisation and reused by
//     every triangular solve.
#pragma once
#include <cuda_runtime.h>
#include <array>
#include <cfloat>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <vector>

#define LB_TILE 128
#define LB_NEV 6 // events per handle: Cholesky fork / panel x2 / a-update x2 / join (the panel query's fork and joins reuse 0..3)

// ---- status codes (include/limbo_b200.h) ----------------------------------
#define LB_OK 0
#define LB_ERR_ARG (-1)
#define LB_ERR_CUDA (-2)
#define LB_ERR_STATE (-3)
#define LB_ERR_ALLOC (-4)
#define LB_ERR_UNSUPPORTED (-5)
#define LB_ERR_TIMEOUT (-6)

#define LB_CUDA(call)                                                                   \
    do {                                                                                \
        cudaError_t e__ = (call);                                                       \
        if (e__ != cudaSuccess) {                                                       \
            lb_set_last_cuda_error(e__, __FILE__, __LINE__);                            \
            return LB_ERR_CUDA;                                                         \
        }                                                                               \
    } while (0)

void lb_set_last_cuda_error(cudaError_t e, const char* file, int line);

enum { LB_K_SE_ARD = 0, LB_K_MATERN52 = 1, LB_K_MATERN32 = 2, LB_K_EXP = 3 };
#define LB_MAX_D 64
#define LB_MAX_LAMBDA 4 // columns of the SE-ARD Lambda matrix (Params::kernel_squared_exp_ard::k)
#define LB_MAX_HPARAMS (LB_MAX_D * (1 + LB_MAX_LAMBDA) + 2) // SE-ARD: log ell, Lambda columns, log sigma_f, (noise)

// Kernel parameters passed by value to device code.
struct KernParams {
    int id;
    int D;
    double sf2;      // exp(2 p_last)                    squared_exp_ard.hpp:104
    double l;        // isotropic length scale            matern_five_halves.hpp:100
    double noise;    // kernel/kernel.hpp:76-79
    double inv_ell[LB_MAX_D]; // SE-ARD: 1/exp(p_d)
    double c1;       // Matern: sqrt(5)/l resp. sqrt(3)/l ; Exp: 1/l^2   (host-precomputed, saves a divide per pair)
    double c2;       // Matern-5/2: 5/(3 l^2)
    // SE-ARD with k > 0 (squared_exp_ard.hpp:109-126,142-146): z = d^T (A A^T + diag(ell^-2)) d = |W^T d|^2 with
    // W = [diag(1/ell) | A].  The staged samples carry D = Draw + klam coordinates (x/ell, A^T x), so every kernel that
    // consumes the staged tiles is unchanged; only the staging and the gradient wrt A know about A.
    int Draw;        // input dimension of the caller's points
    int klam;        // number of columns of A
    const double* lambda; // device, Draw x klam column-major (nullptr when klam == 0)
};

// ---------------------------------------------------------------------------
// Device-side kernel functor: value from the (scaled) squared distance.
//   SE-ARD : z = sum_d ((x_d - y_d)/ell_d)^2  (X is pre-scaled by 1/ell_d)
//   others : z = sum_d (x_d - y_d)^2          (raw X)
// Operation order after z follows the reference functors so that the result
// differs from the Eigen path only by the rounding of z itself.
// ---------------------------------------------------------------------------
__device__ __forceinline__ double lb_kernel_from_z(int id, double z, double sf2, double l)
{
    switch (id) {
    case LB_K_SE_ARD: // squared_exp_ard.hpp:150
        return sf2 * exp(-0.5 * z);
    case LB_K_MATERN52: { // matern_five_halves.hpp:104-113
        double d = sqrt(z);
        double d_sq = d * d;
        double l_sq = l * l;
        double term1 = sqrt(5.0) * d / l;
        double term2 = 5. * d_sq / (3. * l_sq);
        return sf2 * (1 + term1 + term2) * exp(-term1);
    }
    case LB_K_MATERN32: { // matern_three_halves.hpp:102-108
        double d = sqrt(z);
        double term = sqrt(3.0) * d / l;
        return sf2 * (1 + term) * exp(-term);
    }
    default: { // exp.hpp:94-99
        double r = z / (l * l);
        return sf2 * exp(-0.5 * r);
    }
    }
}

// exp(t) for t <= 0, branch-free: n = rint(t log2 e), r = t - n ln 2 (two-term), degree-13 Taylor in |r| <= 0.347
// (truncation < 5e-18), 2^n by an exponent-field add.  Relative error < 3e-16 for t >= -708 (tests/test_gpu_tf32.py),
// exactly 0 below (where the reference's std::exp returns a denormal < 2.3e-308).  ~18 fp64 instructions and no slow-path
// branch, so the 32 evaluations a thread holds interleave: the kernel-evaluation loops (K build, K*, gradient) are bound
// by the fp64 pipe whenever they are not bound by HBM.
__device__ __forceinline__ double lb_exp_nonpos(double t)
{
    const double MAGIC = 6755399441055744.0; // 1.5 * 2^52
    double fn = fma(t, 1.4426950408889634074, MAGIC);
    const int n = __double2loint(fn);
    fn -= MAGIC;
    double r = fma(fn, -6.93147180369123816490e-01, t);
    r = fma(fn, -1.90821492927058770002e-10, r);
    double p = 1.6059043836821614599e-10; // 1/13!
    p = fma(p, r, 2.0876756987868098979e-09);
    p = fma(p, r, 2.5052108385441718775e-08);
    p = fma(p, r, 2.7557319223985890653e-07);
    p = fma(p, r, 2.7557319223985890653e-06);
    p = fma(p, r, 2.4801587301587301587e-05);
    p = fma(p, r, 1.9841269841269841270e-04);
    p = fma(p, r, 1.3888888888888888889e-03);
    p = fma(p, r, 8.3333333333333333333e-03);
    p = fma(p, r, 4.1666666666666666667e-02);
    p = fma(p, r, 1.6666666666666666667e-01);
    p = fma(p, r, 0.5);
    p = fma(p, r, 1.0);
    p = fma(p, r, 1.0);
    const int hi = __double2hiint(p) + (n << 20);
    const double e = __hiloint2double(hi, __double2loint(p));
    return t < -708.0 ? 0.0 : e;
}

// Same functors with the per-pair divisions and the square root replaced by host-precomputed reciprocals and a
// branch-free rsqrt (<= a few ulp from the reference's operation order; K stays within 1e-15 of the Eigen path).
__device__ __forceinline__ double lb_rsqrt_nr(double x)
{
    double r;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    const double h = 0.5 * x;
    r = fma(r, fma(-h * r, r, 0.5), r);
    r = fma(r, fma(-h * r, r, 0.5), r);
    return r;
}
// d = sqrt(z) for the Matern functors.  rsqrt.approx.ftz flushes a subnormal z to zero (seed +inf, NaN after the Newton steps),
// so z < DBL_MIN (d < 1.5e-154, c1 d < 1e-150) gives d = 0, which is exact to rounding in every formula that uses d.
__device__ __forceinline__ double lb_dist_from_z(double z)
{
    return (z >= DBL_MIN) ? z * lb_rsqrt_nr(z) : 0.0;
}
__device__ __forceinline__ double lb_kernel_from_z(int id, double z, const KernParams& kp)
{
    switch (id) {
    case LB_K_SE_ARD:
        return kp.sf2 * exp(-0.5 * z); // libm here: the SE-ARD K build is HBM bound with it (0.85 of peak) and compute bound (0.67) with lb_exp_nonpos
    case LB_K_MATERN52: {
        // sigma_f^2 (1 + c1 d + c2 d^2) exp(-c1 d) with d^2 = z and sigma_f^2 folded into the polynomial (two FMAs instead of
        // two products and two sums; <= 2 ulp from the reference's operation order, matern_five_halves.hpp:106-112): the
        // Matern K build is bound by the fp64 pipe, not by HBM (~45 fp64 instructions per element)
        const double d = lb_dist_from_z(z);
        const double term1 = kp.c1 * d;
        return fma(kp.c2 * kp.sf2, z, fma(kp.sf2, term1, kp.sf2)) * lb_exp_nonpos(-term1);
    }
    case LB_K_MATERN32: {
        const double d = lb_dist_from_z(z);
        const double term = kp.c1 * d;
        return fma(kp.sf2, term, kp.sf2) * lb_exp_nonpos(-term);
    }
    default:
        return kp.sf2 * exp(-0.5 * (z * kp.c1));
    }
}

// Normalised kernel value (sigma_f^2 = 1) from the (scaled) squared distance, kernel id as a template parameter.
template <int KID>
__device__ __forceinline__ double lb_unit_kernel_from_z(double z, const KernParams& kp)
{
    if (KID == LB_K_SE_ARD) return lb_exp_nonpos(-0.5 * z);
    if (KID == LB_K_MATERN52) {
        const double d = lb_dist_from_z(z);
        const double term1 = kp.c1 * d;
        return (1 + term1 + kp.c2 * (d * d)) * lb_exp_nonpos(-term1);
    }
    if (KID == LB_K_MATERN32) {
        const double d = lb_dist_from_z(z);
        const double term = kp.c1 * d;
        return (1 + term) * lb_exp_nonpos(-term);
    }
    return lb_exp_nonpos(-0.5 * (z * kp.c1));
}

// The pair derivatives the likelihood gradient weights (lml.cu grad_kernel, lml_batch.cu), from the (scaled) squared distance:
//   SE-ARD   g0 = k (the ell / Lambda entries multiply it by their pair factor), g1 = dk / dlog sigma_f = 2k  squared_exp_ard.hpp:127-135
//   others   g0 = dk / dlog l, g1 = dk / dlog sigma_f      matern_five_halves.hpp:115-133, matern_three_halves.hpp:110-124, exp.hpp:101-110
// with the branch-free lb_exp_nonpos (<= 3e-16 relative, inside the 1e-9 bar of the gradient).
template <int KID>
__device__ __forceinline__ void lb_kernel_grad_pair(double zz, const KernParams& kp, double& g0, double& g1)
{
    if (KID == LB_K_SE_ARD) {
        const double k = kp.sf2 * lb_exp_nonpos(-0.5 * zz);
        g0 = k;
        g1 = 2.0 * k;
    }
    else if (KID == LB_K_MATERN52) {
        const double d = sqrt(zz), d_sq = d * d, l_sq = kp.l * kp.l;
        const double term1 = sqrt(5.0) * d / kp.l;
        const double term2 = 5. * d_sq / (3. * l_sq);
        const double r = lb_exp_nonpos(-term1);
        g0 = kp.sf2 * (r * term1 * (1 + term1 + term2) + (-term1 - 2. * term2) * r);
        g1 = 2 * kp.sf2 * (1 + term1 + term2) * r;
    }
    else if (KID == LB_K_MATERN32) {
        const double d = sqrt(zz);
        const double term = sqrt(3.0) * d / kp.l;
        const double r = lb_exp_nonpos(-term);
        g0 = kp.sf2 * (-term * r + (1 + term) * term * r);
        g1 = 2 * kp.sf2 * (1 + term) * r;
    }
    else {
        const double r = zz / (kp.l * kp.l);
        const double k = kp.sf2 * lb_exp_nonpos(-0.5 * r);
        g0 = r * k;
        g1 = 2 * k;
    }
}

// expected improvement of mu over f_max + jitter, 0 when sigma < 1e-10: ei.hpp:92-115, and the factor eci.hpp:86-106 weights
__device__ __forceinline__ double lb_ei_factor(double mu, double s2, double f_max, double jitter)
{
    double sigma = sqrt(s2);
    if (sigma < 1e-10) return 0.0;
    double X = mu - f_max - jitter;
    double Z = X / sigma;
    double phi = exp(-0.5 * (Z * Z)) / sqrt(2.0 * M_PI);
    double Phi = 0.5 * erfc(-Z / sqrt(2.0));
    return X * Phi + sigma * phi;
}

// acquisition value per candidate (FirstElem aggregator, bo_base.hpp:99-105)
//   acq_id 0: UCB / GP_UCB  mu + p0 * sqrt(s2)                 ucb.hpp:89, gp_ucb.hpp:102
//   acq_id 1: EI  (p0 = f_max, p1 = jitter)                    ei.hpp:92-115
__device__ __forceinline__ double lb_acq_value(int acq_id, double mu, double s2, double p0, double p1)
{
    if (acq_id == 0) return mu + p0 * sqrt(s2);
    return lb_ei_factor(mu, s2, p0, p1);
}

// gradient of lb_acq_value with respect to the candidate from grad mu (the mean's input gradient included) and grad s2, with
// f_max and the jitter held fixed (query_grad.cu, spgp.cu)
//   acq_id 0: UCB / GP_UCB  grad mu + p0 grad s2 / (2 sqrt(s2)), 0 for the second term where s2 <= 0
//   acq_id 1: EI            Phi(Z) grad mu + phi(Z) grad sigma; 0 below sigma = 1e-10 (ei.hpp:92-97)
__device__ __forceinline__ double lb_acq_grad_value(int acq_id, double mu, double s2, double gmu, double gs2, double p0, double p1)
{
    double g;
    if (acq_id == 0)
        g = gmu + (s2 > 0.0 ? p0 * gs2 / (2.0 * sqrt(s2)) : 0.0);
    else {
        const double sigma = sqrt(s2);
        g = 0.0;
        if (!(sigma < 1e-10)) {
            const double Z = (mu - p0 - p1) / sigma;
            const double phi = exp(-0.5 * (Z * Z)) / sqrt(2.0 * M_PI);
            const double Phi = 0.5 * erfc(-Z / sqrt(2.0));
            g = Phi * gmu + phi * (gs2 / (2.0 * sigma));
        }
    }
    return g;
}

// What the candidate-gradient pass (query_grad.cu) writes for one candidate chunk; every pointer may be NULL and starts at
// the chunk's first candidate.
struct LbGradOut {
    int acq_id;               // -1: no acquisition; otherwise an lb_acq_value id
    double p0, p1;            // acquisition parameters, as lb_acq_argmax takes them
    const double* mean;       // M first components of mean(v), or NULL and mean_const
    double mean_const;
    const double* mean_grad;  // M x Draw gradient of the mean's first component, or NULL (= 0)
    double* dmu;              // M x Draw: gradient of k^T alpha[:, 0]
    double* ds2;              // M x Draw: gradient of sigma^2, 0 where the clamp of gp.hpp:623 is active
    double* acq;              // M acquisition values
    double* grad;             // M x Draw acquisition gradients
};

// One model's side of a two-model acquisition gradient (ECI, EHVI), every pointer on the device from candidate 0
struct LbPairModel {
    const double* mu;         // M x p: k^T alpha (NULL: no such model)
    int p;
    const double* mean;       // M first components of mean(v), or NULL and mean_const
    double mean_const;
    const double* s2;         // M: sigma^2 (clamped + noise)
    const double* dmu;        // M x D: gradient of k^T alpha[:, 0]
    const double* ds2;        // M x D: gradient of sigma^2
    const double* mean_grad;  // M x D gradient of the mean's first component, or NULL (= 0)
};

// staged coordinate d (0 <= d < kp.D) of a raw point given by x(r), r < kp.Draw
template <typename F>
__device__ __forceinline__ double lb_staged_coord(const KernParams& kp, int d, F&& x)
{
    if (kp.id != LB_K_SE_ARD) return x(d);
    if (d < kp.Draw) return x(d) * kp.inv_ell[d]; // squared_exp_ard.hpp:148: cwiseQuotient(_ell), applied once per point
    double s = 0.0;
    const double* a = kp.lambda + (int64_t)(d - kp.Draw) * kp.Draw;
    for (int r = 0; r < kp.Draw; ++r) s = fma(a[r], x(r), s);
    return s;
}

// ---------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lb_smem_u32(const void* p)
{
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// fp64 tensor-core MMA (DMMA).  wgmma has no f64 kind; on sm_90a the fp64 tensor path is warp-level mma.sync.
// The m16n8k{4,8,16} f64 shapes exist from sm_90 on, and ptxas keeps each of them as ONE native instruction
// (DMMA.16x8x4 / DMMA.16x8x8 / DMMA.16x8x16).  Fragments of m16n8kK (KS = K):
//   A frag (16xK, row): a[i], i < KS/2: row = g + 8*(i&1), col = t + 4*(i>>1)
//   B frag (Kx8,  col): b[i], i < KS/4: k = t + 4*i, n = g
//   C frag (16x8)     : c[i], i < 4   : row = g + 8*(i>>1), col = 2*t + (i&1)
// with g = lane>>2, t = lane&3.  The C fragment is the same for every K (and equals two stacked m8n8k4 C fragments).
template <int KS>
__device__ __forceinline__ void lb_dmma_16x8(double (&c)[4], const double (&a)[KS / 2], const double (&b)[KS / 4])
{
    static_assert(KS == 4 || KS == 8 || KS == 16, "f64 mma.sync shapes: m16n8k4, m16n8k8, m16n8k16");
    if constexpr (KS == 4)
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(b[0]));
    else if constexpr (KS == 8)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                     "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                     : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

// m8n8k4 (DMMA.8x8x4), the only f64 shape before sm_90.  The GEMM core and the diagonal-block kernel use the
// m16n8kK shapes above; the single-point / slab query kernels and the tf32 path's K* dot products still issue this one.
//   a: A[row g][k t]   b: B[k t][n g]   c0,c1: C[row g][cols 2t, 2t+1]
__device__ __forceinline__ void lb_dmma_8x8x4(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

__device__ __forceinline__ void lb_cp_async16(void* smem_dst, const void* gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(lb_smem_u32(smem_dst)), "l"(gmem_src));
}
__device__ __forceinline__ void lb_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void lb_cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// mbarrier + TMA 1-D bulk copy (cp.async.bulk -> SASS UBLKCP)
__device__ __forceinline__ void lb_mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(lb_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void lb_fence_barrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::);
}
__device__ __forceinline__ void lb_fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;\n" ::);
}
__device__ __forceinline__ void lb_mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(lb_smem_u32(bar)), "r"(bytes));
}
__device__ __forceinline__ void lb_mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(lb_smem_u32(bar)),
        "r"(parity));
}
// bytes must be a multiple of 16; src/dst 16-byte aligned
__device__ __forceinline__ void lb_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(
                     lb_smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(lb_smem_u32(bar))
                 : "memory");
}

__device__ __forceinline__ double lb_warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---------------------------------------------------------------------------
// Device buffers
// ---------------------------------------------------------------------------
// pooled, reference-counted device buffers (pool.cu): every buffer a handle owns comes from here
void* lb_pool_alloc(int device, size_t bytes);
void lb_pool_free(void* p);     // drops one reference; the buffer returns to the pool with the last one
void lb_pool_retain(void* p);
bool lb_pool_shared(void* p);   // more than one handle references the buffer

struct lb_gp;

// Sole owner of one pool lease: the buffers of a handle that lb_clone never shares.  No implicit conversion to T*, so a
// DevBuf cannot be handed to lb_pool_free or overwritten with a raw pointer.  cudaFree synchronises implicitly, the pool
// does not: a reallocation waits for `stream` before the old buffer goes back, release() does not wait (the owner
// guarantees that no work on the buffer is pending).
template <typename T>
class DevBuf {
public:
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr; o.bytes_ = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept
    {
        if (this != &o) {
            release();
            p_ = o.p_; bytes_ = o.bytes_;
            o.p_ = nullptr; o.bytes_ = 0;
        }
        return *this;
    }
    ~DevBuf() { release(); }
    T* get() const { return p_; }
    explicit operator bool() const { return p_ != nullptr; }
    size_t bytes() const { return bytes_; }
    // grow-only: at least `bytes`; a reallocation takes `slack` bytes more
    int reserve(int device, cudaStream_t stream, size_t bytes, size_t slack = 0)
    {
        return (p_ && bytes_ >= bytes) ? LB_OK : take(device, stream, bytes + slack);
    }
    // exactly `bytes`
    int resize(int device, cudaStream_t stream, size_t bytes) { return (p_ && bytes_ == bytes) ? LB_OK : take(device, stream, bytes); }
    int reserve(const lb_gp* h, size_t bytes, size_t slack = 0);
    int resize(const lb_gp* h, size_t bytes);
    void release()
    {
        lb_pool_free(p_);
        p_ = nullptr;
        bytes_ = 0;
    }

private:
    int take(int device, cudaStream_t stream, size_t bytes)
    {
        if (p_) {
            cudaStreamSynchronize(stream); // kernels in flight may still use the old buffer
            release();
        }
        p_ = static_cast<T*>(lb_pool_alloc(device, bytes));
        if (!p_) return LB_ERR_ALLOC;
        bytes_ = bytes;
        return LB_OK;
    }
    T* p_ = nullptr;
    size_t bytes_ = 0;
};

// Buffers that live for one call on one stream: the destructor synchronises the stream once and returns every lease.
class StreamTemps {
public:
    StreamTemps(int device, cudaStream_t stream) : device_(device), stream_(stream) {}
    StreamTemps(const StreamTemps&) = delete;
    StreamTemps& operator=(const StreamTemps&) = delete;
    ~StreamTemps()
    {
        if (leases_.empty()) return;
        cudaStreamSynchronize(stream_);
        for (void* p : leases_) lb_pool_free(p);
    }
    template <typename T>
    int alloc(size_t bytes, T** out)
    {
        *out = static_cast<T*>(lb_pool_alloc(device_, bytes));
        if (!*out) return LB_ERR_ALLOC;
        leases_.push_back(*out);
        return LB_OK;
    }

private:
    int device_;
    cudaStream_t stream_;
    std::vector<void*> leases_;
};

// The values, means and argmax records of an M-candidate acquisition.  Callers size vals / mean; reserve() sizes the
// per-block (256 candidates) records and the final record.
struct ArgmaxWs {
    DevBuf<double> vals, mean, blk_val, best_val;
    DevBuf<long long> blk_idx, best_idx;
    // records of `cols` columns (lb_launch_acq_cols): cols x ceil(M / 256) block records and cols final records
    int reserve(int device, cudaStream_t stream, int64_t M, int cols = 1)
    {
        const size_t nblk = (size_t)((M + 255) / 256) * (size_t)cols;
        int rc;
        if ((rc = blk_val.reserve(device, stream, sizeof(double) * nblk)) || (rc = blk_idx.reserve(device, stream, sizeof(long long) * nblk))
            || (rc = best_val.reserve(device, stream, sizeof(double) * cols)) || (rc = best_idx.reserve(device, stream, sizeof(long long) * cols)))
            return rc;
        return LB_OK;
    }
    // the `cols` final records, and the nvals values when vals_out, to the host; synchronises the stream
    int read_best(cudaStream_t stream, double* best, int64_t* idx, double* vals_out, int64_t nvals, int cols = 1) const
    {
        static_assert(sizeof(long long) == sizeof(int64_t), "best_idx is copied as int64_t");
        if (vals_out) LB_CUDA(cudaMemcpyAsync(vals_out, vals.get(), sizeof(double) * nvals, cudaMemcpyDeviceToHost, stream));
        LB_CUDA(cudaMemcpyAsync(best, best_val.get(), sizeof(double) * cols, cudaMemcpyDeviceToHost, stream));
        LB_CUDA(cudaMemcpyAsync(idx, best_idx.get(), sizeof(long long) * cols, cudaMemcpyDeviceToHost, stream));
        LB_CUDA(cudaStreamSynchronize(stream));
        return LB_OK;
    }
};

// ---------------------------------------------------------------------------
// Host-side handle
// ---------------------------------------------------------------------------
struct lb_gp {
    int device = 0;
    int precision = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaStream_t side = nullptr;   // high-priority stream for the look-ahead panel factorisation
    cudaStream_t group[3] = {};    // streams of the panel query's second to fourth column groups, created on first use
    cudaEvent_t ev[LB_NEV] = {};

    int64_t N = 0;   // live samples
    int64_t Np = 0;  // padded capacity (multiple of 128)
    int D = 0, P = 0;

    KernParams kp{};
    bool kernel_set = false;
    int n_hparams = 0;

    double* dX = nullptr;    // D x Np raw samples (SoA)
    double* dXs = nullptr;   // (D + LB_MAX_LAMBDA) x Np samples staged for the kernel (SE-ARD: x/ell, then A^T x)
    DevBuf<double> dLambda;  // D x LB_MAX_LAMBDA (SE-ARD A matrix)
    DevBuf<double> dLinvW;   // reduced-precision path: |L^-1 e_k|^2 per column (rounding-bias weights)
    double* dY = nullptr;    // Np x P  obs_mean (col-major), zero padded
    double* dL = nullptr;    // Np x Np K then L (col-major)
    double* dInvD = nullptr; // T x 128 x 128
    double* dAlpha = nullptr; // Np x P
    DevBuf<double> dLinv;    // Np x Np (lazy: L^-1)
    DevBuf<double> dKinv;    // Np x Np (lazy: K^-1, lower valid + mirrored)
    DevBuf<float> dLinv32; bool linv32_valid = false; double linv32_scale = 1.0; // reduced-precision path: row-major fp32 / fp16 L^-1
    DevBuf<int> dInfo;       // [0] first failing pivot (1-based) or 0; [1] solver error
    DevBuf<int> dFlags;      // T+8 ints: ticket counters of the persistent solves
    DevBuf<double> dTrsvX;   // trsv: published solution blocks (sentinel-filled per launch)
    DevBuf<double> dScratch;

    bool fitted = false;
    bool linv_valid = false;
    int linv_levels = 0;     // diagonal blocks of this many 128-tiles of dLinv hold the inverse (0: nothing, >= T: all of L^-1)
    bool kinv_valid = false;
    bool kinv_sym = false;   // upper triangle of dKinv mirrored (needed by the LOO products and lb_get)
    DevBuf<double> dWork;    // Np x Np workspace (dK/dtheta of the LOO gradient)
    bool force_unfused = false; // tests: use the multi-launch query path

    // counters for bench.py ("gpu_launches")
    long long launches = 0;
    void* prof = nullptr; // Profiler* when per-kernel-class event timing is enabled (abi.cu)
};

template <typename T>
inline int DevBuf<T>::reserve(const lb_gp* h, size_t bytes, size_t slack) { return reserve(h->device, h->stream, bytes, slack); }
template <typename T>
inline int DevBuf<T>::resize(const lb_gp* h, size_t bytes) { return resize(h->device, h->stream, bytes); }

// The factor changed: every cache derived from it (L^-1 and its diagonal-block levels, K^-1, the reduced-precision copy)
// is stale.
inline void lb_factor_changed(lb_gp* h)
{
    h->linv_valid = false;
    h->linv_levels = 0;
    h->kinv_valid = false;
    h->linv32_valid = false;
}

// Every extern "C" entry that takes a handle runs on the handle's device and restores the caller's current device on
// return (one process may hold handles on several GPUs, e.g. one MultiGP output per device).
struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int device)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != device && cudaSetDevice(device) != cudaSuccess) ok = false;
    }
    ~DeviceGuard()
    {
        if (prev >= 0) {
            int cur = -1;
            if (cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
        }
    }
};
#define LB_DEVICE(h)                        \
    DeviceGuard lb_dev_guard__((h)->device); \
    if (!lb_dev_guard__.ok) return LB_ERR_CUDA

// cudaFuncSetAttribute applies to the CURRENT device: once-only flags must be per device (one process may hold handles on
// several GPUs, e.g. one MultiGP output per device).  need() is true the first time it is called on a device.
struct LbOncePerDevice {
    bool done[64] = {};
    bool need()
    {
        int d = 0;
        if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return true;
        if (done[d]) return false;
        done[d] = true;
        return true;
    }
};

// the buffers lb_clone shares copy-on-write (ref-counted raw pointers)
template <typename T>
inline int lb_dalloc(const lb_gp* h, T** p, size_t bytes)
{
    *p = static_cast<T*>(lb_pool_alloc(h->device, bytes));
    return *p ? LB_OK : LB_ERR_ALLOC;
}
#define LB_ALLOC(h, ptr, bytes)                      \
    do {                                             \
        int rc_alloc__ = lb_dalloc((h), &(ptr), (bytes)); \
        if (rc_alloc__) return rc_alloc__;           \
    } while (0)

// per-kernel-class CUDA-event timing (bench.py roofline): no-ops unless enabled
enum { LB_PC_KBUILD = 0, LB_PC_POTF2, LB_PC_TRSM_PANEL, LB_PC_SYRK, LB_PC_SYRK_COL, LB_PC_TRSV, LB_PC_KSTAR, LB_PC_QSTEP, LB_PC_QREDUCE,
    LB_PC_ACQ, LB_PC_TRTRI, LB_PC_LAUUM, LB_PC_GRAD, LB_PC_OTHER, LB_PC_COUNT };
void lb_prof_begin(const lb_gp* h, cudaStream_t st, int cls);
void lb_prof_end(const lb_gp* h, cudaStream_t st, int cls);
struct LbProfScope {
    const lb_gp* h; cudaStream_t st; int cls;
    LbProfScope(const lb_gp* h_, cudaStream_t st_, int c) : h(h_), st(st_), cls(c) { if (h->prof) lb_prof_begin(h, st, cls); }
    ~LbProfScope() { if (h->prof) lb_prof_end(h, st, cls); }
};

// internal entry points: what one .cu defines and another calls is declared here and nowhere else, under the file that defines it
// (the pool, the profiler hooks and lb_set_last_cuda_error: above, ahead of the types that use them)
// abi.cu
int lb_ensure_scratch(lb_gp* h, size_t bytes);
// kbuild.cu
int lb_launch_scale_x(lb_gp* h);
int lb_launch_kbuild(lb_gp* h, double* dK);
// potrf.cu
int lb_launch_potrf(lb_gp* h);
int lb_launch_potf2_block(lb_gp* h, int k, int do_factor);
int lb_debug_potf2_clocks(lb_gp* h, int k, long long* out_host, int n);
// trsv.cu
int lb_launch_solve_alpha(lb_gp* h);
int lb_launch_trsv(lb_gp* h, double* dB, int nrhs, bool forward);
// query.cu
int lb_launch_trsm_lower(const lb_gp* h, cudaStream_t st, double* dV, int64_t Mp, int i_begin, long long* launches);
int lb_launch_query(const lb_gp* h, cudaStream_t st, int64_t M, const double* dXq_soa /*D x Mp*/, int64_t Mp,
    double* dV /*Np x Mp*/, double* dMu /*Mp x P*/, double* dS2 /*Mp*/, long long* launches);
int lb_launch_acq_full(cudaStream_t st, int acq_id, double p0, double p1, int64_t M, const double* dMu, int mu_stride,
    const double* dMeanAtQ, double mean_const, const double* dS2, double* dAcq, double* dBlkVal, long long* dBlkIdx,
    double* dBestVal, long long* dBestIdx, long long* launches);
// acq_full over the P columns of mu (query.cu: acq_cols_kernel): dParams (P x 2), dMeanAtQ (M x P) or dMeanConst (P) per column.  Without
// dInstCol: the M x P values (dAcq, may be NULL) and one record per column (dBlkVal / dBlkIdx: P x ceil(M / 256); dBestVal / dBestIdx: P).
// With dInstCol: candidate m scored in column dInstCol[m / lam] only, M values and one record over all of them.
int lb_launch_acq_cols(cudaStream_t st, int acq_id, const double* dParams, int64_t M, const double* dMu, int P, const double* dMeanAtQ,
    const double* dMeanConst, const double* dS2, const int* dInstCol, int lam, double* dAcq, double* dBlkVal, long long* dBlkIdx,
    double* dBestVal, long long* dBestIdx, long long* launches);
int lb_launch_eci_full(cudaStream_t st, double f_max, double jitter, int64_t M, const double* dMuObj, int p_obj, const double* dMeanObj,
    double mean_obj_const, const double* dS2Obj, const double* dMuCon, int p_con, const double* dMeanCon, double mean_con_const,
    const double* dS2Con, double* dAcq, double* dBlkVal, long long* dBlkIdx, double* dBestVal, long long* dBestIdx, long long* launches);
int lb_launch_values_argmax(cudaStream_t st, int64_t M, const double* dVals, double* dBlkVal, long long* dBlkIdx, double* dBestVal,
    long long* dBestIdx, long long* launches);
int lb_launch_eci_grad(cudaStream_t st, double f_max, double jitter, int64_t M, int D, const LbPairModel& obj, const LbPairModel& con,
    double* dAcq, double* dGrad, long long* launches);
size_t lb_query_panel_scratch_doubles(const lb_gp* h, int64_t Mp);
double* lb_query_panel_tbuf(const lb_gp* h, double* dWork, int64_t Mp);
double* lb_query_panel_norms(const lb_gp* h, double* dWork, int64_t Mp);
int lb_query_panel_groups(lb_gp* h, cudaStream_t st, int ctiles, cudaStream_t sts[4], int gbeg[5]);
int lb_launch_query_panel(lb_gp* h, cudaStream_t st, int64_t M, const double* dQs, int64_t Mp, double* dWork, double* dMu, double* dS2,
    long long* launches);
int64_t lb_linv_columns_width(const lb_gp* h, int G);
size_t lb_linv_columns_scratch_doubles(const lb_gp* h, int G);
int lb_launch_linv_columns(lb_gp* h, cudaStream_t st, int rank, int G, double* dWork, long long* launches);
int lb_query_fused_supported(const lb_gp* h);
size_t lb_query_fused_scratch_doubles(const lb_gp* h, int grid);
int lb_launch_query_point(const lb_gp* h, cudaStream_t st, const double* x_host, double* dQs, double* dVscratch, double* dOutMapped,
    long long* launches);
int lb_launch_query_fused(const lb_gp* h, cudaStream_t st, int64_t M, const double* dQs, int64_t Mp, double* dVscratch,
    int grid, double* dMu, double* dS2, long long* launches);
// query_grad.cu
int lb_launch_query_grad(lb_gp* h, cudaStream_t st, int64_t M, const double* dQs, int64_t Mp, double* dWork, double* dMu, double* dS2,
    const LbGradOut& out, long long* launches);
int lb_launch_prior_grad(cudaStream_t st, int64_t M, int D, int P, double s2, const LbGradOut& out, double* dMu, double* dS2);
// lml.cu
int lb_launch_loglik(lb_gp* h, double* dOut /*3 doubles: a, logdet, loglik*/);
int lb_launch_linv_levels(lb_gp* h, int want_tiles); // inverse of the diagonal blocks of `want_tiles` 128-tiles (power of two)
int lb_launch_linv(lb_gp* h);
int lb_launch_kinv(lb_gp* h);
int lb_launch_symmetrize(lb_gp* h, double* dA);
int lb_launch_grad(lb_gp* h, int optimize_noise, double* dGrad);
// lml_batch.cu: one launch over the R kernel states kps (one kernel and layout; lambda unset) with the Lambda columns of the host
// rows hparams (R x n_hparams, lb_lml_grad_batch's); dGrad NULL = likelihood only
int lb_launch_lml_batch(cudaStream_t st, StreamTemps& tmp, const KernParams* kps, const double* hparams, int n_hparams, int R,
    const double* dX, int64_t ldx, const double* dY, int N, int P, int nh, int optimize_noise, double* dLik, double* dGrad, int* dInfo,
    long long* launches);
// loo.cu
int lb_launch_loo_value(lb_gp* h, double* dOut);
int lb_launch_loo_grad(lb_gp* h, int optimize_noise, double* dGrad);
int lb_launch_grad_lambda(lb_gp* h, double* dGrad);
int lb_launch_kinv_obs(lb_gp* h, double* dOut);
// tf32_query.cu
int lb_tf32_prepare(lb_gp* h);
size_t lb_dinv_chunk_bytes_impl(const lb_gp* h, int G);
int lb_dinv_absmax(lb_gp* h, const double* dV, int G, double* out);
int lb_dinv_pack_impl(lb_gp* h, const double* dV, int rank, int G, double absmax_all, void* dChunk);
int lb_dinv_adopt_impl(lb_gp* h, int G, const void* dAll, double absmax_all);
int lb_launch_kstar_tf32(const lb_gp* h, cudaStream_t st, int64_t Mc, const double* dQs, int64_t Mcp, float* dKt, double* dMuPart,
    double* dMu, double* dBias, long long* launches);
int lb_launch_sigma_tf32(const lb_gp* h, cudaStream_t st, int64_t Mc, int64_t Mcp, const float* dKt, float* dNorm2, int* dErr,
    const double* dBias, double* dS2, long long* launches);
// ehvi.cu
int lb_launch_ehvi(cudaStream_t st, double r0, double r1, int64_t k, const double* dFront, int64_t M, const double* dMu0, int p0,
    const double* dMean0, double mean0_const, const double* dS2_0, const double* dMu1, int p1, const double* dMean1, double mean1_const,
    const double* dS2_1, double* dAcq, long long* launches);
int lb_launch_ehvi_grad(cudaStream_t st, double r0, double r1, int64_t k, const double* dFront, int64_t M, int D, const LbPairModel& g0,
    const LbPairModel& g1, double* dAcq, double* dGrad, long long* launches);
int lb_launch_pareto(cudaStream_t st, int64_t n, int K, const double* dObjs, int* dKeep, int* dErr, long long* launches);
// one model of lb_ehvi3d_argmax at the candidates: mu (M x p; FirstElem is read), the mean added to it (per candidate, or the
// constant when mean is NULL) and sigma^2 + noise (M)
struct LbEhvi3Model {
    const double* mu;
    int p;
    const double* mean;
    double mean_const;
    const double* s2;
};
// doubles of the ehvi3d passes' workspace for a front of k points and M candidates
size_t lb_ehvi3d_ws_doubles(int64_t k, int64_t M);
// ehvi3d_sliceupdate in two passes over dWs (lb_ehvi3d_ws_doubles(k, M) doubles); dFront is the 9 k doubles lb_ehvi3d_argmax
// uploads.  The front pass builds the per-cell planes, which depend on the front and ref_point only; the cell pass scores every
// candidate into dAcq (M) from them, and may run any number of times after one front pass for the same front, k and M.
int lb_launch_ehvi3d_front(cudaStream_t st, const double* r, int64_t k, const double* dFront, double* dWs, long long* launches);
int lb_launch_ehvi3d_cells(cudaStream_t st, const double* r, int64_t k, const double* dFront, int64_t M, const LbEhvi3Model& m0,
    const LbEhvi3Model& m1, const LbEhvi3Model& m2, double* dWs, double* dAcq, long long* launches);
// cmaes.cu: the batched CMA-ES of lb_acq_cmaes / lb_eci_cmaes / lb_ehvi_cmaes / lb_spgp_acq_cmaes (DESIGN.md §4.15).  Per instance, the device state is
// lb_cmaes_state_doubles(D) doubles: m, p_sigma, p_c, best_x (D each), C and A (D x D row-major each; A lower), then sigma,
// best_val and the stop flag.
#define LB_CMAES_MAX_D 64
#define LB_CMAES_MAX_LAMBDA 256
struct lb_cmaes_opts; // include/limbo_b200.h
struct LbCmaes {
    int R, D, lam, mu, bounded;
    uint64_t seed;
    double cs, ds, cc, c1, cmu, mueff, chi, sumw, tolx;
    const double* w;   // lam recombination weights (device)
    double* state;     // R x lb_cmaes_state_doubles(D)
    double* z;         // R x lam x D: the draws of the current generation
    double* y;         // R x lam x D: A z
    double* cand;      // R x lam x D: the phenotypes, the scorer's candidates
};
__host__ __device__ inline int64_t lb_cmaes_state_doubles(int D) { return 4 * (int64_t)D + 2 * (int64_t)D * D + 3; }
// The strategy constants and the weights (host, lam doubles) of lb_cmaes_opts o in dimension D, into s (pointers untouched);
// LB_ERR_UNSUPPORTED past LB_CMAES_MAX_D / LB_CMAES_MAX_LAMBDA, LB_ERR_ARG for a bad option.
int lb_cmaes_setup(const lb_cmaes_opts& o, int D, int R, LbCmaes* s, std::vector<double>* w);
// the initial state of instance r from its start (phenotype), into st (lb_cmaes_state_doubles(D) doubles)
void lb_cmaes_init_state(const LbCmaes& s, double sigma0, const double* start, double* st);
// generation g: draws, A z and the phenotypes into s.cand
int lb_launch_cmaes_ask(cudaStream_t st, const LbCmaes& s, int g, long long* launches);
// *dFlag |= *dErr (a scoring pass's reduced-precision timeout flag) on st
int lb_launch_cmaes_flag(cudaStream_t st, const int* dErr, int* dFlag, long long* launches);
// generation g's update from the R x lam values dVals; dLive (NULL: not counted) gains the instances still live after it
int lb_launch_cmaes_tell(cudaStream_t st, const LbCmaes& s, int g, const double* dVals, int* dLive, long long* launches);
// abi.cu: the search loop that every device CMA-ES entry point drives with its own scorer.  What it needs of the model: the
// device and stream it runs on (its pool leases are returned when the search ends), D, the launch counter its kernels add to, and
// the reduced-precision timeout word of each scored handle (NULL: none; fp64 scorers have none), read after every scoring since
// the first fill may allocate it.  The caller holds every lock the scorer needs for the whole search.
struct LbCmaesHost {
    int device;
    cudaStream_t stream;
    int D;
    long long* launches;
    std::array<const DevBuf<int>*, 3> timeouts;
};
using LbCmaesPrepare = std::function<int(int64_t M)>; // once, before the first generation
// enqueues the values of the M device candidates dCand into dVals and their argmax into dBestVal / dBestIdx, on the search's stream
using LbCmaesScore = std::function<int(const double* dCand, int64_t M, double* dVals, double* dBestVal, long long* dBestIdx)>;
// With cols (R host ints in [0, q)), instance r is bound to column cols[r], and best_x (q x D) / best_val (q) hold each column's best
// over its instances (ties to the lower instance); without, one best over all of them.
int lb_cmaes_search(const LbCmaesHost& on, const lb_cmaes_opts* opts, int64_t R, const double* starts, const LbCmaesPrepare& prepare,
    const LbCmaesScore& score, double* best_x, double* best_val, int64_t* n_evals, const int* cols = nullptr, int q = 1);
// the checks every entry point makes before any lock: pointers, 0 < R <= INT32_MAX and finite starts (R x D)
int lb_cmaes_args(const lb_cmaes_opts* opts, int64_t R, const double* starts, int D, const double* best_x, const double* best_val,
    const int64_t* n_evals);
// sparsify.cu
int lb_run_sparsify(const lb_gp* h, cudaStream_t st, int64_t N, int D, const double* dX, int64_t max_points, long long* dKept,
    int64_t* n_kept, long long* dRemoved, double* dRemovedScore, long long* launches);
