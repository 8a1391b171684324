/* include/limbo_b200.h — C ABI of the H100-native (sm_90a) GP compute backend for Limbo.
 *
 * The reference (resibots/limbo @ 43c67a6) has no FFI for this path: the seam
 * is the C++ "Model concept" implemented by limbo::model::GP
 * (src/limbo/model/gp.hpp:81-511).  This header is the boundary a drop-in
 * model type binds to (include/limbo_b200/model/gp.hpp does exactly that, and
 * INTEGRATION.md shows the maintainer-side glue).  Each entry point names the
 * reference member it replaces.
 *
 * Conventions
 *   - all pointers are HOST pointers unless the function name ends in _dev;
 *   - matrices are column-major like Eigen::MatrixXd; sample/candidate arrays
 *     are row-major "one point per row" (the reference holds them as
 *     std::vector<Eigen::VectorXd>);
 *   - mean functions stay on the host (they are arbitrary user functors,
 *     src/limbo/mean/mean.hpp:60-77): callers pass obs_mean = Y - M
 *     (gp.hpp:547) and add mean(v) to the returned mu (gp.hpp:615);
 *   - every function returns 0 on success; > 0 = 1-based index of the first
 *     non-positive Cholesky pivot (LAPACK-style info; the reference never
 *     checks Eigen's info(), gp.hpp:565); < 0 = LB_ERR_*;
 *   - lb_query / lb_acq_argmax on one handle may be called from several host
 *     threads (the reference's query() is const and called concurrently from
 *     TBB workers, opt/parallel_repeater.hpp:103); mutating calls need
 *     exclusive access to the handle.
 *   - there is no CPU fallback: without a CUDA device lb_create fails.
 */
#ifndef LIMBO_B200_H
#define LIMBO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lb_gp lb_gp;

#define LB_OK 0
#define LB_ERR_ARG (-1)
#define LB_ERR_CUDA (-2)
#define LB_ERR_STATE (-3)
#define LB_ERR_ALLOC (-4)
#define LB_ERR_UNSUPPORTED (-5)
#define LB_ERR_TIMEOUT (-6)

/* kernel ids (the functors under src/limbo/kernel/) */
#define LB_KERNEL_SQUARED_EXP_ARD 0 /* kernel/squared_exp_ard.hpp   h-params [log l_1..log l_D, (A(:,0) .. A(:,k-1): D each, k <= 4), log sigma_f];
                                       k = Params::kernel_squared_exp_ard::k() is inferred from n_hparams = D + D k + 1 */
#define LB_KERNEL_MATERN_FIVE_HALVES 1 /* kernel/matern_five_halves.hpp      h-params [log l, log sigma_f] */
#define LB_KERNEL_MATERN_THREE_HALVES 2 /* kernel/matern_three_halves.hpp */
#define LB_KERNEL_EXP 3 /* kernel/exp.hpp */

/* acquisition ids */
#define LB_ACQ_UCB 0 /* acqui/ucb.hpp:83-90 and acqui/gp_ucb.hpp:96-103; params[0] = alpha (resp. beta) */
#define LB_ACQ_EI 1  /* acqui/ei.hpp:85-116; params[0] = f_max, params[1] = jitter */

/* lb_get selectors */
#define LB_GET_K 0     /* _kernel     gp.hpp:553-562 (N x N, both triangles) */
#define LB_GET_L 1     /* _matrixL    gp.hpp:565     (N x N, zero upper part) */
#define LB_GET_ALPHA 2 /* _alpha      gp.hpp:605-611 (N x P) */
#define LB_GET_KINV 3  /* _inv_kernel gp.hpp:254-264 (N x N) */

/* precision modes */
#define LB_PREC_FP64 0
/* fit / likelihood in fp64; lb_query and lb_acq_argmax compute sigma^2 on the tf32 tensor cores (wgmma, fp32
 * accumulation) from an fp64-inverted factor; mu stays fp64.  |d sigma^2| = a few 1e-3 k(v,v), growing with cond(K)
 * (the bounds tests/test_gpu_tf32.py asserts) */
#define LB_PREC_TF32 1
/* same path with fp16 operands (same 11-bit significand as tf32, half the operand bytes, twice the tensor rate);
 * K* is scaled by 1/sigma_f^2 and L^-1 by a power of two so that both stay inside the fp16 range */
#define LB_PREC_FP16 2
/* fp16 split operands: every operand is hi + 2^-11 lo (two fp16 planes, 22 significant bits), three tensor-core products per
 * k-step, hi x hi and the cross terms in separate fp32 accumulators, combined and squared in fp64.  About 3x the scoring time of
 * LB_PREC_FP16; |d sigma^2| <= 2e-5 k(v,v) up to N = 4096 and <= 1e-4 at N = 16384, cond(K) ~ 1.6e6 (the fp32 accumulation of the
 * tensor core is the floor there; tests/test_gpu_tf32.py, tests/test_gpu_config4.py), against 2-4e-3 for the one-plane modes */
#define LB_PREC_FP16X3 3

/* Lifetime.  Replaces GP(int dim_in, int dim_out) / ~GP / the copy constructor
 * KernelLFOptimization relies on (model/gp/kernel_lf_opt.hpp:79). */
int lb_create(lb_gp** out, int device, int precision);
int lb_destroy(lb_gp* h);
int lb_clone(const lb_gp* h, lb_gp** out);

/* Run all work of this handle on an existing CUDA stream (cudaStream_t cast
 * to void*); NULL restores the handle's own stream. */
int lb_set_stream(lb_gp* h, void* cuda_stream);
int lb_sync(lb_gp* h);
/* number of kernels launched by this handle so far */
long long lb_launch_count(const lb_gp* h);

/* GP::compute data part (gp.hpp:88-116): N samples of dimension D (row-major
 * N x D) and obs_mean = observations - mean (column-major N x P). */
int lb_set_data(lb_gp* h, int64_t N, int D, int P, const double* X_rowmajor, const double* obs_mean_colmajor);
int lb_set_data_dev(lb_gp* h, int64_t N, int D, int P, const double* dX_rowmajor, const double* dObsMean_colmajor);

/* Kernel functor state: BaseKernel::set_h_params (kernel/kernel.hpp:116-123).
 * log_hparams are the kernel's own log-space parameters (without the noise
 * entry); noise is the signal noise itself (kernel.hpp:126). */
int lb_set_kernel(lb_gp* h, int kernel_id, const double* log_hparams, int n_hparams, double noise);

/* GP::_compute_full_kernel (gp.hpp:550-571): K -> L -> alpha. */
int lb_fit(lb_gp* h);
/* GP::recompute(update_obs_mean, update_full_kernel=false) (gp.hpp:241-252):
 * new obs_mean, same factor, re-solve alpha. */
int lb_refit_alpha(lb_gp* h, const double* obs_mean_colmajor);
/* GP::add_sample / _compute_incremental_kernel (gp.hpp:126-152, 573-603):
 * x is the new sample (D), obs_mean_all the refreshed (N+1) x P obs_mean. */
int lb_append(lb_gp* h, const double* x, const double* obs_mean_all_colmajor);

/* GP::load(archive, recompute = false) (gp.hpp:505-509): adopt a stored factor (N x N column-major, lower) and alpha
 * (N x P) for the data / kernel already set, instead of refactorising. */
int lb_load_factor(lb_gp* h, const double* L_colmajor, const double* alpha_colmajor);

/* Batched GP::query (gp.hpp:159-167) for M candidates (row-major M x D):
 * mu_minus_mean is M x P row-major (k^T alpha, WITHOUT mean(v));
 * sigma2 is M (clamped as gp.hpp:623, + noise as gp.hpp:166).
 * With N == 0 returns the prior (gp.hpp:161-163). */
int lb_query(const lb_gp* h, int64_t M, const double* Xq_rowmajor, double* mu_minus_mean, double* sigma2);
int lb_query_dev(const lb_gp* h, int64_t M, const double* dXq_rowmajor, double* dMu_minus_mean, double* dSigma2);

/* Batched acquisition + argmax over M candidates with the FirstElem
 * aggregator (bayes_opt/bo_base.hpp:99-105).  mean_at_q: M values of the
 * first component of mean(v), or NULL to add mean_const to every mu.
 * acq_out (optional, M values) receives the acquisition values.  Ties resolve
 * to the lowest index, like the reference's sequential scan. */
int lb_acq_argmax(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* Xq_rowmajor,
    const double* mean_at_q, double mean_const, double* acq_out, double* best_val, int64_t* best_idx);
/* same, device pointers; d_best = {value, (double) index bit-copied as int64} */
int lb_acq_argmax_dev(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* dXq_rowmajor,
    const double* dMean_at_q, double mean_const, double* dAcq_out, double* dBest_val, int64_t* dBest_idx);
/* lb_acq_argmax over each of the handle's q = P output columns from one query of the M candidates: ParEGO's q scalarisations of
 * the objectives (experimental/model/gp_parego.hpp:103-117) share the factor, the candidates' K* and sigma^2, and column r is scored
 * with its own acquisition (acq_params[2 r], acq_params[2 r + 1]: UCB / GP_UCB alpha and an unused slot, or EI f_max and jitter) and
 * its own mean (mean_at_q: M x q row-major, or NULL to add mean_const[r] to column r).  acq_out (optional) receives the M x q
 * row-major values; best_val[r] / best_idx[r] the best candidate of column r, ties to the lowest index.  With q = 1 every output
 * is bit-identical to lb_acq_argmax's.  The lock, stream and path rules of lb_acq_argmax.  LB_ERR_ARG for a NULL argument, M <= 0
 * or q other than the handle's P (1 for a handle without observations); LB_ERR_UNSUPPORTED for an unknown acq_id, a
 * reduced-precision handle or q > LB_ACQ_MAX_COLS (the launch has one grid row per column). */
#define LB_ACQ_MAX_COLS 65535
int lb_acq_argmax_cols(const lb_gp* h, int acq_id, int64_t q, const double* acq_params, int64_t M, const double* Xq_rowmajor,
    const double* mean_at_q, const double* mean_const, double* acq_out, double* best_val, int64_t* best_idx);
/* same, device pointers except acq_params and mean_const (host, q x 2 and q); bit-identical to lb_acq_argmax_cols */
int lb_acq_argmax_cols_dev(const lb_gp* h, int acq_id, int64_t q, const double* acq_params, int64_t M, const double* dXq_rowmajor,
    const double* dMean_at_q, const double* mean_const, double* dAcq_out, double* dBest_val, int64_t* dBest_idx);

/* Candidate gradients for M candidates (row-major M x D), extending lb_query with what the reference's gradient optimisers
 * (opt/gradient_ascent.hpp, opt/adam.hpp, opt/rprop.hpp) ask of f(x, gradient), which acqui/ucb.hpp:83-90 and acqui/ei.hpp:85-116
 * leave unimplemented (assert(!gradient)).  mu_minus_mean (M x P row-major, without mean(v)) and sigma2 (M, clamped + noise) are
 * bit-identical to lb_query's on its large-batch path; dmu (M x D row-major) is the gradient of the first output of mu_minus_mean,
 * dsigma2 (M x D) that of sigma2, 0 where the clamp of gp.hpp:623 is active.  Any output may be NULL.  With N == 0 the gradients are
 * 0.  fp64 handles only (LB_ERR_UNSUPPORTED otherwise); LB_ERR_ARG for M <= 0 or a non-finite coordinate.  May be called from
 * several threads, as lb_query. */
int lb_query_grad(const lb_gp* h, int64_t M, const double* Xq_rowmajor, double* mu_minus_mean, double* sigma2,
    double* dmu, double* dsigma2);
/* same, device pointers (the coordinates are not checked) */
int lb_query_grad_dev(const lb_gp* h, int64_t M, const double* dXq_rowmajor, double* dMu_minus_mean, double* dSigma2,
    double* dDmu, double* dDsigma2);
/* Acquisition value (M) and gradient (M x D row-major) with the FirstElem aggregator, extending lb_acq_argmax (same acq_id and
 * acq_params, same values on its large-batch path): UCB / GP_UCB grad = grad mu + params[0] grad sigma2 / (2 sqrt(sigma2)), EI
 * (ei.hpp:85-116) grad = Phi(Z) grad mu + phi(Z) grad sigma with f_max and the jitter fixed, value and gradient 0 where
 * sigma < 1e-10.  mean_at_q / mean_const as in lb_acq_argmax; mean_grad_at_q: M x D gradient of mean(v)'s first component, or NULL
 * when the mean does not depend on v.  LB_ERR_ARG for M <= 0, a non-finite coordinate or an unknown acq_id; fp64 handles only. */
int lb_acq_grad(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* Xq_rowmajor,
    const double* mean_at_q, double mean_const, const double* mean_grad_at_q, double* acq_out, double* grad_out);
/* same, device pointers except acq_params (the coordinates are not checked) */
int lb_acq_grad_dev(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* dXq_rowmajor,
    const double* dMean_at_q, double mean_const, const double* dMean_grad_at_q, double* dAcq_out, double* dGrad_out);

/* experimental/acqui/eci.hpp:76-107 over an objective and a constraint model, FirstElem aggregator:
 *   ECI = Pf * EI,  EI as LB_ACQ_EI on obj,  Pf = Phi((mu_c[0] - 1) / sigma_c) on con (eci.hpp:116-130).
 * eci_params = {f_max, jitter}; con may be NULL (no constraints: Pf = 1), as may a con without samples.  An obj without samples
 * scores 0 everywhere (index 0).  obj and con must be distinct handles on the same device with the same input dimension; both
 * are locked for the call, and their queries run on their own streams.  The means are added as in lb_acq_argmax (an array of
 * M first components, or NULL and a constant).  Ties resolve to the lowest index. */
int lb_eci_argmax(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* Xq_rowmajor,
    const double* obj_mean_at_q, double obj_mean_const, const double* con_mean_at_q, double con_mean_const,
    double* acq_out, double* best_val, int64_t* best_idx);
/* same, device pointers (eci_params stays on the host); no synchronisation, results on obj's stream */
int lb_eci_argmax_dev(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* dXq_rowmajor,
    const double* dObj_mean_at_q, double obj_mean_const, const double* dCon_mean_at_q, double con_mean_const,
    double* dAcq_out, double* dBest_val, int64_t* dBest_idx);

/* ECI value (M) and gradient (M x D row-major) with respect to the candidates, extending lb_eci_argmax as lb_acq_grad extends
 * lb_acq_argmax: with f_max and the jitter fixed,
 *   grad ECI = Pf grad EI + EI grad Pf,   grad EI as LB_ACQ_EI's in lb_acq_grad,
 *   grad Pf = phi(Z_c) (grad mu_c - Z_c grad sigma_c^2 / (2 sigma_c)) / sigma_c,   Z_c = (mu_c[0] - 1) / sigma_c.
 * Value and gradient are 0 where sigma < 1e-10 and everywhere when obj has no samples; grad Pf is 0 where sigma_c < 1e-10, and
 * without con or constraint samples (Pf = 1).  The values are bit-identical to lb_eci_argmax's on its large-batch path.  Both
 * handles' gradient passes run on their own streams, as in lb_eci_argmax.  The means as there; *_mean_grad_at_q: M x D gradient
 * of that mean's first component, or NULL when it does not depend on v.  Either output may be NULL.  LB_ERR_ARG for M <= 0, a
 * non-finite coordinate, obj == con or a different input dimension; LB_ERR_UNSUPPORTED unless both handles are fp64.  As in
 * lb_eci_argmax, an obj without samples gives 0 without its kernel being set; unlike there, its input dimension must be set
 * (lb_set_data, N = 0 allowed), since the gradient has D columns (LB_ERR_STATE otherwise). */
int lb_eci_grad(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* Xq_rowmajor,
    const double* obj_mean_at_q, double obj_mean_const, const double* obj_mean_grad_at_q, const double* con_mean_at_q,
    double con_mean_const, const double* con_mean_grad_at_q, double* acq_out, double* grad_out);
/* same, device pointers except eci_params (the coordinates are not checked); no synchronisation, results on obj's stream */
int lb_eci_grad_dev(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* dXq_rowmajor,
    const double* dObj_mean_at_q, double obj_mean_const, const double* dObj_mean_grad_at_q, const double* dCon_mean_at_q,
    double con_mean_const, const double* dCon_mean_grad_at_q, double* dAcq_out, double* dGrad_out);

/* Largest front lb_ehvi_argmax takes, and largest number of objectives lb_pareto_set takes (LB_ERR_UNSUPPORTED above). */
#define LB_EHVI_MAX_K 4096
#define LB_PARETO_MAX_K 8

/* experimental/acqui/ehvi.hpp:70-79 (ehvi2d, src/ehvi/ehvi_calculations.cc:16-79) over two models, FirstElem aggregator:
 *   EHVI(v) = ehvi2d(front, ref_point, (mu_0(v)[0], mu_1(v)[0]), (s_0(v), s_1(v))),
 * with s the models' sigma() = sigma^2 + noise, as the reference passes it (ehvi2d expects a standard deviation there).  front is
 * k x 2 row-major (k = 0: one cell against ref_point), ref_point has 2 entries; both stay on the host in the _dev variant too.
 * m0 and m1 must be distinct handles on the same device with the same input dimension; both are locked for the call and their
 * queries run on their own streams.  A model without samples scores with its prior.  The means are added as in lb_acq_argmax.
 * Ties resolve to the lowest index.  LB_ERR_ARG for M <= 0 or a non-finite front or ref_point; LB_ERR_UNSUPPORTED when
 * k > LB_EHVI_MAX_K. */
int lb_ehvi_argmax(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* Xq_rowmajor, const double* mean0_at_q, double mean0_const, const double* mean1_at_q, double mean1_const,
    double* acq_out, double* best_val, int64_t* best_idx);
/* same, device pointers except ref_point and front; no synchronisation, results on m0's stream */
int lb_ehvi_argmax_dev(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* dXq_rowmajor, const double* dMean0_at_q, double mean0_const, const double* dMean1_at_q, double mean1_const,
    double* dAcq_out, double* dBest_val, int64_t* dBest_idx);
/* EHVI value (M) and gradient (M x D row-major) with respect to the candidates, extending lb_ehvi_argmax: the partials of ehvi2d
 * in (mu_0, s_0, mu_1, s_1) chained with each model's grad mu (plus mean*_grad_at_q, M x D or NULL) and grad sigma^2 (s = sigma^2 +
 * noise stands where ehvi2d expects a deviation, so ds/dv = grad sigma^2).  A cell adds to the gradient where it adds to the value
 * (its sum > 0); a model with s <= 0 adds nothing.  The values are bit-identical to lb_ehvi_argmax's on its large-batch path.
 * Either output may be NULL.  Argument rules as lb_ehvi_argmax's, plus LB_ERR_ARG for a non-finite coordinate; LB_ERR_UNSUPPORTED
 * unless both handles are fp64. */
int lb_ehvi_grad(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* Xq_rowmajor, const double* mean0_at_q, double mean0_const, const double* mean0_grad_at_q, const double* mean1_at_q,
    double mean1_const, const double* mean1_grad_at_q, double* acq_out, double* grad_out);
/* same, device pointers except ref_point and front (the coordinates are not checked); no synchronisation, results on m0's stream */
int lb_ehvi_grad_dev(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* dXq_rowmajor, const double* dMean0_at_q, double mean0_const, const double* dMean0_grad_at_q,
    const double* dMean1_at_q, double mean1_const, const double* dMean1_grad_at_q, double* dAcq_out, double* dGrad_out);

/* Largest front lb_ehvi3d_argmax takes (LB_ERR_UNSUPPORTED above).  The front pass keeps two (k + 1) x k x k planes of fp64 in m0's
 * query workspace: 271 MB at the cap. */
#define LB_EHVI3D_MAX_K 256

/* Three-objective EHVI: ehvi3d_sliceupdate (src/ehvi/ehvi_sliceupdate.cc:13-185) over three models, FirstElem aggregator:
 *   EHVI3(v) = ehvi3d_sliceupdate(front, ref_point, (mu_0(v)[0], mu_1(v)[0], mu_2(v)[0]), (s_0(v), s_1(v), s_2(v))),
 * with s the models' sigma() = sigma^2 + noise, the convention lb_ehvi_argmax keeps (the reference has no three-objective
 * functor).  front is k x 3 row-major (k = 0: one cell from ref_point to +inf), ref_point has 3 entries; both stay on the host in
 * the _dev variant too.  The front is sorted per axis stably by input index.  Ties resolve to the lowest index.
 *   LB_ERR_ARG          a NULL argument, the same handle twice, handles on different devices, different input dimensions,
 *                       M <= 0, a non-finite front or ref_point;
 *   LB_ERR_STATE        a model without a kernel;
 *   LB_ERR_UNSUPPORTED  k > LB_EHVI3D_MAX_K (before the front is read).
 * A model without samples scores with its prior.  The three handles are locked for the call and their queries run on their own
 * streams; the means are added as in lb_acq_argmax. */
int lb_ehvi3d_argmax(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k, const double* front_rowmajor,
    int64_t M, const double* Xq_rowmajor, const double* mean0_at_q, double mean0_const, const double* mean1_at_q, double mean1_const,
    const double* mean2_at_q, double mean2_const, double* acq_out, double* best_val, int64_t* best_idx);
/* same, device pointers except ref_point and front; no synchronisation, results on m0's stream */
int lb_ehvi3d_argmax_dev(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k,
    const double* front_rowmajor, int64_t M, const double* dXq_rowmajor, const double* dMean0_at_q, double mean0_const,
    const double* dMean1_at_q, double mean1_const, const double* dMean2_at_q, double mean2_const, double* dAcq_out, double* dBest_val,
    int64_t* dBest_idx);

/* Batched CMA-ES acquisition optimiser (DESIGN.md §4.15): R independent (mu/mu_w, lambda)-CMA-ES instances with the active
 * covariance update, in the default setting of Hansen's tutorial (arXiv:1604.00772, Table 1), sampling through the Cholesky
 * factor of C.  It is not a port of libcmaes (the reference's opt::Cmaes).  One generation of every instance is one batched
 * scoring of R * lambda candidates on the device; ask, score and tell are stream-ordered and the host reads one word every 8
 * generations.  Instance r starts from starts[r] (row-major R x D); bounded searches run in [0, 1]^D through Hansen's
 * linear-quadratic box transform.  An instance stops after `generations` generations, when sigma sqrt(max diag C) < tolx, or when
 * the factorisation of C fails.  Returns the best point scored over every instance and generation (best_x, D values), its value
 * (ties to the lower instance, within an instance to the earlier generation) and the number of candidates scored (n_evals).  The draws come from
 * u(i) = (splitmix64(seed + i) >> 11) 2^-53, so a seed gives the same bits on every run. */
typedef struct lb_cmaes_opts {
    int lambda;       /* offspring per instance, <= 256; <= 0: 4 + floor(3 ln D) */
    double sigma0;    /* initial step size, > 0 (the reference's opt::Cmaes: 0.5) */
    int generations;  /* generations per instance, > 0 */
    double tolx;      /* > 0 */
    uint64_t seed;
    int bounded;      /* nonzero: [0, 1]^D; zero: unbounded */
} lb_cmaes_opts;

/* lb_acq_argmax's UCB / GP_UCB / EI (acq_id, acq_params) with an input-free mean (mean_const added to every mu).  Any precision
 * mode; LB_ERR_TIMEOUT when a reduced-precision scoring pass of any generation timed out.  h is locked for the whole search.
 * LB_ERR_ARG for a NULL argument, R <= 0, a non-finite start, sigma0 or tolx <= 0, generations <= 0 or an unknown acq_id;
 * LB_ERR_UNSUPPORTED for D > 64 or lambda > 256; LB_ERR_STATE for a handle without a kernel.  Synchronises h's stream. */
int lb_acq_cmaes(const lb_gp* h, int acq_id, const double* acq_params, double mean_const, const lb_cmaes_opts* opts, int64_t R,
    const double* starts_rowmajor, double* best_x, double* best_val, int64_t* n_evals);
/* lb_acq_cmaes over lb_acq_argmax_cols's q = P columns: instance r searches column cols[r] (R host ints), so one generation is
 * one query of R lambda candidates, each scored in its instance's column with that column's parameters (acq_params, q x 2) and
 * input-free mean (mean_const, q); every value is lb_acq_argmax_cols's in that column.  best_x (q x D row-major) and best_val (q)
 * hold each column's best point over the instances bound to it (ties to the lower instance); n_evals counts every column.  With
 * q = 1 and every cols[r] = 0 the result is bit-identical to lb_acq_cmaes's for the same options.  fp64 handles only
 * (LB_ERR_UNSUPPORTED otherwise); LB_ERR_ARG for q other than the handle's P, a cols entry outside [0, q), a column without an
 * instance, and lb_acq_cmaes's cases.  h is locked for the whole search; synchronises h's stream. */
int lb_acq_cmaes_cols(const lb_gp* h, int acq_id, int64_t q, const double* acq_params, const double* mean_const, const lb_cmaes_opts* opts,
    int64_t R, const double* starts_rowmajor, const int* cols, double* best_x, double* best_val, int64_t* n_evals);
/* two-objective (m2 NULL, lb_ehvi_argmax, k x 2 front) or three-objective (lb_ehvi3d_argmax, k x 3 front) EHVI with input-free
 * means; the argument and lock rules of those calls (every handle is locked for the whole search), and lb_acq_cmaes's.  The
 * three-objective front pass runs once per search. */
int lb_ehvi_cmaes(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k, const double* front_rowmajor,
    double mean0_const, double mean1_const, double mean2_const, const lb_cmaes_opts* opts, int64_t R, const double* starts_rowmajor,
    double* best_x, double* best_val, int64_t* n_evals);
/* lb_eci_argmax's ECI (eci_params = {f_max, jitter}) with input-free means (obj_mean_const, con_mean_const); every value the
 * search scores is lb_eci_argmax_dev's on the same candidates.  con may be NULL, and a con without samples gives Pf = 1.  An obj
 * without samples scores 0 everywhere: best_x is the first start, best_val 0 and n_evals 0, and nothing is launched (its input
 * dimension must be set, LB_ERR_STATE otherwise).  Both handles are locked for the whole search; LB_ERR_TIMEOUT when a
 * reduced-precision pass of either timed out in any generation.  LB_ERR_ARG for obj == con, handles on different devices or a con
 * with samples and another input dimension, and lb_acq_cmaes's cases; LB_ERR_STATE as lb_eci_argmax. */
int lb_eci_cmaes(const lb_gp* obj, const lb_gp* con, const double* eci_params, double obj_mean_const, double con_mean_const,
    const lb_cmaes_opts* opts, int64_t R, const double* starts_rowmajor, double* best_x, double* best_val, int64_t* n_evals);

/* pareto::impl::pareto_set_std (experimental/tools/pareto.hpp:138-162) over n points of K objectives (row-major n x K): the
 * indices of the points no other point dominates (dominate_flag == 1), duplicates kept, in compare_objs_lex order
 * (lexicographically descending, exact ties by ascending index).  Runs on h's device and stream under h's query lock; h's model
 * state is not touched.  idx has room for n.  LB_ERR_ARG for a non-finite value; LB_ERR_UNSUPPORTED when K > LB_PARETO_MAX_K. */
int lb_pareto_set(const lb_gp* h, int64_t n, int K, const double* objs_rowmajor, int64_t* idx, int64_t* n_front);
/* same, device pointers except n_front (host); synchronises h's stream */
int lb_pareto_set_dev(const lb_gp* h, int64_t n, int K, const double* dObjs_rowmajor, int64_t* dIdx, int64_t* n_front);

/* model::SparsifiedGP::_sparsify (model/sparsified_gp.hpp:121-183): while more than max_points of the N points (row-major N x D)
 * remain, remove the densest one, the point whose k = D nearest remaining neighbours have the smallest sum of Euclidean distances
 * (lowest index on equal sums), until max_points remain or no sum is below DBL_MAX.  Runs on h's device and stream with its pool
 * under h's query lock; h's model state is not touched.  kept (room for N): the n_kept kept indices, ascending; removed /
 * removed_score (room for N - max_points each, may be NULL): the removal order and the sum each removed point had when it was
 * chosen.  N <= max_points keeps every point and launches nothing.  LB_ERR_ARG when max_points < D or a coordinate is not finite
 * (both undefined in the reference); LB_ERR_UNSUPPORTED when D > 64; LB_ERR_TIMEOUT when a device-side wait timed out. */
int lb_sparsify(const lb_gp* h, int64_t N, int D, const double* X_rowmajor, int64_t max_points, int64_t* kept, int64_t* n_kept,
    int64_t* removed, double* removed_score);
/* same, device pointers except n_kept (host); synchronises h's stream */
int lb_sparsify_dev(const lb_gp* h, int64_t N, int D, const double* dX_rowmajor, int64_t max_points, int64_t* dKept,
    int64_t* n_kept, int64_t* dRemoved, double* dRemovedScore);

/* experimental::model::SPGP (experimental/model/spgp.hpp): Snelson and Ghahramani's sparse GP with M pseudo-inputs, single
 * output, SE-ARD.  Same conventions as lb_gp; lb_spgp_query, lb_spgp_acq_argmax, their _dev variants, lb_spgp_acq_cmaes,
 * lb_spgp_query_grad and lb_spgp_acq_grad may be called from several threads, the other calls need exclusive access.  w is the reference's parameter vector (HyperParams, spgp.hpp:94-101) of n_w = (M+1) D + 2
 * entries: [xb (M x D, column-major), log b (D; b = inverse squared length scales), log c (signal variance), log sig (noise
 * variance)].  lb_spgp_lik and lb_spgp_compute return LB_ERR_ARG for M < 1, M > N, n_w != (M+1) D + 2 or a non-finite w, and
 * the 1-based index (> 0) of the first non-positive pivot of Q = K(xb, xb) + jitter I, or else of A = sig I + V V^T. */
typedef struct lb_spgp lb_spgp;
int lb_spgp_create(lb_spgp** out, int device);
int lb_spgp_destroy(lb_spgp* s);
/* SPGP::_init data (spgp.hpp:353-370): N samples (row-major N x D) and y_zm = observations - mean (N).  LB_ERR_UNSUPPORTED
 * when D > 64, LB_ERR_ARG for a non-finite value. */
int lb_spgp_set_data(lb_spgp* s, int64_t N, int D, const double* X_rowmajor, const double* y_zm);
/* SPGP::_likelihood(w, grad != NULL) (spgp.hpp:446-580) with inverse = true: f = -fw and grad = -dfw (n_w entries).  The value
 * keeps the reference's integer (N - M) / 2 in the log(sig) term. */
int lb_spgp_lik(lb_spgp* s, int64_t M, int64_t n_w, const double* w, double jitter, double* f, double* grad);
/* SPGP::_compute(false) (spgp.hpp:389-407) at HyperParams(w): leaves L, Lm and bet on the device for the queries. */
int lb_spgp_compute(lb_spgp* s, int64_t M, int64_t n_w, const double* w, double jitter);
/* SPGP::_predict (spgp.hpp:582-610) for Mq candidates (row-major Mq x D): mu_minus_mean (Mq, without mean(v)) and sigma2 (Mq,
 * + sig when optimized != 0).  LB_ERR_STATE before lb_spgp_compute. */
int lb_spgp_query(const lb_spgp* s, int64_t Mq, const double* Xq_rowmajor, int optimized, double* mu_minus_mean, double* sigma2);
/* same, device pointers; bit-identical to lb_spgp_query on the same candidates.  No synchronisation: the results are ordered on
 * the model's stream, behind which any synchronising lb_spgp_* call or a device synchronisation waits. */
int lb_spgp_query_dev(const lb_spgp* s, int64_t Mq, const double* dXq_rowmajor, int optimized, double* dMu_minus_mean, double* dSigma2);
/* lb_acq_argmax over lb_spgp_query's mu and sigma^2 (ties to the lowest index). */
int lb_spgp_acq_argmax(const lb_spgp* s, int acq_id, const double* acq_params, int64_t Mq, const double* Xq_rowmajor, int optimized,
    const double* mean_at_q, double mean_const, double* acq_out, double* best_val, int64_t* best_idx);
/* same, device pointers except acq_params, as lb_acq_argmax_dev; bit-identical to lb_spgp_acq_argmax on the same candidates.  No
 * synchronisation, results on the model's stream as in lb_spgp_query_dev. */
int lb_spgp_acq_argmax_dev(const lb_spgp* s, int acq_id, const double* acq_params, int64_t Mq, const double* dXq_rowmajor, int optimized,
    const double* dMean_at_q, double mean_const, double* dAcq_out, double* dBest_val, int64_t* dBest_idx);
/* lb_acq_cmaes over the model: lb_spgp_acq_argmax's UCB / GP_UCB / EI with an input-free mean (mean_const); every value the search
 * scores is lb_spgp_acq_argmax_dev's on the same candidates.  The model is locked for the whole search.  LB_ERR_STATE before
 * lb_spgp_compute; LB_ERR_ARG for an unknown acq_id, and lb_acq_cmaes's cases.  Synchronises the model's stream. */
int lb_spgp_acq_cmaes(const lb_spgp* s, int acq_id, const double* acq_params, int optimized, double mean_const, const lb_cmaes_opts* opts,
    int64_t R, const double* starts_rowmajor, double* best_x, double* best_val, int64_t* n_evals);
/* Candidate gradients for Mq candidates (row-major Mq x D), extending lb_spgp_query as lb_query_grad extends lb_query:
 * mu_minus_mean and sigma2 are bit-identical to lb_spgp_query's on the same batch; dmu (Mq x D row-major) is the gradient of
 * mu_minus_mean, dsigma2 (Mq x D) that of sigma2.  With b the inverse squared length scales, x~ = x o sqrt(b), k_m the kernel
 * value at pseudo-input m and x~b_m = xb_m o sqrt(b) (k(x, x) = c does not depend on x):
 *   grad mu = -sqrt(b) o sum_m b1_m k_m (x~ - x~b_m),  b1 = L^-T Lm^-T bet,
 *   grad sigma2 = 2 sqrt(b) o sum_m u_m k_m (x~ - x~b_m),  u = L^-T (L^-1 k - sig Lm^-T Lm^-1 L^-1 k).
 * optimized adds sig to sigma2 and nothing to its gradient.  Any output may be NULL.  LB_ERR_ARG for a NULL handle or Xq_rowmajor,
 * Mq < 1 or a non-finite coordinate; LB_ERR_STATE before lb_spgp_compute.  May be called from several threads, as lb_spgp_query. */
int lb_spgp_query_grad(const lb_spgp* s, int64_t Mq, const double* Xq_rowmajor, int optimized, double* mu_minus_mean, double* sigma2,
    double* dmu, double* dsigma2);
/* Acquisition value (Mq) and gradient (Mq x D row-major) with the FirstElem aggregator, extending lb_spgp_acq_argmax (same acq_id,
 * acq_params, mean_at_q and mean_const; the values are bit-identical to its acq_out) with lb_acq_grad's formulas over
 * lb_spgp_query_grad's gradients: UCB / GP_UCB grad = grad mu + params[0] grad sigma2 / (2 sqrt(sigma2)); EI grad = Phi(Z) grad mu +
 * phi(Z) grad sigma with f_max and the jitter fixed, value and gradient 0 where sigma < 1e-10.  mean_grad_at_q: Mq x D gradient of
 * mean(v)'s first component, added to grad mu, or NULL when the mean does not depend on v.  Either output may be NULL.  LB_ERR_ARG
 * for a NULL handle, acq_params or Xq_rowmajor, Mq < 1, a non-finite coordinate or an unknown acq_id; LB_ERR_STATE before
 * lb_spgp_compute.  May be called from several threads, as lb_spgp_query. */
int lb_spgp_acq_grad(const lb_spgp* s, int acq_id, const double* acq_params, int64_t Mq, const double* Xq_rowmajor, int optimized,
    const double* mean_at_q, double mean_const, const double* mean_grad_at_q, double* acq_out, double* grad_out);
/* kernels launched by this model so far */
long long lb_spgp_launch_count(const lb_spgp* s);

/* GP::compute_log_lik (gp.hpp:267-282) */
int lb_log_lik(lb_gp* h, double* out);
/* GP::compute_kernel_grad_log_lik (gp.hpp:285-311); grad has n_hparams
 * (+1 when optimize_noise, kernel.hpp:86-96) entries. */
int lb_kernel_grad_log_lik(lb_gp* h, int optimize_noise, double* grad);
/* GP::compute_inv_kernel (gp.hpp:254-264) */
int lb_compute_inv_kernel(lb_gp* h);

/* Largest N lb_lml_grad_batch takes (LB_ERR_UNSUPPORTED above): the largest N at which one batched call of 10 vectors beat ten
 * evaluations through lb_set_kernel / lb_fit / lb_log_lik / lb_kernel_grad_log_lik on an H100 (tools/bench_lml_batch.py,
 * DESIGN.md §4.12). */
#define LB_LML_BATCH_MAX_N 200
/* GP::compute_log_lik and GP::compute_kernel_grad_log_lik (gp.hpp:267-311) of this handle's data and obs_mean, evaluated at R
 * kernel states, as KernelLFOptimization (kernel_lf_opt.hpp:77-92) evaluates one:
 *   log_hparams: R x n_hparams row-major, the kernel's own log-space parameters as lb_set_kernel takes them
 *                (SE-ARD Lambda columns inferred from n_hparams as there);
 *   noise:       R values of the signal noise;
 *   lik:         R values;
 *   grad:        R x (n_hparams + optimize_noise) row-major, laid out as lb_kernel_grad_log_lik's; may be NULL (no K^-1, no gradient);
 *   info:        R values, 0 or the 1-based first non-positive pivot of that vector's factor (lik and grad NaN there); may be NULL.
 * One launch; one CTA per vector.  A vector's results do not depend on R or on its place in the batch.  The handle's model state
 * (factor, alpha, caches, kernel) is not touched.  Runs on the handle's stream and pool, under its query lock, in every precision
 * mode (the likelihood is fp64 in all of them).  LB_ERR_STATE without data; LB_ERR_ARG for R <= 0, an unknown kernel id, a wrong
 * n_hparams or a non-finite input; LB_ERR_UNSUPPORTED for N > LB_LML_BATCH_MAX_N or outside the kernels' existing bounds
 * (D + k <= 64, Lambda k <= 4). */
int lb_lml_grad_batch(lb_gp* h, int kernel_id, int64_t R, int n_hparams, const double* log_hparams, const double* noise,
    int optimize_noise, double* lik, double* grad, int* info);
/* same, device pointers (the inputs are read back to the host, where the per-vector kernel state is derived and checked) */
int lb_lml_grad_batch_dev(lb_gp* h, int kernel_id, int64_t R, int n_hparams, const double* dLog_hparams, const double* dNoise,
    int optimize_noise, double* dLik, double* dGrad, int* dInfo);

/* GP::compute_log_loo_cv (gp.hpp:339-351): leave-one-out log predictive probability from diag(K^-1) and alpha */
int lb_log_loo_cv(lb_gp* h, double* out);
/* GP::compute_kernel_grad_log_loo_cv (gp.hpp:353-399), the gradient KernelLooOpt (model/gp/kernel_loo_opt.hpp:57-97)
 * climbs; grad has n_hparams (+1 when optimize_noise) entries. */
int lb_kernel_grad_log_loo_cv(lb_gp* h, int optimize_noise, double* grad);
/* obs_mean^T K^-1 of GP::compute_mean_grad_log_lik (gp.hpp:313-330): out = K^-1 * obs_mean, N x P column-major; the
 * caller contracts it with its mean functor's gradient (mean/mean.hpp:72-76), which is host code. */
int lb_kinv_obs_mean(lb_gp* h, double* out_colmajor);

/* accessors matrixL(), alpha(), ... (gp.hpp:411-436): dst is column-major,
 * N x N (K, L, KINV) or N x P (ALPHA). */
int lb_get(lb_gp* h, int what, double* dst_colmajor);
int64_t lb_nb_samples(const lb_gp* h);

const char* lb_strerror(int code);
/* text of the last CUDA error seen by this library on the calling thread */
const char* lb_last_cuda_error(void);

#ifdef __cplusplus
}
#endif
#endif
