// oracle/limbo_oracle.hpp — TEST INFRASTRUCTURE ONLY.
//
// A dependency-free CPU restatement of the GP hot path of resibots/limbo
// (reference @ 43c67a6), templated on the scalar type (double = the
// reference's arithmetic; long double / __float128 = "truth" used to separate
// ill-conditioning from bugs).  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may use it; the product path
// (limbo_b200/) never includes, links or calls anything in oracle/.
//
// PARITY STATUS: partially pinned.  The reference holds no golden vectors for
// this path (SURVEY.md §8c).  What it does hold — the SE-ARD known answers of
// src/tests/test_kernel.cpp:196-224, the prior-variance check of
// src/tests/test_gp.cpp:697-758 and the property tests of test_gp.cpp — is
// re-stated in tests/test_oracle.py against this file; in addition
// oracle/ref_shim/ compiles the reference's OWN headers (model/gp.hpp,
// kernel/*.hpp, acqui/*.hpp, opt/rprop.hpp) against a minimal Eigen/Boost
// stand-in into oracle/_ref/ and this restatement is checked against that
// (tests/test_oracle_vs_ref.py).  The dense linear algebra itself lives in
// Eigen 3 (un-vendored, un-pinned: ci/install_eigen3.sh:2), so the summation
// order of the Cholesky / triangular solves is "a correct fp64 ordering", not
// a bit-exact target.
//
// Every function cites the reference file:line it follows (paths relative to
// the reference's src/limbo/).
#pragma once
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <vector>

namespace lbo {

enum KernelId { K_SE_ARD = 0, K_MATERN52 = 1, K_MATERN32 = 2, K_EXP = 3 };

template <typename T> inline T t_exp(T x) { using std::exp; return exp(x); }
template <typename T> inline T t_sqrt(T x) { using std::sqrt; return sqrt(x); }
template <typename T> inline T t_log(T x) { using std::log; return log(x); }
template <typename T> inline T t_erfc(T x) { using std::erfc; return erfc(x); }
#ifdef LBO_HAVE_QUAD
extern "C" {
__float128 expq(__float128); __float128 sqrtq(__float128); __float128 logq(__float128); __float128 erfcq(__float128);
}
template <> inline __float128 t_exp(__float128 x) { return expq(x); }
template <> inline __float128 t_sqrt(__float128 x) { return sqrtq(x); }
template <> inline __float128 t_log(__float128 x) { return logq(x); }
template <> inline __float128 t_erfc(__float128 x) { return erfcq(x); }
#endif

// ---------------------------------------------------------------------------
// Kernel functors.  h-params are in log space exactly as the reference keeps
// them (kernel/kernel.hpp:105-123).
// ---------------------------------------------------------------------------
template <typename T>
struct Kernel {
    int id = K_SE_ARD;
    int D = 1;
    std::vector<T> ell; // SE-ARD: exp(p_d)      squared_exp_ard.hpp:96-105
    T l = 1;            // isotropic kernels      matern_five_halves.hpp:97-102
    T sf2 = 1;          // exp(2 p_last)
    T noise = T(0.01);  // kernel/kernel.hpp:57,76-79
    int klam = 0;       // Params::kernel_squared_exp_ard::k(): columns of the Lambda matrix _A (squared_exp_ard.hpp:83,91)
    std::vector<T> A;   // D x klam column-major

    int n_params() const { return id == K_SE_ARD ? D + D * klam + 1 : 2; }

    void set_params(const double* p)
    {
        if (id == K_SE_ARD) { // squared_exp_ard.hpp:96-105
            ell.resize(D);
            for (int d = 0; d < D; ++d) ell[d] = t_exp(T(p[d]));
            A.resize((size_t)D * klam);
            for (int j = 0; j < klam; ++j)
                for (int i = 0; i < D; ++i) A[i + (size_t)j * D] = T(p[(j + 1) * D + i]);
            sf2 = t_exp(T(2.0) * T(p[n_params() - 1]));
        }
        else {
            l = t_exp(T(p[0]));
            sf2 = t_exp(T(2.0) * T(p[1]));
        }
    }

    // pure kernel, no noise (Kernel::kernel of each functor)
    T pure(const T* x1, const T* x2) const
    {
        switch (id) {
        case K_SE_ARD: { // squared_exp_ard.hpp:138-151
            if (klam > 0) return sf2 * t_exp(T(-0.5) * lambda_z(x1, x2));
            T z = 0;
            for (int d = 0; d < D; ++d) {
                T q = (x1[d] - x2[d]) / ell[d];
                z += q * q;
            }
            return sf2 * t_exp(T(-0.5) * z);
        }
        case K_MATERN52: { // matern_five_halves.hpp:104-113
            T s = 0;
            for (int d = 0; d < D; ++d) { T q = x1[d] - x2[d]; s += q * q; }
            T dd = t_sqrt(s);
            T d_sq = dd * dd;
            T l_sq = l * l;
            T term1 = t_sqrt(T(5)) * dd / l;
            T term2 = T(5) * d_sq / (T(3) * l_sq);
            return sf2 * (T(1) + term1 + term2) * t_exp(-term1);
        }
        case K_MATERN32: { // matern_three_halves.hpp:102-108
            T s = 0;
            for (int d = 0; d < D; ++d) { T q = x1[d] - x2[d]; s += q * q; }
            T dd = t_sqrt(s);
            T term = t_sqrt(T(3)) * dd / l;
            return sf2 * (T(1) + term) * t_exp(-term);
        }
        default: { // exp.hpp:94-99
            T s = 0;
            for (int d = 0; d < D; ++d) { T q = x1[d] - x2[d]; s += q * q; }
            T r = s / (l * l);
            return sf2 * t_exp(T(-0.5) * r);
        }
        }
    }

    // squared_exp_ard.hpp:112-114 / :142-146: K = A A^T, K.diagonal() += ell^-2, z = (d^T K) d
    T lambda_z(const T* x1, const T* x2) const
    {
        std::vector<T> Km((size_t)D * D), t(D);
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j) {
                T s = 0;
                for (int c = 0; c < klam; ++c) s += A[i + (size_t)c * D] * A[j + (size_t)c * D];
                Km[i + (size_t)j * D] = s;
            }
        for (int i = 0; i < D; ++i) {
            T inv = T(1) / ell[i];
            Km[i + (size_t)i * D] += inv * inv;
        }
        for (int j = 0; j < D; ++j) {
            T s = 0;
            for (int i = 0; i < D; ++i) s += (x1[i] - x2[i]) * Km[i + (size_t)j * D];
            t[j] = s;
        }
        T z = 0;
        for (int j = 0; j < D; ++j) z += t[j] * (x1[j] - x2[j]);
        return z;
    }

    // BaseKernel::operator()  kernel/kernel.hpp:81-84
    T operator()(const T* x1, const T* x2, long i = -1, long j = -2) const
    {
        return pure(x1, x2) + ((i == j) ? noise + T(1e-8) : T(0));
    }

    // Kernel::gradient (pure part); g has n_params() entries.
    void gradient(const T* x1, const T* x2, T* g) const
    {
        switch (id) {
        case K_SE_ARD: { // squared_exp_ard.hpp:107-136
            if (klam > 0) {
                T k = sf2 * t_exp(T(-0.5) * lambda_z(x1, x2));
                for (int d = 0; d < D; ++d) {
                    T q = (x1[d] - x2[d]) / ell[d];
                    g[d] = q * q * k;
                }
                for (int j = 0; j < klam; ++j) { // :119-122  G = -((x1-x2)^T A.col(j)) * (x1-x2) * k
                    T s = 0;
                    for (int i = 0; i < D; ++i) s += (x1[i] - x2[i]) * A[i + (size_t)j * D];
                    for (int i = 0; i < D; ++i) g[(j + 1) * D + i] = (-s) * (x1[i] - x2[i]) * k;
                }
                g[n_params() - 1] = T(2) * k;
                return;
            }
            T zs = 0;
            for (int d = 0; d < D; ++d) {
                T q = (x1[d] - x2[d]) / ell[d];
                g[d] = q * q;
                zs += g[d];
            }
            T k = sf2 * t_exp(T(-0.5) * zs);
            for (int d = 0; d < D; ++d) g[d] = g[d] * k;
            g[D] = T(2) * k;
            return;
        }
        case K_MATERN52: { // matern_five_halves.hpp:115-133
            T s = 0;
            for (int d = 0; d < D; ++d) { T q = x1[d] - x2[d]; s += q * q; }
            T dd = t_sqrt(s);
            T d_sq = dd * dd;
            T l_sq = l * l;
            T term1 = t_sqrt(T(5)) * dd / l;
            T term2 = T(5) * d_sq / (T(3) * l_sq);
            T r = t_exp(-term1);
            g[0] = sf2 * (r * term1 * (T(1) + term1 + term2) + (-term1 - T(2) * term2) * r);
            g[1] = T(2) * sf2 * (T(1) + term1 + term2) * r;
            return;
        }
        case K_MATERN32: { // matern_three_halves.hpp:110-124
            T s = 0;
            for (int d = 0; d < D; ++d) { T q = x1[d] - x2[d]; s += q * q; }
            T dd = t_sqrt(s);
            T term = t_sqrt(T(3)) * dd / l;
            T r = t_exp(-term);
            g[0] = sf2 * (-term * r + (T(1) + term) * term * r);
            g[1] = T(2) * sf2 * (T(1) + term) * r;
            return;
        }
        default: { // exp.hpp:101-110
            T s = 0;
            for (int d = 0; d < D; ++d) { T q = x1[d] - x2[d]; s += q * q; }
            T r = s / (l * l);
            T k = sf2 * t_exp(T(-0.5) * r);
            g[0] = r * k;
            g[1] = T(2) * k;
            return;
        }
        }
    }
};

// ---------------------------------------------------------------------------
// Dense helpers, column-major (Eigen::MatrixXd default), ld = n.
// ---------------------------------------------------------------------------

// In-place lower Cholesky following the structure of Eigen 3.3/3.4
// LLT.h llt_inplace<Scalar, Lower> (un-vendored; structure restated from the
// published algorithm): unblocked for n < 32, otherwise right-looking blocked
// with blockSize = clamp((n/8)/16*16, 8, 128).  Call site: gp.hpp:565.
// Returns -1 on success, else the index of the failing pivot (like
// Eigen's internal return); the reference never reads it (SURVEY §5).
template <typename T>
long chol_unblocked(T* A, long n, long ld)
{
    for (long k = 0; k < n; ++k) {
        T x = A[k + k * ld];
        for (long p = 0; p < k; ++p) x -= A[k + p * ld] * A[k + p * ld];
        if (!(x > T(0))) return k;
        x = t_sqrt(x);
        A[k + k * ld] = x;
        long rs = n - k - 1;
        if (rs > 0) {
            T* a21 = A + (k + 1) + k * ld;
            for (long p = 0; p < k; ++p) {
                T akp = A[k + p * ld];
                const T* a20 = A + (k + 1) + p * ld;
                for (long i = 0; i < rs; ++i) a21[i] -= a20[i] * akp;
            }
            for (long i = 0; i < rs; ++i) a21[i] /= x;
        }
    }
    return -1;
}

template <typename T>
long chol_blocked(T* A, long n, long ld)
{
    if (n < 32) return chol_unblocked(A, n, ld);
    long bs = n / 8;
    bs = (bs / 16) * 16;
    bs = std::min<long>(std::max<long>(bs, 8), 128);
    for (long k = 0; k < n; k += bs) {
        long b = std::min(bs, n - k);
        long rs = n - k - b;
        T* A11 = A + k + k * ld;
        T* A21 = A + (k + b) + k * ld;
        T* A22 = A + (k + b) + (k + b) * ld;
        long ret = chol_unblocked(A11, b, ld);
        if (ret >= 0) return k + ret;
        if (rs > 0) {
            // A21 = A21 * A11^{-T}   (solve X A11^T = A21, column by column)
            for (long j = 0; j < b; ++j) {
                T* xj = A21 + j * ld;
                for (long p = 0; p < j; ++p) {
                    T l = A11[j + p * ld];
                    const T* xp = A21 + p * ld;
                    for (long i = 0; i < rs; ++i) xj[i] -= xp[i] * l;
                }
                T d = A11[j + j * ld];
                for (long i = 0; i < rs; ++i) xj[i] /= d;
            }
            // A22 -= A21 * A21^T  (lower part only)
            for (long j = 0; j < rs; ++j) {
                T* cj = A22 + j * ld;
                for (long p = 0; p < b; ++p) {
                    T ajp = A21[j + p * ld];
                    const T* ap = A21 + p * ld;
                    for (long i = j; i < rs; ++i) cj[i] -= ap[i] * ajp;
                }
            }
        }
    }
    return -1;
}

// x <- L^{-1} x   (forward substitution, column-oriented as Eigen's
// triangular_solve_vector<..., Lower, ColMajor>; call sites gp.hpp:608,620)
template <typename T>
void trsv_lower(const T* L, long n, long ld, T* x)
{
    for (long j = 0; j < n; ++j) {
        x[j] /= L[j + j * ld];
        T xj = x[j];
        const T* lj = L + j * ld;
        for (long i = j + 1; i < n; ++i) x[i] -= lj[i] * xj;
    }
}

// x <- L^{-T} x  (backward substitution on the adjoint; gp.hpp:610)
template <typename T>
void trsv_lower_t(const T* L, long n, long ld, T* x)
{
    for (long j = n - 1; j >= 0; --j) {
        const T* lj = L + j * ld;
        T s = x[j];
        for (long i = j + 1; i < n; ++i) s -= lj[i] * x[i];
        x[j] = s / lj[j];
    }
}

// ---------------------------------------------------------------------------
// The GP (model/gp.hpp).  The mean function is evaluated by the caller (it is
// arbitrary host code in the reference, mean/mean.hpp:60-77): the oracle takes
// obs_mean = Y - M (gp.hpp:547) and returns mu WITHOUT mean(v) added.
// ---------------------------------------------------------------------------
template <typename T>
struct GP {
    long N = 0;
    int D = 0, P = 0;
    Kernel<T> kern;
    std::vector<T> X;        // N x D row-major (sample i at X[i*D])
    std::vector<T> obs_mean; // N x P col-major
    std::vector<T> K, L, alpha, Kinv;
    bool inv_updated = false;
    long chol_info = -1;

    void set_data(long n, int d, int p, const double* x, const double* om)
    {
        N = n; D = d; P = p;
        X.assign(x, x + n * d);
        obs_mean.assign(om, om + n * p);
    }

    // gp.hpp:550-571  _compute_full_kernel
    void compute_full_kernel()
    {
        K.assign((size_t)N * N, T(0));
        for (long i = 0; i < N; ++i)
            for (long j = 0; j <= i; ++j)
                K[i + j * N] = kern(&X[i * D], &X[j * D], i, j); // gp.hpp:556-558
        for (long i = 0; i < N; ++i)
            for (long j = 0; j < i; ++j)
                K[j + i * N] = K[i + j * N]; // gp.hpp:560-562
        L = K;
        chol_info = chol_blocked(L.data(), N, N); // gp.hpp:565
        for (long j = 0; j < N; ++j) // matrixL() is a dense copy with zero upper part
            for (long i = 0; i < j; ++i) L[i + j * N] = T(0);
        compute_alpha();
        inv_updated = false;
    }

    // gp.hpp:605-611  _compute_alpha
    void compute_alpha()
    {
        alpha = obs_mean;
        for (int p = 0; p < P; ++p) {
            trsv_lower(L.data(), N, N, &alpha[(size_t)p * N]);
            trsv_lower_t(L.data(), N, N, &alpha[(size_t)p * N]);
        }
    }

    // gp.hpp:573-603 _compute_incremental_kernel (after the caller appended the
    // sample and refreshed obs_mean, gp.hpp:139-151)
    void append(const double* x, const double* new_obs_mean)
    {
        long n = N + 1;
        std::vector<T> Kn((size_t)n * n, T(0)), Ln((size_t)n * n, T(0));
        for (long j = 0; j < N; ++j)
            for (long i = 0; i < N; ++i) {
                Kn[i + j * n] = K[i + j * N];
                Ln[i + j * n] = L[i + j * N];
            }
        X.insert(X.end(), x, x + D);
        N = n;
        K.swap(Kn);
        L.swap(Ln);
        obs_mean.assign(new_obs_mean, new_obs_mean + (size_t)n * P);
        for (long i = 0; i < n; ++i) { // gp.hpp:583-586
            K[i + (n - 1) * n] = kern(&X[i * D], &X[(n - 1) * D], i, n - 1);
            K[(n - 1) + i * n] = K[i + (n - 1) * n];
        }
        T L_j;
        for (long j = 0; j < n - 1; ++j) { // gp.hpp:591-594
            T dot = 0;
            for (long p = 0; p < j; ++p) dot += L[j + p * n] * L[(n - 1) + p * n];
            L_j = K[(n - 1) + j * n] - dot;
            L[(n - 1) + j * n] = L_j / L[j + j * n];
        }
        T dot = 0;
        for (long p = 0; p < n - 1; ++p) dot += L[(n - 1) + p * n] * L[(n - 1) + p * n];
        L_j = K[(n - 1) + (n - 1) * n] - dot; // gp.hpp:596-597
        L[(n - 1) + (n - 1) * n] = t_sqrt(L_j);
        compute_alpha();
        inv_updated = false;
    }

    // gp.hpp:626-632 _compute_k ; :613-616 _mu ; :618-624 _sigma ; :159-167 query
    // mu_out: P values (WITHOUT the mean function), *sigma2 includes + noise.
    void query(const double* v_in, T* mu_out, T* sigma2, std::vector<T>& k) const
    {
        std::vector<T> v(v_in, v_in + D);
        if (N == 0) { // gp.hpp:161-163
            for (int p = 0; p < P; ++p) mu_out[p] = T(0);
            *sigma2 = kern(v.data(), v.data()) + kern.noise;
            return;
        }
        k.resize(N);
        for (long i = 0; i < N; ++i) k[i] = kern(&X[i * D], v.data());
        for (int p = 0; p < P; ++p) {
            T s = 0;
            for (long i = 0; i < N; ++i) s += k[i] * alpha[i + (size_t)p * N];
            mu_out[p] = s;
        }
        trsv_lower(L.data(), N, N, k.data());
        T zz = 0;
        for (long i = 0; i < N; ++i) zz += k[i] * k[i];
        T res = kern(v.data(), v.data()) - zz;
        // clamp against the double epsilon whatever T is (gp.hpp:623)
        res = (res <= T(std::numeric_limits<double>::epsilon())) ? T(0) : res;
        *sigma2 = res + kern.noise; // gp.hpp:166
    }

    // gp.hpp:267-282 compute_log_lik
    T log_lik() const
    {
        T logdet = 0;
        for (long i = 0; i < N; ++i) logdet += t_log(L[i + i * N]);
        logdet = T(2) * logdet;
        T a = 0;
        for (int p = 0; p < P; ++p)
            for (long i = 0; i < N; ++i) a += obs_mean[i + (size_t)p * N] * alpha[i + (size_t)p * N];
        const T two_pi = T(6.283185307179586476925286766559005768L);
        return T(-0.5) * a - T(0.5) * logdet - T(0.5) * T(N) * t_log(two_pi);
    }

    // gp.hpp:254-264 compute_inv_kernel: two dense triangular solves on I
    void compute_inv_kernel()
    {
        Kinv.assign((size_t)N * N, T(0));
        for (long j = 0; j < N; ++j) {
            T* col = &Kinv[(size_t)j * N];
            col[j] = T(1);
            // forward solve can start at row j (leading zeros stay zero)
            trsv_lower(L.data() + j + j * N, N - j, N, col + j);
            trsv_lower_t(L.data(), N, N, col);
        }
        inv_updated = true;
    }

    // gp.hpp:285-311 compute_kernel_grad_log_lik (+ BaseKernel::grad kernel.hpp:86-96)
    void kernel_grad_log_lik(T* grad, bool optimize_noise)
    {
        if (!inv_updated) compute_inv_kernel();
        int np = kern.n_params();
        int nh = np + (optimize_noise ? 1 : 0);
        for (int q = 0; q < nh; ++q) grad[q] = T(0);
        std::vector<T> g(nh);
        for (long i = 0; i < N; ++i)
            for (long j = 0; j <= i; ++j) {
                T w = -Kinv[i + j * N];
                for (int p = 0; p < P; ++p) w += alpha[i + (size_t)p * N] * alpha[j + (size_t)p * N];
                kern.gradient(&X[i * D], &X[j * D], g.data());
                if (optimize_noise) g[np] = (i == j) ? T(2) * kern.noise : T(0);
                T f = (i == j) ? T(0.5) : T(1);
                for (int q = 0; q < nh; ++q) grad[q] += w * g[q] * f;
            }
    }

    // gp.hpp:339-351 compute_log_loo_cv
    T log_loo_cv()
    {
        if (!inv_updated) compute_inv_kernel();
        const T two_pi = T(6.283185307179586476925286766559005768L);
        T tot = 0;
        for (int p = 0; p < P; ++p)
            for (long i = 0; i < N; ++i) {
                T inv_diag = T(1) / Kinv[i + i * N];
                T a = alpha[i + (size_t)p * N];
                tot += T(-0.5) * a * a * inv_diag - T(0.5) * t_log(inv_diag) - T(0.5) * t_log(two_pi);
            }
        return tot;
    }

    // gp.hpp:353-399 compute_kernel_grad_log_loo_cv: for every h-param j, Zeta_j = K^-1 dK/dtheta_j and
    // grads(j,p) = sum_i (alpha_ip (Zeta_j alpha)_ip - 0.5 (1 + alpha_ip^2 / Kinv_ii) (Zeta_j K^-1)_ii) / Kinv_ii
    void kernel_grad_log_loo_cv(T* grad, bool optimize_noise)
    {
        if (!inv_updated) compute_inv_kernel();
        const int np = kern.n_params();
        const int nh = np + (optimize_noise ? 1 : 0);
        std::vector<T> dk((size_t)N * N * nh), g(nh);
        for (long i = 0; i < N; ++i)
            for (long j = 0; j <= i; ++j) { // gp.hpp:367-376: lower part from the functor, mirrored
                kern.gradient(&X[i * D], &X[j * D], g.data());
                if (optimize_noise) g[np] = (i == j) ? T(2) * kern.noise : T(0);
                for (int q = 0; q < nh; ++q) dk[(size_t)q * N * N + i + j * N] = dk[(size_t)q * N * N + j + i * N] = g[q];
            }
        std::vector<T> Z((size_t)N * N);
        for (int q = 0; q < nh; ++q) {
            const T* dK = &dk[(size_t)q * N * N];
            for (long i = 0; i < N; ++i)
                for (long l = 0; l < N; ++l) {
                    T s = 0;
                    for (long k = 0; k < N; ++k) s += Kinv[i + k * N] * dK[k + l * N];
                    Z[i + l * N] = s;
                }
            T tot = 0;
            for (int p = 0; p < P; ++p)
                for (long i = 0; i < N; ++i) {
                    T za = 0, zk = 0;
                    for (long l = 0; l < N; ++l) {
                        za += Z[i + l * N] * alpha[l + (size_t)p * N];
                        zk += Z[i + l * N] * Kinv[l + i * N];
                    }
                    const T inv_diag = T(1) / Kinv[i + i * N];
                    const T a = alpha[i + (size_t)p * N];
                    tot += (a * za - T(0.5) * (T(1) + a * a * inv_diag) * zk) * inv_diag;
                }
            grad[q] = tot;
        }
    }

    // the data-dependent factor of gp.hpp:325-327 (compute_mean_grad_log_lik): w(n, p) = obs_mean.col(p)^T * Kinv.col(n)
    void kinv_obs(T* out)
    {
        if (!inv_updated) compute_inv_kernel();
        for (int p = 0; p < P; ++p)
            for (long n = 0; n < N; ++n) {
                T s = 0;
                for (long r = 0; r < N; ++r) s += obs_mean[r + (size_t)p * N] * Kinv[r + n * N];
                out[n + (size_t)p * N] = s;
            }
    }
};

// ---------------------------------------------------------------------------
// Acquisition functions (scalar, FirstElem aggregator = mu[0], bo_base.hpp:99-105)
// ---------------------------------------------------------------------------
// acqui/ucb.hpp:83-90 ; acqui/gp_ucb.hpp:96-103 (same form, alpha := beta)
template <typename T>
inline T ucb(T mu0, T sigma2, T alpha) { return mu0 + alpha * t_sqrt(sigma2); }

// acqui/ei.hpp:85-116
template <typename T>
inline T ei(T mu0, T sigma2, T f_max, T jitter)
{
    T sigma = t_sqrt(sigma2);
    if (sigma < T(1e-10)) return T(0);
    T Xv = mu0 - f_max - jitter;
    T Z = Xv / sigma;
    const T two_pi = T(6.283185307179586476925286766559005768L);
    T phi = t_exp(T(-0.5) * Z * Z) / t_sqrt(two_pi);
    T Phi = T(0.5) * t_erfc(-Z / t_sqrt(T(2)));
    return Xv * Phi + sigma * phi;
}

// acqui/gp_ucb.hpp:83-88
inline double gp_ucb_beta(int iteration, int dim_in, double delta)
{
    double nt = std::pow((double)iteration, dim_in / 2.0 + 2.0);
    double delta3 = delta * 3;
    double pi2 = M_PI * M_PI;
    return std::sqrt(2.0 * std::log(nt * pi2 / delta3));
}

// ---------------------------------------------------------------------------
// opt::Rprop (opt/rprop.hpp:84-144), maximising f; f(params, grad_out) -> value
// ---------------------------------------------------------------------------
template <typename F>
std::vector<double> rprop(F&& f, const std::vector<double>& init, int iterations, double eps_stop, bool bounded,
    long* n_evals = nullptr)
{
    size_t n = init.size();
    double delta0 = 0.1, deltamin = 1e-6, deltamax = 50, etaminus = 0.5, etaplus = 1.2;
    std::vector<double> delta(n, delta0), grad_old(n, 0.0), params(init), grad(n), best_params;
    if (bounded)
        for (size_t j = 0; j < n; ++j) params[j] = std::min(1.0, std::max(0.0, params[j]));
    best_params = params;
    double best = -std::numeric_limits<double>::infinity(); // log(0)
    for (int i = 0; i < iterations; ++i) {
        double lik = f(params, grad.data());
        if (n_evals) ++*n_evals;
        if (lik > best) { best = lik; best_params = params; }
        for (size_t j = 0; j < n; ++j) {
            grad[j] = -grad[j];
            grad_old[j] = grad_old[j] * grad[j];
        }
        for (size_t j = 0; j < n; ++j) {
            if (grad_old[j] > 0) delta[j] = std::min(delta[j] * etaplus, deltamax);
            else if (grad_old[j] < 0) { delta[j] = std::max(delta[j] * etaminus, deltamin); grad[j] = 0; }
            int sg = (0.0 < grad[j]) - (grad[j] < 0.0); // tools/math.hpp:71-91
            params[j] += -sg * delta[j];
            if (bounded && params[j] < 0) params[j] = 0;
            if (bounded && params[j] > 1) params[j] = 1;
        }
        grad_old = grad;
        double nrm = 0;
        for (size_t j = 0; j < n; ++j) nrm += grad_old[j] * grad_old[j];
        if (std::sqrt(nrm) < eps_stop) break;
    }
    return best_params;
}

} // namespace lbo
