// limbo_b200/csrc/cmaes.cu — the batched CMA-ES of lb_acq_cmaes / lb_ehvi_cmaes (DESIGN.md §4.15).
//
// (mu/mu_w, lambda)-CMA-ES with the active covariance update in the default setting of Hansen, "The CMA Evolution Strategy: A
// Tutorial" (arXiv:1604.00772, Table 1 and Fig. 6), sampling through the Cholesky factor A of C instead of an eigendecomposition.
// It is not a port of libcmaes.  R independent instances advance in lockstep, one generation of all of them being one batched
// scoring of R * lambda candidates:
//   cmaes_ask_kernel   one CTA per offspring: z ~ N(0, I) from the splitmix64 stream, y = A z, x = m + sigma y, and the
//                      phenotype T(x) straight into the scorer's candidate buffer
//   cmaes_tell_kernel  one CTA per instance: rank the lambda values, recombine, update p_sigma, sigma, p_c and C, refactor A in
//                      shared memory, track the best phenotype and set the stop flag
// Every sum runs in a fixed order, so a seed gives the same bits on every run.
#include "../../include/limbo_b200.h"
#include "common.cuh"
#include <algorithm>
#include <cmath>

namespace {

// state offsets of one instance (lb_cmaes_state_doubles)
struct StateLayout {
    int D;
    __host__ __device__ int m() const { return 0; }
    __host__ __device__ int ps() const { return D; }
    __host__ __device__ int pc() const { return 2 * D; }
    __host__ __device__ int bx() const { return 3 * D; }
    __host__ __device__ int C() const { return 4 * D; }
    __host__ __device__ int A() const { return 4 * D + D * D; }
    __host__ __device__ int sigma() const { return 4 * D + 2 * D * D; }
    __host__ __device__ int bv() const { return sigma() + 1; }
    __host__ __device__ int stop() const { return sigma() + 2; }
};

__device__ __forceinline__ uint64_t splitmix64(uint64_t x)
{
    uint64_t z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ double unif(uint64_t seed, uint64_t i) { return (double)(splitmix64(seed + i) >> 11) * (1.0 / 9007199254740992.0); }

// Hansen's linear-quadratic box transform onto [lb, ub]
__host__ __device__ inline void box_widths(double lb, double ub, double* al, double* au)
{
    *al = fmin((ub - lb) / 2.0, (1.0 + fabs(lb)) / 20.0);
    *au = fmin((ub - lb) / 2.0, (1.0 + fabs(ub)) / 20.0);
}
__device__ double box_transform(double x, double lb, double ub)
{
    double al, au;
    box_widths(lb, ub, &al, &au);
    const double r = 2.0 * (ub - lb + al + au);
    const double xlow = lb - 2.0 * al - (ub - lb) / 2.0, xup = ub + 2.0 * au + (ub - lb) / 2.0;
    if (x < xlow) x += r * (1.0 + floor((xlow - x) / r));
    if (x > xup) x -= r * (1.0 + floor((x - xup) / r));
    if (x < lb - al) x += 2.0 * (lb - al - x);
    if (x > ub + au) x -= 2.0 * (x - ub - au);
    if (x < lb + al) {
        const double t = x - lb + al;
        x = lb + t * t / (4.0 * al);
    } else if (x > ub - au) {
        const double t = x - ub - au;
        x = ub - t * t / (4.0 * au);
    }
    return x;
}

__global__ void __launch_bounds__(LB_CMAES_MAX_D) cmaes_ask_kernel(LbCmaes s, int g)
{
    __shared__ double zs[LB_CMAES_MAX_D];
    const int D = s.D, d = threadIdx.x;
    const int64_t off = (int64_t)blockIdx.x; // r lam + k
    const int r = (int)(off / s.lam);
    const StateLayout L{D};
    const double* st = s.state + r * lb_cmaes_state_doubles(D);
    if (d < D) {
        const uint64_t c = (((uint64_t)g * s.R * s.lam) + (uint64_t)off) * D + d;
        const double u1 = unif(s.seed, 2 * c), u2 = unif(s.seed, 2 * c + 1);
        zs[d] = sqrt(-2.0 * log(1.0 - u1)) * cos(2.0 * 3.141592653589793 * u2);
    }
    __syncthreads();
    if (d >= D) return;
    const double* A = st + L.A() + (int64_t)d * D;
    double y = 0.0;
    for (int j = 0; j <= d; ++j) y = fma(A[j], zs[j], y);
    const double x = st[L.m() + d] + st[L.sigma()] * y;
    s.z[off * D + d] = zs[d];
    s.y[off * D + d] = y;
    s.cand[off * D + d] = s.bounded ? box_transform(x, 0.0, 1.0) : x;
}

constexpr int TELL_T = 256;

// offspring j ranks before k: the larger value, NaN last, ties to the lower index
__device__ __forceinline__ bool ranks_before(double vj, int j, double vk, int k)
{
    const bool nj = isnan(vj), nk = isnan(vk);
    if (nj != nk) return nk;
    if (!nj && vj != vk) return vj > vk;
    return j < k;
}

__global__ void __launch_bounds__(TELL_T) cmaes_tell_kernel(LbCmaes s, int g, const double* __restrict__ vals, int* live)
{
    __shared__ double Cs[LB_CMAES_MAX_D * LB_CMAES_MAX_D];
    __shared__ double v[LB_CMAES_MAX_LAMBDA], wo[LB_CMAES_MAX_LAMBDA];
    __shared__ int order[LB_CMAES_MAX_LAMBDA];
    __shared__ double yw[LB_CMAES_MAX_D];
    __shared__ double hs_s, nps_s;
    __shared__ int fail;
    const int r = blockIdx.x, t = threadIdx.x, D = s.D, lam = s.lam, mu = s.mu;
    const StateLayout L{D};
    double* st = s.state + r * lb_cmaes_state_doubles(D);
    if (st[L.stop()] != 0.0) return;
    const double* Z = s.z + (int64_t)r * lam * D;
    const double* Y = s.y + (int64_t)r * lam * D;
    for (int k = t; k < lam; k += TELL_T) v[k] = vals[(int64_t)r * lam + k];
    if (t == 0) fail = 0;
    __syncthreads();
    for (int k = t; k < lam; k += TELL_T) {
        int rank = 0;
        for (int j = 0; j < lam; ++j) rank += ranks_before(v[j], j, v[k], k);
        order[rank] = k;
    }
    __syncthreads();
    const double sigma = st[L.sigma()];
    {   // the best phenotype so far
        const int j = order[0];
        const bool better = v[j] > st[L.bv()];
        __syncthreads(); // every thread has read best_val before thread 0 writes it
        if (better) {
            for (int d = t; d < D; d += TELL_T) st[L.bx() + d] = s.cand[((int64_t)r * lam + j) * D + d];
            if (t == 0) st[L.bv()] = v[j];
        }
    }
    for (int d = t; d < D; d += TELL_T) {
        double sy = 0.0, sz = 0.0;
        for (int i = 0; i < mu; ++i) {
            const int64_t o = (int64_t)order[i] * D + d;
            sy = fma(s.w[i], Y[o], sy);
            sz = fma(s.w[i], Z[o], sz);
        }
        yw[d] = sy;
        st[L.m() + d] += sigma * sy;
        st[L.ps() + d] = (1.0 - s.cs) * st[L.ps() + d] + sqrt(s.cs * (2.0 - s.cs) * s.mueff) * sz;
    }
    for (int i = t; i < lam; i += TELL_T) {
        if (i < mu) {
            wo[i] = s.w[i];
        } else {
            double n2 = 0.0;
            const double* zi = Z + (int64_t)order[i] * D;
            for (int d = 0; d < D; ++d) n2 = fma(zi[d], zi[d], n2);
            wo[i] = s.w[i] * D / n2;
        }
    }
    __syncthreads();
    if (t == 0) {
        double n2 = 0.0;
        for (int d = 0; d < D; ++d) n2 = fma(st[L.ps() + d], st[L.ps() + d], n2);
        const double nps = sqrt(n2);
        nps_s = nps;
        hs_s = nps / sqrt(1.0 - pow(1.0 - s.cs, 2.0 * (g + 1))) < (1.4 + 2.0 / (D + 1.0)) * s.chi ? 1.0 : 0.0;
    }
    __syncthreads();
    const double hs = hs_s;
    for (int d = t; d < D; d += TELL_T)
        st[L.pc() + d] = (1.0 - s.cc) * st[L.pc() + d] + hs * sqrt(s.cc * (2.0 - s.cc) * s.mueff) * yw[d];
    __syncthreads();
    // C <- coef C + c1 p_c p_c^T + c_mu sum_i wo_i y_i y_i^T over the lower triangle, mirrored
    const double coef = 1.0 + s.c1 * (1.0 - hs) * s.cc * (2.0 - s.cc) - s.c1 - s.cmu * s.sumw;
    const double* pc = st + L.pc();
    double* C = st + L.C();
    for (int e = t; e < D * D; e += TELL_T) {
        const int a = e / D, b = e % D;
        if (b > a) continue;
        double acc = 0.0;
        for (int i = 0; i < lam; ++i) {
            const double* yi = Y + (int64_t)order[i] * D;
            acc = fma(wo[i] * yi[a], yi[b], acc);
        }
        const double c = coef * C[a * D + b] + s.c1 * pc[a] * pc[b] + s.cmu * acc;
        Cs[a * D + b] = c;
        Cs[b * D + a] = c;
    }
    __syncthreads();
    for (int e = t; e < D * D; e += TELL_T) C[e] = Cs[e];
    double sigma_new = 0.0;
    if (t == 0) {
        sigma_new = sigma * exp(s.cs / s.ds * (nps_s / s.chi - 1.0));
        st[L.sigma()] = sigma_new;
    }
    __syncthreads();
    // A = chol(C), right-looking in shared memory
    for (int j = 0; j < D; ++j) {
        if (t == 0) {
            const double p = Cs[j * D + j];
            if (!(p > 0.0)) fail = 1;
            Cs[j * D + j] = sqrt(p);
        }
        __syncthreads();
        if (fail) break;
        const double piv = Cs[j * D + j];
        for (int i = j + 1 + t; i < D; i += TELL_T) Cs[i * D + j] /= piv;
        __syncthreads();
        const int n = D - j - 1;
        for (int e = t; e < n * n; e += TELL_T) {
            const int i = j + 1 + e / n, k = j + 1 + e % n;
            if (k <= i) Cs[i * D + k] -= Cs[i * D + j] * Cs[k * D + j];
        }
        __syncthreads();
    }
    if (fail) {
        if (t == 0) st[L.stop()] = 1.0;
        return;
    }
    for (int e = t; e < D * D; e += TELL_T) st[L.A() + e] = (e % D <= e / D) ? Cs[e] : 0.0;
    if (t == 0) {
        double cmax = C[0];
        for (int d = 1; d < D; ++d) cmax = fmax(cmax, C[d * D + d]);
        const bool stop = !isfinite(sigma_new) || !(sigma_new * sqrt(cmax) >= s.tolx);
        if (stop) st[L.stop()] = 1.0;
        else if (live) atomicAdd(live, 1);
    }
}

__global__ void cmaes_flag_kernel(const int* err, int* flag)
{
    if (*err) *flag = 1;
}

} // namespace

int lb_cmaes_setup(const lb_cmaes_opts& o, int D, int R, LbCmaes* s, std::vector<double>* w)
{
    if (R <= 0 || D <= 0 || !std::isfinite(o.sigma0) || !(o.sigma0 > 0.0) || !std::isfinite(o.tolx) || !(o.tolx > 0.0) || o.generations <= 0)
        return LB_ERR_ARG;
    if (D > LB_CMAES_MAX_D || o.lambda > LB_CMAES_MAX_LAMBDA) return LB_ERR_UNSUPPORTED;
    const int lam = o.lambda > 0 ? o.lambda : 4 + (int)std::floor(3.0 * std::log((double)D));
    if (lam < 2) return LB_ERR_ARG;
    const int mu = lam / 2;
    w->assign((size_t)lam, 0.0);
    double sp = 0.0, sp2 = 0.0, sn = 0.0, sn2 = 0.0, sna = 0.0;
    for (int i = 0; i < lam; ++i) {
        const double wp = std::log((lam + 1) / 2.0) - std::log((double)(i + 1));
        (*w)[(size_t)i] = wp;
        if (i < mu) { sp += wp; sp2 += wp * wp; }
        else { sn += wp; sn2 += wp * wp; sna += std::fabs(wp); }
    }
    const double n = D;
    const double mueff = sp * sp / sp2;
    const double mueff_neg = sna > 0.0 ? sn * sn / sn2 : 0.0;
    s->R = R; s->D = D; s->lam = lam; s->mu = mu; s->bounded = o.bounded != 0; s->seed = o.seed; s->tolx = o.tolx;
    s->mueff = mueff;
    s->cc = (4.0 + mueff / n) / (n + 4.0 + 2.0 * mueff / n);
    s->cs = (mueff + 2.0) / (n + mueff + 5.0);
    s->c1 = 2.0 / ((n + 1.3) * (n + 1.3) + mueff);
    // c_mu as in arXiv:1604.00772v1 (2016), Table 1, alpha_cov = 2; later revisions add 1/4 to the numerator.  The NumPy
    // restatement of the tests states the same form.
    s->cmu = std::fmin(1.0 - s->c1, 2.0 * (mueff - 2.0 + 1.0 / mueff) / ((n + 2.0) * (n + 2.0) + mueff));
    s->ds = 1.0 + 2.0 * std::fmax(0.0, std::sqrt((mueff - 1.0) / (n + 1.0)) - 1.0) + s->cs;
    s->chi = std::sqrt(n) * (1.0 - 1.0 / (4.0 * n) + 1.0 / (21.0 * n * n));
    const double a_mu = s->cmu > 0.0 ? 1.0 + s->c1 / s->cmu : INFINITY;
    const double a_mueff = 1.0 + 2.0 * mueff_neg / (mueff + 2.0);
    const double a_posdef = s->cmu > 0.0 ? (1.0 - s->c1 - s->cmu) / (n * s->cmu) : INFINITY;
    const double neg = sna > 0.0 ? std::fmin(a_mu, std::fmin(a_mueff, a_posdef)) / sna : 0.0;
    double sumw = 0.0;
    for (int i = 0; i < lam; ++i) {
        double& wi = (*w)[(size_t)i];
        wi = i < mu ? wi / sp : neg * wi;
        sumw += wi;
    }
    s->sumw = sumw;
    return LB_OK;
}

void lb_cmaes_init_state(const LbCmaes& s, double sigma0, const double* start, double* st)
{
    const int D = s.D;
    const StateLayout L{D};
    std::fill(st, st + lb_cmaes_state_doubles(D), 0.0);
    double al, au;
    box_widths(0.0, 1.0, &al, &au);
    for (int d = 0; d < D; ++d) {
        double x = start[d];
        if (s.bounded) { // T^-1 of the start, clipped into the box
            x = std::fmin(std::fmax(x, 0.0), 1.0);
            st[L.bx() + d] = x;
            if (x < al) x = -al + 2.0 * std::sqrt(al * x);
            else if (x > 1.0 - au) x = 1.0 + au - 2.0 * std::sqrt(au * (1.0 - x));
        } else {
            st[L.bx() + d] = x;
        }
        st[L.m() + d] = x;
        st[L.C() + d * D + d] = 1.0;
        st[L.A() + d * D + d] = 1.0;
    }
    st[L.sigma()] = sigma0;
    st[L.bv()] = -INFINITY;
}

int lb_launch_cmaes_ask(cudaStream_t st, const LbCmaes& s, int g, long long* launches)
{
    cmaes_ask_kernel<<<(unsigned)(s.R * s.lam), LB_CMAES_MAX_D, 0, st>>>(s, g);
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_cmaes_tell(cudaStream_t st, const LbCmaes& s, int g, const double* dVals, int* dLive, long long* launches)
{
    cmaes_tell_kernel<<<(unsigned)s.R, TELL_T, 0, st>>>(s, g, dVals, dLive);
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_cmaes_flag(cudaStream_t st, const int* dErr, int* dFlag, long long* launches)
{
    cmaes_flag_kernel<<<1, 1, 0, st>>>(dErr, dFlag);
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
