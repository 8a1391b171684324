// limbo_b200/csrc/ehvi.cu — two-objective expected hypervolume improvement and the Pareto filter of the multi-objective loop.
//
// Replaces, for a batch of M candidates at once, the one-point-at-a-time
//   experimental::acqui::Ehvi (experimental/acqui/ehvi.hpp:70-79) over ehvi2d (src/ehvi/ehvi_calculations.cc:16-79)
//                                           -> ehvi_kernel + the 256-wide block argmax (query.cu)
//   pareto::impl::pareto_set_std<K>'s O(n^2 K) domination test (experimental/tools/pareto.hpp:138-162)
//                                           -> pareto_kernel (the final lexicographic sort runs on the host, abi.cu)
//
// ehvi2d sums (k+1)(k+2)/2 grid cells over a front of k points sorted by f[0].  Cell (i, j), i = 0..k, j = k-i..k, has the
// bounds cl1 = bx[j], cu1 = bx[j+1] and cl2 = by[i], cu2 = by[i+1] with
//   bx = (r0, f0[0], ..., f0[k-1], +inf),   by = (r1, f1[k-1], ..., f1[0], +inf),
// and the staircase corner fmax = (i == k ? r0 : f0[k-i-1], j == k ? r1 : f1[j]).  exipsi(a, c, m, s) = s phi((c-m)/s) +
// (a - m) Phi((c-m)/s) is linear in a, so per candidate the kernel evaluates s phi and Phi once at each of the 2 (k+2) bounds
// (helper.cc's gausspdf / gausscdf with its truncated constants) and every cell is then a handful of fp64 FMAs.  Sminus (the
// correction term) depends on the front only; it is accumulated along each row in the reference's order.
#include "../../include/limbo_b200.h"
#include "common.cuh"
#include <algorithm>
#include <cfloat>
#include <math_constants.h>

namespace {

// helper.cc / ehvi_consts.h: the reference's truncated constants, not M_SQRT2 / M_2_SQRTPI
constexpr double SQRT_TWO = 1.41421356237;
constexpr double SQRT_TWOPI_NEG = 0.3989422804;

// One CTA of 256 threads scores 256 / T candidates; a team of T threads (T a power of two) owns one candidate.  Thread `lane`
// of a team takes the row pairs (p, k - p), p = lane, lane + T, ..., so that every pair has k + 2 cells (a row i has i + 1).
// Dynamic shared memory: per team, (s phi, Phi) at the k + 2 x-bounds, then at the k + 2 y-bounds (double2 each).
__device__ __forceinline__ double ehvi_row(int64_t i, int64_t k, const double2* __restrict__ F, double r0, double r1, double m0, double m1,
    const double2* __restrict__ tx, const double2* __restrict__ ty)
{
    const double fmax0 = (i == k) ? r0 : __ldg(&F[k - i - 1].x);
    const double am = fmax0 - m0;
    const double2 yl = ty[i], yu = ty[i + 1];
    const double cdf2 = yu.y - yl.y;
    const int64_t j0 = k - i;
    double2 xl = tx[j0];
    double2 fprev = make_double2(0.0, 0.0); // F[j - 1]
    double S = 0.0, acc = 0.0;
    for (int64_t j = j0; j <= k; ++j) {
        const double2 xu = tx[j + 1];
        const double2 fj = (j < k) ? __ldg(&F[j]) : make_double2(0.0, r1);
        const double fmax1 = fj.y;
        if (j > j0) S += (fprev.x - fmax0) * (fprev.y - fmax1); // ehvi_calculations.cc:62-65, sequential in j
        const double psi1 = (xl.x + am * xl.y) - (xu.x + am * xu.y);
        const double bm = fmax1 - m1;
        const double psi2 = (yl.x + bm * yl.y) - (yu.x + bm * yu.y);
        const double cdf1 = xu.y - xl.y;
        const double sum = (psi1 * psi2) - (S * cdf1 * cdf2);
        if (sum > 0) acc += sum; // a NaN cell adds nothing
        xl = xu;
        fprev = fj;
    }
    return acc;
}

// (s phi(t), Phi(t)) at t = (c - m) / s (helper.cc:17-26); the bound c = +inf gives (0, 1), as the reference's arithmetic does
// for s > 0
__device__ __forceinline__ double2 bound_terms(bool inf, double c, double m, double s)
{
    if (inf) return make_double2(0.0, 1.0);
    const double t = (c - m) / s;
    return make_double2(s * (SQRT_TWOPI_NEG * exp(-(t * t) / 2)), 0.5 * (1 + erf(t / SQRT_TWO)));
}

__global__ void __launch_bounds__(256)
ehvi_kernel(int T, int64_t k, const double2* __restrict__ F, double r0, double r1, int64_t M, const double* __restrict__ mu0, int p0,
    const double* __restrict__ mean0, double mean0_const, const double* __restrict__ s2_0, const double* __restrict__ mu1, int p1,
    const double* __restrict__ mean1, double mean1_const, const double* __restrict__ s2_1, double* __restrict__ acq)
{
    extern __shared__ double2 tab[];
    __shared__ double red[256];
    const int team = threadIdx.x / T, lane = threadIdx.x % T;
    const int64_t q = (int64_t)blockIdx.x * (256 / T) + team;
    const int64_t nb = k + 2;
    double2* tx = tab + (size_t)team * 2 * nb;
    double2* ty = tx + nb;
    double m0 = 0.0, m1 = 0.0;
    if (q < M) {
        // acqui/ehvi.hpp:75-76: FirstElem of each model's mu, and sigma() (sigma^2 + noise) where ehvi2d expects a deviation
        m0 = mu0[q * p0] + (mean0 ? mean0[q] : mean0_const);
        m1 = mu1[q * p1] + (mean1 ? mean1[q] : mean1_const);
        const double s0 = s2_0[q], s1 = s2_1[q];
        for (int64_t b = lane; b < 2 * nb; b += T) {
            if (b < nb) tx[b] = bound_terms(b > k, b == 0 ? r0 : (b <= k ? __ldg(&F[b - 1].x) : 0.0), m0, s0);
            else {
                const int64_t t = b - nb;
                ty[t] = bound_terms(t > k, t == 0 ? r1 : (t <= k ? __ldg(&F[k - t].y) : 0.0), m1, s1);
            }
        }
    }
    __syncthreads();
    double acc = 0.0;
    if (q < M) {
        for (int64_t p = lane; 2 * p <= k; p += T) {
            acc += ehvi_row(p, k, F, r0, r1, m0, m1, tx, ty);
            if (k - p != p) acc += ehvi_row(k - p, k, F, r0, r1, m0, m1, tx, ty);
        }
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = T / 2; o > 0; o >>= 1) { // fixed tree per team: repeat calls are bit-identical
        if (lane < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (q < M && lane == 0) acq[q] = red[threadIdx.x];
}

// ---- candidate gradient ------------------------------------------------------------------------------------------------
// d/d(m0, s0, m1, s1) of one candidate's ehvi2d, chained with the models' input gradients.  A table entry (a, b) = (s phi(t),
// Phi(t)), t = (c - m) / s, has (phi = gausspdf, documented as the derivative of gausscdf to about 1e-11 relative)
//   da/dm = t a / s,  da/ds = a (1 + t^2) / s,  db/dm = -a / s^2,  db/ds = -t a / s^2,
// all 0 at c = +inf (stored as a = 0, t = 0).  Per cell sum = psi1 psi2 - S cdf1 cdf2 with am = fmax0 - m0 inside psi1 (so
// dpsi1/dm0 gains -b at each bound) and bm = fmax1 - m1 inside psi2.  A cell adds to the partials only where it adds to the
// value (sum > 0).  The value is ehvi_row's, in its order of operations.

// the four partials of one table entry, from (a, b), t and 1/s
struct BoundGrad { double am, as, bm, bs; };
__device__ __forceinline__ BoundGrad bound_grad(double a, double t, double is)
{
    const double bm = -a * is * is;
    return {t * a * is, a * fma(t, t, 1.0) * is, bm, t * bm};
}

// bound_terms and t; t = 0 wherever a = 0 (every partial carries a factor a), which keeps t^2 finite far in the tails
__device__ __forceinline__ double2 bound_terms_t(bool inf, double c, double m, double s, double* tout)
{
    if (inf) {
        *tout = 0.0;
        return make_double2(0.0, 1.0);
    }
    const double t = (c - m) / s;
    const double2 r = make_double2(s * (SQRT_TWOPI_NEG * exp(-(t * t) / 2)), 0.5 * (1 + erf(t / SQRT_TWO)));
    *tout = (r.x == 0.0) ? 0.0 : t;
    return r;
}

struct EhviPartials { double m0, s0, m1, s1; };

// ehvi_row's value (returned, same operations) and the row's partials (added to g)
__device__ __forceinline__ double ehvi_row_grad(int64_t i, int64_t k, const double2* __restrict__ F, double r0, double r1, double m0,
    double m1, double is0, double is1, const double2* __restrict__ tx, const double2* __restrict__ ty, const double* __restrict__ ttx,
    const double* __restrict__ tty, EhviPartials& g)
{
    const double fmax0 = (i == k) ? r0 : __ldg(&F[k - i - 1].x);
    const double am = fmax0 - m0;
    const double2 yl = ty[i], yu = ty[i + 1];
    const double cdf2 = yu.y - yl.y;
    const BoundGrad gyl = bound_grad(yl.x, tty[i], is1), gyu = bound_grad(yu.x, tty[i + 1], is1);
    const double dcdf2_m = gyu.bm - gyl.bm, dcdf2_s = gyu.bs - gyl.bs;
    const int64_t j0 = k - i;
    double2 xl = tx[j0];
    BoundGrad gxl = bound_grad(xl.x, ttx[j0], is0);
    double2 fprev = make_double2(0.0, 0.0); // F[j - 1]
    double S = 0.0, acc = 0.0;
    for (int64_t j = j0; j <= k; ++j) {
        const double2 xu = tx[j + 1];
        const BoundGrad gxu = bound_grad(xu.x, ttx[j + 1], is0);
        const double2 fj = (j < k) ? __ldg(&F[j]) : make_double2(0.0, r1);
        const double fmax1 = fj.y;
        if (j > j0) S += (fprev.x - fmax0) * (fprev.y - fmax1);
        const double psi1 = (xl.x + am * xl.y) - (xu.x + am * xu.y);
        const double bm = fmax1 - m1;
        const double psi2 = (yl.x + bm * yl.y) - (yu.x + bm * yu.y);
        const double cdf1 = xu.y - xl.y;
        const double sum = (psi1 * psi2) - (S * cdf1 * cdf2);
        if (sum > 0) {
            acc += sum;
            const double dpsi1_m = (gxl.am + am * gxl.bm - xl.y) - (gxu.am + am * gxu.bm - xu.y);
            const double dpsi1_s = (gxl.as + am * gxl.bs) - (gxu.as + am * gxu.bs);
            const double dpsi2_m = (gyl.am + bm * gyl.bm - yl.y) - (gyu.am + bm * gyu.bm - yu.y);
            const double dpsi2_s = (gyl.as + bm * gyl.bs) - (gyu.as + bm * gyu.bs);
            const double Sc2 = S * cdf2, Sc1 = S * cdf1;
            g.m0 += dpsi1_m * psi2 - Sc2 * (gxu.bm - gxl.bm);
            g.s0 += dpsi1_s * psi2 - Sc2 * (gxu.bs - gxl.bs);
            g.m1 += psi1 * dpsi2_m - Sc1 * dcdf2_m;
            g.s1 += psi1 * dpsi2_s - Sc1 * dcdf2_s;
        }
        xl = xu;
        gxl = gxu;
        fprev = fj;
    }
    return acc;
}

// ehvi_kernel's teams, row pairs and reduction tree, with t beside every table entry and four more reductions.  Dynamic shared
// memory: the (a, b) tables of every team (as ehvi_kernel), then the t tables of every team.  Then
//   grad EHVI = dm0 grad mu0 + ds0 grad sigma^2_0 + dm1 grad mu1 + ds1 grad sigma^2_1
// (s = sigma^2 + noise stands where ehvi2d expects a deviation, so ds/dx = grad sigma^2); a model with s <= 0 adds nothing.
__global__ void __launch_bounds__(256)
ehvi_grad_kernel(int T, int64_t k, const double2* __restrict__ F, double r0, double r1, int64_t M, int D, const LbPairModel g0,
    const LbPairModel g1, double* __restrict__ acq, double* __restrict__ grad)
{
    extern __shared__ double2 tab[];
    __shared__ double red[5][256];
    const int team = threadIdx.x / T, lane = threadIdx.x % T;
    const int64_t q = (int64_t)blockIdx.x * (256 / T) + team;
    const int64_t nb = k + 2;
    double2* tx = tab + (size_t)team * 2 * nb;
    double2* ty = tx + nb;
    double* ttx = reinterpret_cast<double*>(tab + (size_t)(256 / T) * 2 * nb) + (size_t)team * 2 * nb;
    double* tty = ttx + nb;
    double m0 = 0.0, m1 = 0.0, s0 = 0.0, s1 = 0.0;
    if (q < M) {
        m0 = g0.mu[q * g0.p] + (g0.mean ? g0.mean[q] : g0.mean_const);
        m1 = g1.mu[q * g1.p] + (g1.mean ? g1.mean[q] : g1.mean_const);
        s0 = g0.s2[q];
        s1 = g1.s2[q];
        for (int64_t b = lane; b < 2 * nb; b += T) {
            if (b < nb) tx[b] = bound_terms_t(b > k, b == 0 ? r0 : (b <= k ? __ldg(&F[b - 1].x) : 0.0), m0, s0, &ttx[b]);
            else {
                const int64_t t = b - nb;
                ty[t] = bound_terms_t(t > k, t == 0 ? r1 : (t <= k ? __ldg(&F[k - t].y) : 0.0), m1, s1, &tty[t]);
            }
        }
    }
    __syncthreads();
    double acc = 0.0;
    EhviPartials g = {0.0, 0.0, 0.0, 0.0};
    if (q < M) {
        const double is0 = 1.0 / s0, is1 = 1.0 / s1;
        for (int64_t p = lane; 2 * p <= k; p += T) {
            acc += ehvi_row_grad(p, k, F, r0, r1, m0, m1, is0, is1, tx, ty, ttx, tty, g);
            if (k - p != p) acc += ehvi_row_grad(k - p, k, F, r0, r1, m0, m1, is0, is1, tx, ty, ttx, tty, g);
        }
    }
    red[0][threadIdx.x] = acc;
    red[1][threadIdx.x] = g.m0;
    red[2][threadIdx.x] = g.s0;
    red[3][threadIdx.x] = g.m1;
    red[4][threadIdx.x] = g.s1;
    __syncthreads();
    for (int o = T / 2; o > 0; o >>= 1) { // ehvi_kernel's tree
        if (lane < o)
#pragma unroll
            for (int r = 0; r < 5; ++r) red[r][threadIdx.x] += red[r][threadIdx.x + o];
        __syncthreads();
    }
    if (q >= M) return;
    const int lead = team * T;
    if (lane == 0 && acq) acq[q] = red[0][lead];
    if (!grad) return;
    const bool live0 = s0 > 0.0, live1 = s1 > 0.0;
    const double pm0 = live0 ? red[1][lead] : 0.0, ps0 = live0 ? red[2][lead] : 0.0;
    const double pm1 = live1 ? red[3][lead] : 0.0, ps1 = live1 ? red[4][lead] : 0.0;
    for (int d = lane; d < D; d += T) {
        const int64_t o = q * D + d;
        const double gm0 = g0.dmu[o] + (g0.mean_grad ? g0.mean_grad[o] : 0.0);
        const double gm1 = g1.dmu[o] + (g1.mean_grad ? g1.mean_grad[o] : 0.0);
        grad[o] = pm0 * gm0 + ps0 * g0.ds2[o] + pm1 * gm1 + ps1 * g1.ds2[o];
    }
}

// pareto.hpp:60-95: point i is kept unless some point j has dominate_flag(j, i) == 1 (j is greater than i in some objective
// and smaller in none).  One thread per point; the objectives stream through shared memory in tiles of 256
// points.  A non-finite value sets *err.
__global__ void __launch_bounds__(256)
pareto_kernel(int64_t n, int K, const double* __restrict__ objs, int* __restrict__ keep, int* __restrict__ err)
{
    __shared__ double tile[LB_PARETO_MAX_K][256];
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    double mine[LB_PARETO_MAX_K];
    bool finite = true;
#pragma unroll
    for (int d = 0; d < LB_PARETO_MAX_K; ++d) {
        mine[d] = (d < K && i < n) ? objs[i * K + d] : 0.0;
        finite = finite && isfinite(mine[d]);
    }
    if (i < n && !finite) atomicOr(err, 1);
    int dominated = i >= n; // no point to decide
    for (int64_t j0 = 0; j0 < n; j0 += 256) {
        const int nt = (int)min((int64_t)256, n - j0);
        __syncthreads();
        if (threadIdx.x < nt)
#pragma unroll
            for (int d = 0; d < LB_PARETO_MAX_K; ++d) tile[d][threadIdx.x] = (d < K) ? objs[(j0 + threadIdx.x) * K + d] : 0.0;
        if (__syncthreads_and(dominated)) break; // (a barrier too) every point of the block is decided
        for (int jj = 0; jj < nt && !dominated; ++jj) {
            bool gt = false, lt = false; // gt: j is greater somewhere (flag1), lt: i is greater somewhere (flag2)
#pragma unroll
            for (int d = 0; d < LB_PARETO_MAX_K; ++d) {
                const double a = tile[d][jj], b = mine[d];
                gt = gt || a > b;
                lt = lt || (!(a > b) && b > a);
            }
            dominated = gt && !lt;
        }
    }
    if (i < n) keep[i] = !dominated;
}

LbOncePerDevice g_ehvi_attr_once;

// ---- three objectives: ehvi3d_sliceupdate (src/ehvi/ehvi_sliceupdate.cc:13-185) -------------------------------------------
// The front pass rebuilds Pstruct (n = k points; cell (x, y) of a plane is x + y n) from the host's per-axis orders:
//   ehvi3d_dom_kernel    highestdominator (as a double), xlim[y + z n], ylim[x + z n]: each entry is the last point, in the
//                        reference's loop order, whose orders cover it (sliceupdate.cc:65-78)
//   ehvi3d_slice_kernel  slice of every z-plane: a plane depends only on highestdominator, so one CTA per plane walks its
//                        anti-diagonals (each cell reads its left, lower and lower-left neighbours: sliceupdate.cc:87-107)
//   ehvi3d_chunk_kernel  chunk[z] = chunk[z-1] + slice[z-1] * (z-slab z-1's length), a walk in z per cell (sliceupdate.cc:82-85)
// with the reference's operations, unfused, so every entry equals the reference's bit for bit.  The scoring pass derives each
// cell's Sminus, slice[3], v[3] and skip rule from those planes (sliceupdate.cc:111-156) once per CTA and shares them across 128
// candidates.

// the host's upload (lb_ehvi3d): 9 n doubles.  X, Y, Z: the front's coordinates sorted per axis (stably by input index); then per
// z-order point its x- and y-order, per x-order point its y- and z-order, per y-order point its x- and z-order.
struct Front3 {
    const double *X, *Y, *Z, *zx, *zy, *xy, *xz, *yx, *yz;
};
__host__ __device__ inline Front3 front3(const double* f, int n)
{
    return {f, f + n, f + 2 * n, f + 3 * n, f + 4 * n, f + 5 * n, f + 6 * n, f + 7 * n, f + 8 * n};
}

__global__ void __launch_bounds__(256)
ehvi3d_dom_kernel(int n, const double* __restrict__ dF, double r0, double r1, double* __restrict__ hd, double* __restrict__ xlim,
    double* __restrict__ ylim)
{
    const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (c >= (int64_t)n * n) return;
    const Front3 F = front3(dF, n);
    const int a = (int)(c % n), b = (int)(c / n);
    int h = -1, ix = -1, iy = -1;
    for (int i = n - 1; i >= 0 && h < 0; --i)
        if (F.zx[i] >= a && F.zy[i] >= b) h = i;
    for (int i = n - 1; i >= 0 && ix < 0; --i)
        if (F.xy[i] >= a && F.xz[i] >= b) ix = i;
    for (int i = n - 1; i >= 0 && iy < 0; --i)
        if (F.yx[i] >= a && F.yz[i] >= b) iy = i;
    hd[c] = h;
    xlim[c] = ix < 0 ? 0.0 : F.X[ix] - r0;
    ylim[c] = iy < 0 ? 0.0 : F.Y[iy] - r1;
}

__global__ void __launch_bounds__(256)
ehvi3d_slice_kernel(int n, const double* __restrict__ dF, double r0, double r1, const double* __restrict__ hd, double* slice)
{
    const int z = blockIdx.x;
    const Front3 F = front3(dF, n);
    double* S = slice + (size_t)z * n * n;
    for (int d = 0; d <= 2 * (n - 1); ++d) {
        const int x0 = max(0, d - (n - 1)), x1 = min(d, n - 1);
        for (int x = x0 + (int)threadIdx.x; x <= x1; x += 256) {
            const int y = d - x;
            double v;
            if (hd[x + y * n] < z) {
                if (x > 0 && y > 0) v = (S[x + (y - 1) * n] - S[(x - 1) + (y - 1) * n]) + S[(x - 1) + y * n];
                else if (y > 0) v = S[x + (y - 1) * n];
                else if (x > 0) v = S[(x - 1) + y * n];
                else v = 0.0;
            } else {
                v = __dmul_rn(F.X[x] - r0, F.Y[y] - r1);
            }
            S[x + y * n] = v;
        }
        __syncthreads(); // the next diagonal reads this one
    }
}

__global__ void __launch_bounds__(256)
ehvi3d_chunk_kernel(int n, const double* __restrict__ dF, double r2, const double* __restrict__ slice, double* __restrict__ chunk)
{
    const int64_t c = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t nn = (int64_t)n * n;
    if (c >= nn) return;
    const Front3 F = front3(dF, n);
    double acc = 0.0;
    chunk[c] = acc;
    for (int z = 1; z <= n; ++z) {
        const double len = F.Z[z - 1] - (z == 1 ? r2 : F.Z[z - 2]); // cellength[2] of slab z - 1
        acc = __dadd_rn(acc, __dmul_rn(slice[(z - 1) * nn + c], len));
        chunk[z * nn + c] = acc;
    }
}

constexpr int E3_TX = 32;  // cells along x per CTA (blockIdx.y picks the x-block)
constexpr int E3_TY = 8;   // rows of y per staged tile, held in registers per candidate
constexpr int E3_Q = 128;  // candidates per CTA, one per thread
constexpr size_t E3_SMEM = sizeof(double) * (E3_TX * 3 * E3_Q + E3_TX * E3_TY * 8); // 112 KiB: two CTAs per SM

// the cell's front-only coefficients (Sminus, slice[0..2], v[0..2]; Sminus = NaN for a skipped cell, which then adds nothing, as
// the reference's `continue` and its `sum > 0` test do), in the reference's operations
__device__ __forceinline__ void ehvi3d_cell_coef(int n, int x, int y, int z, const Front3& F, double r0, double r1, double r2,
    const double* __restrict__ hd, const double* __restrict__ xlim, const double* __restrict__ ylim, const double* __restrict__ chunk,
    const double* __restrict__ slice, double* __restrict__ out)
{
    if (x > n || y > n) {
        out[0] = CUDART_NAN;
        return;
    }
    const size_t nn = (size_t)n * n;
    const double* C = chunk + z * nn;
    const double* S = slice + z * nn;
    const double len0 = (x == n ? CUDART_INF : F.X[x]) - (x == 0 ? r0 : F.X[x - 1]);
    const double len1 = (y == n ? CUDART_INF : F.Y[y]) - (y == 0 ? r1 : F.Y[y - 1]);
    const double len2 = (z == n ? CUDART_INF : F.Z[z]) - (z == 0 ? r2 : F.Z[z - 1]);
    const int h = (x < n && y < n) ? (int)hd[x + y * n] : -1;
    double Sm, s0, s1, s2;
    if (x > 0 && y > 0) {
        Sm = C[(x - 1) + (y - 1) * n];
        s0 = x == n ? 0.0 : __ddiv_rn(C[x + (y - 1) * n] - Sm, len0);
        s1 = y == n ? 0.0 : __ddiv_rn(C[(x - 1) + y * n] - Sm, len1);
        s2 = S[(x - 1) + (y - 1) * n];
    } else {
        Sm = 0.0;
        s0 = (y == 0 || x == n) ? 0.0 : __ddiv_rn(C[x + (y - 1) * n] - Sm, len0);
        s1 = (x == 0 || y == n) ? 0.0 : __ddiv_rn(C[(x - 1) + y * n] - Sm, len1);
        s2 = 0.0;
    }
    const bool skip = len0 == 0 || len1 == 0 || len2 == 0 || (x < n && y < n && h >= z);
    out[0] = skip ? CUDART_NAN : Sm;
    out[1] = s0;
    out[2] = s1;
    out[3] = s2;
    out[4] = (y == n || z == n) ? 0.0 : xlim[y + z * n];
    out[5] = (x == n || z == n) ? 0.0 : ylim[x + z * n];
    out[6] = (x == n || y == n || h == -1) ? 0.0 : F.Z[h] - r2;
    out[7] = 0.0;
}

// exipsi(r, c, m, s) and gausscdf((c - m) / s) (helper.cc:17-26) at bound b of an axis with sorted coordinates A[0..n-1]: c = r at
// b = 0, A[b-1] up to b = n, +inf at b = n + 1 (where exipsi = r - m and gausscdf = 1)
__device__ __forceinline__ double2 ehvi3d_bound(int b, int n, const double* __restrict__ A, double r, double m, double s)
{
    if (b > n) return make_double2(r - m, 1.0);
    const double c = b == 0 ? r : A[b - 1];
    const double t = (c - m) / s;
    return make_double2(s * (SQRT_TWOPI_NEG * exp(-(t * t) / 2)) + (r - m) * (0.5 * (1 + erf(t / SQRT_TWO))),
        0.5 * (1 + erf(t / SQRT_TWO)));
}

// the axis terms of cell index i from the bounds i (lo) and i + 1 (hi): psi, gausscdf and ex = psi - gausscdf (cl - r)
struct Axis3 { double psi, G, ex; };
__device__ __forceinline__ Axis3 ehvi3d_axis(double2 lo, double2 hi, double cl_minus_r)
{
    const double psi = lo.x - hi.x, G = hi.y - lo.y;
    return {psi, G, psi - G * cl_minus_r};
}

// The scoring pass.  CTA (blockIdx.x, blockIdx.y) scores candidates 128 blockIdx.x + threadIdx.x over the cells with x in
// [32 blockIdx.y, 32 blockIdx.y + 32) and every y and z, in a fixed order, into part[blockIdx.y M + q].  Per candidate the x-axis
// terms of its 32 cells sit in shared memory; per (z, 8 rows of y) the y/z products sit in registers and the 32 x 8 cells'
// coefficients are staged in shared memory.  With A = psi2 psi3, B = G2 G3, C = G3 ex2, D = G2 ex3, E = ex2 ex3 a cell is
//   sum = psi1 A - G1 (Sminus B + slice1 C + slice2 D + v0 E) - ex1 (slice0 B + v1 D + v2 C)
// (sliceupdate.cc:171-178 regrouped) and adds only where sum > 0.
__global__ void __launch_bounds__(E3_Q)
ehvi3d_cells_kernel(int n, const double* __restrict__ dF, double r0, double r1, double r2, const double* __restrict__ hd,
    const double* __restrict__ xlim, const double* __restrict__ ylim, const double* __restrict__ chunk, const double* __restrict__ slice,
    int64_t M, LbEhvi3Model m0, LbEhvi3Model m1, LbEhvi3Model m2, double* __restrict__ part)
{
    extern __shared__ __align__(16) double e3_smem[];
    double(*xt)[3][E3_Q] = reinterpret_cast<double(*)[3][E3_Q]>(e3_smem);                   // [E3_TX][3][E3_Q]
    double(*coef)[8] = reinterpret_cast<double(*)[8]>(e3_smem + E3_TX * 3 * E3_Q);          // [E3_TX * E3_TY][8]
    const Front3 F = front3(dF, n);
    const int64_t q = (int64_t)blockIdx.x * E3_Q + threadIdx.x;
    const int xb = blockIdx.y * E3_TX;
    const bool live = q < M;
    const int64_t qq = live ? q : 0;
    // acqui/ehvi.hpp:75-76 with a third model: FirstElem of each mu, and sigma() (sigma^2 + noise) where a deviation is expected
    const double mu0 = m0.mu[qq * m0.p] + (m0.mean ? m0.mean[qq] : m0.mean_const), s0 = m0.s2[qq];
    const double mu1 = m1.mu[qq * m1.p] + (m1.mean ? m1.mean[qq] : m1.mean_const), s1 = m1.s2[qq];
    const double mu2 = m2.mu[qq * m2.p] + (m2.mean ? m2.mean[qq] : m2.mean_const), s2 = m2.s2[qq];
    {
        double2 lo = ehvi3d_bound(xb, n, F.X, r0, mu0, s0);
        for (int i = 0; i < E3_TX; ++i) {
            const int x = xb + i;
            Axis3 a = {0.0, 0.0, 0.0};
            if (x <= n) {
                const double2 hi = ehvi3d_bound(x + 1, n, F.X, r0, mu0, s0);
                a = ehvi3d_axis(lo, hi, x == 0 ? r0 - r0 : F.X[x - 1] - r0);
                lo = hi;
            }
            xt[i][0][threadIdx.x] = a.psi;
            xt[i][1][threadIdx.x] = a.G;
            xt[i][2][threadIdx.x] = a.ex;
        }
    }
    double acc = 0.0;
    double2 zlo = ehvi3d_bound(0, n, F.Z, r2, mu2, s2);
    for (int z = 0; z <= n; ++z) {
        const double2 zhi = ehvi3d_bound(z + 1, n, F.Z, r2, mu2, s2);
        const Axis3 az = ehvi3d_axis(zlo, zhi, z == 0 ? r2 - r2 : F.Z[z - 1] - r2);
        zlo = zhi;
        for (int yb = 0; yb <= n; yb += E3_TY) {
            double A[E3_TY], B[E3_TY], Cc[E3_TY], Dd[E3_TY], Ee[E3_TY];
            double2 ylo = ehvi3d_bound(yb, n, F.Y, r1, mu1, s1);
#pragma unroll
            for (int j = 0; j < E3_TY; ++j) {
                const int y = yb + j;
                Axis3 ay = {0.0, 0.0, 0.0};
                if (y <= n) {
                    const double2 yhi = ehvi3d_bound(y + 1, n, F.Y, r1, mu1, s1);
                    ay = ehvi3d_axis(ylo, yhi, y == 0 ? r1 - r1 : F.Y[y - 1] - r1);
                    ylo = yhi;
                }
                A[j] = ay.psi * az.psi;
                B[j] = ay.G * az.G;
                Cc[j] = az.G * ay.ex;
                Dd[j] = ay.G * az.ex;
                Ee[j] = ay.ex * az.ex;
            }
            __syncthreads(); // the previous tile's readers are done
            for (int c = threadIdx.x; c < E3_TX * E3_TY; c += E3_Q)
                ehvi3d_cell_coef(n, xb + c % E3_TX, yb + c / E3_TX, z, F, r0, r1, r2, hd, xlim, ylim, chunk, slice, coef[c]);
            __syncthreads();
            const int xe = min(E3_TX, n + 1 - xb);
            for (int i = 0; i < xe; ++i) {
                const double psi1 = xt[i][0][threadIdx.x], G1 = xt[i][1][threadIdx.x], ex1 = xt[i][2][threadIdx.x];
#pragma unroll
                for (int j = 0; j < E3_TY; ++j) {
                    const double2* cf = reinterpret_cast<const double2*>(coef[j * E3_TX + i]);
                    const double2 c01 = cf[0], c23 = cf[1], c45 = cf[2], c67 = cf[3];
                    const double g = c01.x * B[j] + c23.x * Cc[j] + c23.y * Dd[j] + c45.x * Ee[j];
                    const double e = c01.y * B[j] + c45.y * Dd[j] + c67.x * Cc[j];
                    const double sum = psi1 * A[j] - G1 * g - ex1 * e;
                    if (sum > 0) acc += sum; // a skipped (NaN) or non-positive cell adds nothing
                }
            }
        }
    }
    if (live) part[(int64_t)blockIdx.y * M + q] = acc;
}

// acq[q] = the x-blocks' partial sums in ascending order: repeat calls are bit-identical
__global__ void __launch_bounds__(256)
ehvi3d_sum_kernel(int64_t M, int nxb, const double* __restrict__ part, double* __restrict__ acq)
{
    const int64_t q = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (q >= M) return;
    double s = 0.0;
    for (int b = 0; b < nxb; ++b) s += part[(int64_t)b * M + q];
    acq[q] = s;
}

} // namespace

// Team size for a front of k points: the largest power of two <= (k/2 + 1) / 4, in [1, 256], so that every thread of a team
// holds about four row pairs and the tables of the 256 / T candidates of a CTA fit in shared memory.
static int ehvi_team(int64_t k)
{
    const int64_t pairs = k / 2 + 1;
    int T = 1;
    while (T < 256 && 2 * T <= pairs / 4) T *= 2;
    return T;
}

size_t lb_ehvi_smem_bytes(int64_t k)
{
    return (size_t)(256 / ehvi_team(k)) * 2 * (size_t)(k + 2) * sizeof(double2);
}

// the largest table over every supported front (about 128 KiB: the team size grows with k)
static size_t ehvi_smem_max()
{
    size_t m = 0;
    for (int64_t k = 0; k <= LB_EHVI_MAX_K; ++k) m = std::max(m, lb_ehvi_smem_bytes(k));
    return m;
}

int lb_launch_ehvi(cudaStream_t st, double r0, double r1, int64_t k, const double* dFront, int64_t M, const double* dMu0, int p0,
    const double* dMean0, double mean0_const, const double* dS2_0, const double* dMu1, int p1, const double* dMean1, double mean1_const,
    const double* dS2_1, double* dAcq, long long* launches)
{
    if (k < 0 || k > LB_EHVI_MAX_K) return LB_ERR_UNSUPPORTED;
    if (g_ehvi_attr_once.need())
        LB_CUDA(cudaFuncSetAttribute(ehvi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ehvi_smem_max()));
    const int T = ehvi_team(k);
    const int64_t per = 256 / T;
    const unsigned grid = (unsigned)((M + per - 1) / per);
    ehvi_kernel<<<grid, 256, lb_ehvi_smem_bytes(k), st>>>(T, k, (const double2*)dFront, r0, r1, M, dMu0, p0, dMean0, mean0_const, dS2_0,
        dMu1, p1, dMean1, mean1_const, dS2_1, dAcq);
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// ehvi_grad_kernel's dynamic shared memory: ehvi_kernel's tables and one t per entry (at most 192 KiB, at k = LB_EHVI_MAX_K; with
// the 10 KiB of reductions 202 KiB of the 227 KiB a CTA may have)
static size_t ehvi_grad_smem_bytes(int64_t k)
{
    return lb_ehvi_smem_bytes(k) / sizeof(double2) * (sizeof(double2) + sizeof(double));
}

int lb_launch_ehvi_grad(cudaStream_t st, double r0, double r1, int64_t k, const double* dFront, int64_t M, int D, const LbPairModel& g0,
    const LbPairModel& g1, double* dAcq, double* dGrad, long long* launches)
{
    static LbOncePerDevice once;
    if (k < 0 || k > LB_EHVI_MAX_K) return LB_ERR_UNSUPPORTED;
    if (once.need())
        LB_CUDA(cudaFuncSetAttribute(ehvi_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
            (int)(ehvi_smem_max() / sizeof(double2) * (sizeof(double2) + sizeof(double)))));
    const int T = ehvi_team(k);
    const int64_t per = 256 / T;
    const unsigned grid = (unsigned)((M + per - 1) / per);
    ehvi_grad_kernel<<<grid, 256, ehvi_grad_smem_bytes(k), st>>>(T, k, (const double2*)dFront, r0, r1, M, D, g0, g1, dAcq, dGrad);
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Workspace: highestdominator, xlim, ylim (n^2 each), then slice and chunk for the n + 1 planes (n^2 (n + 1) each), then the
// x-blocks' partial sums (M each).  At n = LB_EHVI3D_MAX_K that is 271 MB of planes plus 72 bytes per candidate.
static int ehvi3d_xblocks(int64_t k) { return (int)((k + 1 + E3_TX - 1) / E3_TX); }
size_t lb_ehvi3d_ws_doubles(int64_t k, int64_t M)
{
    const size_t nn = (size_t)(k * k);
    return 3 * nn + 2 * nn * (size_t)(k + 1) + (size_t)ehvi3d_xblocks(k) * (size_t)M;
}

// the workspace's planes, in lb_ehvi3d_ws_doubles's order
struct E3Planes { double *hd, *xlim, *ylim, *slice, *chunk, *part; };
static E3Planes ehvi3d_planes(int64_t k, double* dWs)
{
    const size_t nn = (size_t)(k * k);
    E3Planes p;
    p.hd = dWs;
    p.xlim = p.hd + nn;
    p.ylim = p.xlim + nn;
    p.slice = p.ylim + nn;
    p.chunk = p.slice + nn * (size_t)(k + 1);
    p.part = p.chunk + nn * (size_t)(k + 1);
    return p;
}

int lb_launch_ehvi3d_front(cudaStream_t st, const double* r, int64_t k, const double* dFront, double* dWs, long long* launches)
{
    if (k < 0 || k > LB_EHVI3D_MAX_K) return LB_ERR_UNSUPPORTED;
    if (k == 0) return LB_OK;
    const int n = (int)k;
    const E3Planes p = ehvi3d_planes(k, dWs);
    const unsigned g = (unsigned)(((size_t)n * n + 255) / 256);
    ehvi3d_dom_kernel<<<g, 256, 0, st>>>(n, dFront, r[0], r[1], p.hd, p.xlim, p.ylim);
    ehvi3d_slice_kernel<<<n + 1, 256, 0, st>>>(n, dFront, r[0], r[1], p.hd, p.slice);
    ehvi3d_chunk_kernel<<<g, 256, 0, st>>>(n, dFront, r[2], p.slice, p.chunk);
    if (launches) *launches += 3;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_ehvi3d_cells(cudaStream_t st, const double* r, int64_t k, const double* dFront, int64_t M, const LbEhvi3Model& m0,
    const LbEhvi3Model& m1, const LbEhvi3Model& m2, double* dWs, double* dAcq, long long* launches)
{
    if (k < 0 || k > LB_EHVI3D_MAX_K) return LB_ERR_UNSUPPORTED;
    const E3Planes p = ehvi3d_planes(k, dWs);
    static LbOncePerDevice once;
    if (once.need()) LB_CUDA(cudaFuncSetAttribute(ehvi3d_cells_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)E3_SMEM));
    const int nxb = ehvi3d_xblocks(k);
    ehvi3d_cells_kernel<<<dim3((unsigned)((M + E3_Q - 1) / E3_Q), (unsigned)nxb), E3_Q, E3_SMEM, st>>>((int)k, dFront, r[0], r[1], r[2],
        p.hd, p.xlim, p.ylim, p.chunk, p.slice, M, m0, m1, m2, p.part);
    ehvi3d_sum_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(M, nxb, p.part, dAcq);
    if (launches) *launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_pareto(cudaStream_t st, int64_t n, int K, const double* dObjs, int* dKeep, int* dErr, long long* launches)
{
    if (K < 1 || K > LB_PARETO_MAX_K) return LB_ERR_UNSUPPORTED;
    pareto_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(n, K, dObjs, dKeep, dErr);
    if (launches) ++*launches;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
