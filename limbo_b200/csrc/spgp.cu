// limbo_b200/csrc/spgp.cu — Snelson and Ghahramani's pseudo-input sparse GP (FITC) with M learned pseudo-inputs:
// experimental::model::SPGP (src/limbo/experimental/model/spgp.hpp).
//
//   _likelihood / _likelihood_wp  spgp.hpp:446-580  -> lb_spgp_lik
//   _compute(false)               spgp.hpp:389-407  -> lb_spgp_compute
//   _predict                      spgp.hpp:582-610  -> lb_spgp_query / lb_spgp_acq_argmax (and their _dev variants)
//   a device CMA-ES over UCB / EI (not in the reference) -> lb_spgp_acq_cmaes
//   its candidate gradient        (not in the reference) -> lb_spgp_query_grad / lb_spgp_acq_grad
//
// Every M x M factor and inverse reuses the GP path: Q = K(xb, xb) + del I and A = sig I + V~ V~^T are factorised by
// lb_launch_potrf on two internal lb_gp handles (their dL), L^-1 and Lm^-1 come from the recursive trtri of lml.cu and
// Q^-1 from its lauum.  Every M x N x M product (V = L^-1 K, the SYRK of A, Lm^-1 V~, the two L^-T / Lm^-T solves, TT) is one
// launch of spgp_gemm_kernel over gemm.cuh's two-CTA DMMA tile; a triangular left operand only streams its nonzero k range.
// The reference's LU solves with Lt^T = (L Lm)^T and its inverses of L and Lt are the same triangular products:
//   B1 = Lt^-T Lm^-1 V~ = L^-T (Lm^-T (Lm^-1 V~)),  b1 = L^-T (Lm^-T bet),  invA = Lt^-T Lt^-1 = Z^T Z with Z = Lm^-1 L^-1.
// The D-fold loop of :523-553 is regrouped (DESIGN.md §8): with r = y~ - mu and the sqrt(b)-scaled coordinates x~, x~b,
//   G = K~ o (B1 - b1 r^T / sig - (2/sig) invLV o bigsum^T)                (M x N)
//   H = Q  o (invQ - sig invA - (2/sig) TT - b1 b1^T)                       (M x M)
//   dfxb(:,i) = (G x~)(:,i) - x~b(:,i) o rowsum(G) + x~b(:,i) o rowsum(H) - (H x~b)(:,i)
//   dfb(i)    = sum_n x~_ni (G^T x~b)_ni - x~_ni^2 colsum(G)_n
// before the sqrt(b) rescalings of :546-552, so the gradient is one pass over three M x N matrices (spgp_pass_kernel).
// The candidate gradient (DESIGN.md §4.14): with k_m = K*(m, q), lst = L^-1 k, lmst = Lm^-1 lst, k(x, x) = c constant,
//   grad mu = -sqrt(b) o sum_m b1_m k_m (x~ - x~b_m),  grad sigma^2 = 2 sqrt(b) o sum_m u_m k_m (x~ - x~b_m),
//   b1 = L^-T Lm^-T bet (once per lb_spgp_compute),  u = L^-T (lst - sig Lm^-T lmst) (two more triangular products per chunk).
// Layout: M is padded to Mp = roundup(M, 128) and N to Np = roundup(N, 128); padded rows and columns of K are zero, so they
// contribute nothing, and the padded parts of Q and A factor as the identity resp. sig I.
#include "../../include/limbo_b200.h"
#include "gemm.cuh"
#include <algorithm>
#include <cmath>
#include <mutex>
#include <new>

namespace {

using GC = lbg::CfgDual;
constexpr int PASS_DC = 8;    // input dimensions per sweep of spgp_pass_kernel
constexpr int QCHUNK = 8192;  // candidates per prediction chunk
constexpr int GRAD_THREADS = 128; // spgp_query_grad_kernel: one CTA per candidate
constexpr int GRAD_DC = 8;        // input dimensions per sweep of spgp_query_grad_kernel

// scalar slots of the per-evaluation reductions
enum { S_LOGDIAG = 0, S_YY, S_BB, S_LOGEP, S_MUR, S_EPCBIG, S_BIGEP, S_TRQ, S_TRA, S_AQ, S_BQB, S_BB1, S_COUNT };

// C (rows x cols tiles of 128 x 64) = op(A) op(B) (+ diag on the diagonal when not split).  A_KC: A(m, k) = A[k + m lda]
// (a transposed column-major operand), else A[m + k lda]; B_KC: B(k, n) = B[k + n ldb] (column-major), else B[n + k ldb].
// tri = 1: A is lower triangular (k < m0 + 128 only), tri = 2: upper (k >= m0).  blockIdx.y is the split-K slice; with
// gridDim.y > 1 slice s writes C + s * slice and spgp_split_reduce_kernel sums the slices in order.
template <bool A_KC, bool B_KC>
__global__ void __launch_bounds__(GC::THREADS, GC::CTAS_PER_SM)
spgp_gemm_kernel(const double* __restrict__ A, int64_t lda, const double* __restrict__ B, int64_t ldb, double* __restrict__ C,
    int64_t ldc, int64_t slice, int mtiles, int K, int tri, int kchunk, double diag)
{
    extern __shared__ __align__(16) double smem[];
    const int mt = blockIdx.x % mtiles, nt = blockIdx.x / mtiles;
    const int64_t m0 = (int64_t)mt * lbg::BM, n0 = (int64_t)nt * GC::BN;
    int kb = 0, ke = K;
    if (tri == 1) ke = min(K, (int)m0 + lbg::BM);
    if (tri == 2) kb = (int)m0;
    const int s = blockIdx.y;
    const int k0 = kb + s * kchunk, k1 = min(ke, k0 + kchunk);
    lbg::Acc<GC> acc;
    acc.zero();
    if (k1 > k0) {
        const double* gA = A_KC ? A + k0 + m0 * lda : A + m0 + (int64_t)k0 * lda;
        const double* gB = B_KC ? B + k0 + n0 * ldb : B + n0 + (int64_t)k0 * ldb;
        lbg::mainloop<GC, A_KC, B_KC>(acc, gA, lda, gB, ldb, k1 - k0, smem);
    }
    double* Cg = C + (int64_t)s * slice + m0 + n0 * ldc;
    const bool add_diag = gridDim.y == 1;
    lbg::for_each_acc<GC>(acc, [&](int r, int c, double& v) {
        Cg[r + (int64_t)c * ldc] = (add_diag && m0 + r == n0 + c) ? v + diag : v;
    });
}

__global__ void spgp_split_reduce_kernel(const double* __restrict__ W, int splits, int64_t n, int64_t ld, double* __restrict__ C,
    double diag)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n * n) return;
    double s = 0.0;
    for (int k = 0; k < splits; ++k) s += W[(int64_t)k * n * n + i];
    const int64_t r = i % n, c = i / n;
    C[r + c * ld] = (r == c) ? s + diag : s;
}

// x~ = x sqrt(b) for the points (row-major n x D in, dimension-major D x np out, zero padded)
__global__ void spgp_stage_kernel(const double* __restrict__ X, int64_t n, int D, const double* __restrict__ sb, double* __restrict__ out,
    int64_t np)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int d = blockIdx.y;
    if (i >= np) return;
    out[(int64_t)d * np + i] = (i < n) ? X[i * D + d] * sb[d] : 0.0;
}

// x~b = xb sqrt(b), xb read column-major from w (HyperParams, spgp.hpp:99-100)
__global__ void spgp_stage_xb_kernel(const double* __restrict__ w, int M, const double* __restrict__ sb, double* __restrict__ out, int64_t mp)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int d = blockIdx.y;
    if (i >= mp) return;
    out[(int64_t)d * mp + i] = (i < M) ? w[(int64_t)d * M + i] * sb[d] : 0.0;
}

// out(m, n) = c exp(-0.5 ((-2 xr_m . xc_n + |xc_n|^2) + |xr_m|^2))  (spgp.hpp:472-473, 624-625) for m < rows, n < cols, else 0;
// square = the M x M matrix Q: + del on the diagonal, and a second output with the identity in the padding (the factor's input)
__global__ void spgp_kmat_kernel(const double* __restrict__ xr, int64_t ldr, int64_t rows, const double* __restrict__ xc, int64_t ldc_x,
    int64_t cols, int D, double c, double* __restrict__ out, int64_t ld, int64_t ncols_p, int square, double del, double* __restrict__ out_pad)
{
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= ld * ncols_p) return;
    const int64_t m = idx % ld, n = idx / ld;
    double v = 0.0;
    if (m < rows && n < cols) {
        double dot = 0.0, nr = 0.0, nc = 0.0;
        for (int d = 0; d < D; ++d) {
            const double a = xr[(int64_t)d * ldr + m], b = xc[(int64_t)d * ldc_x + n];
            dot = fma(a, b, dot);
            nr = fma(a, a, nr);
            nc = fma(b, b, nc);
        }
        v = exp((-2.0 * dot + nc + nr) * -0.5) * c;
        if (square && m == n) v += del;
    }
    out[idx] = v;
    if (square) out_pad[idx] = (m < rows && n < cols) ? v : (m == n ? 1.0 : 0.0);
}

// ep = 1 + (c - |V(:,n)|^2) / sig from the unscaled V; K~ = K / sqrt(ep), V~ = V / sqrt(ep), y~ = y / sqrt(ep);
// sumVsq from the scaled V (spgp.hpp:480-483, 513).  One warp per column.
__global__ void __launch_bounds__(256) spgp_ep_kernel(double* __restrict__ K, double* __restrict__ V, int64_t ld, int64_t N, int64_t Np,
    const double* __restrict__ y, double c, double sig, double* __restrict__ ep, double* __restrict__ yt, double* __restrict__ sumvsq)
{
    const int64_t n = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= Np) return;
    if (n >= N) {
        if (lane == 0) { ep[n] = 1.0; yt[n] = 0.0; sumvsq[n] = 0.0; }
        return;
    }
    double* Vc = V + n * ld;
    double* Kc = K + n * ld;
    double s = 0.0;
    for (int64_t m = lane; m < ld; m += 32) s = fma(Vc[m], Vc[m], s);
    s = lb_warp_sum(s);
    const double e = 1.0 + (c - s) / sig;
    const double se = sqrt(e);
    double s2 = 0.0;
    for (int64_t m = lane; m < ld; m += 32) {
        const double v = Vc[m] / se;
        Vc[m] = v;
        Kc[m] = Kc[m] / se;
        s2 = fma(v, v, s2);
    }
    s2 = lb_warp_sum(s2);
    if (lane == 0) { ep[n] = e; yt[n] = y[n] / se; sumvsq[n] = s2; }
}

// per column n < cols: dot[n] = sum_m A(m, n) a[m] (when a), sq[n] = sum_m A(m, n)^2.  One warp per column.
__global__ void __launch_bounds__(256) spgp_coldot_kernel(const double* __restrict__ A, int64_t ld, int64_t cols, const double* __restrict__ a,
    double* __restrict__ dot, double* __restrict__ sq)
{
    const int64_t n = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= cols) return;
    const double* Ac = A + n * ld;
    double s = 0.0, q = 0.0;
    for (int64_t m = lane; m < ld; m += 32) {
        const double v = Ac[m];
        if (a) s = fma(v, a[m], s);
        q = fma(v, v, q);
    }
    s = lb_warp_sum(s);
    q = lb_warp_sum(q);
    if (lane == 0) {
        if (dot) dot[n] = s;
        if (sq) sq[n] = q;
    }
}

// part[s * ld + m] = sum_{n in strip s} A(m, n) v[n]
__global__ void __launch_bounds__(128) spgp_rowdot_kernel(const double* __restrict__ A, int64_t ld, int64_t cols, int64_t strip,
    const double* __restrict__ v, double* __restrict__ part)
{
    const int64_t m = blockIdx.x * (int64_t)128 + threadIdx.x;
    const int64_t n0 = blockIdx.y * strip, n1 = min(cols, n0 + strip);
    double s = 0.0;
    for (int64_t n = n0; n < n1; ++n) s = fma(A[m + n * ld], v[n], s);
    part[blockIdx.y * ld + m] = s;
}

__global__ void spgp_sum_parts_kernel(const double* __restrict__ part, int nparts, int64_t n, double* __restrict__ out)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int k = 0; k < nparts; ++k) s += part[(int64_t)k * n + i];
    out[i] = s;
}

__device__ __forceinline__ double block_sum_1024(double v, double* red)
{
    v = lb_warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 32) t = lb_warp_sum(red[threadIdx.x]);
    return t; // valid in thread 0
}

// value terms of spgp.hpp:491: sum log diag(Lm), y~^T y~, bet^T bet, sum log ep
__global__ void __launch_bounds__(1024) spgp_value_kernel(const double* __restrict__ Lm, int64_t ldm, int M, const double* __restrict__ bet,
    const double* __restrict__ yt, const double* __restrict__ ep, int64_t N, double* __restrict__ S)
{
    __shared__ double red[32];
    double a = 0.0, b = 0.0, c = 0.0, d = 0.0;
    for (int m = threadIdx.x; m < M; m += 1024) {
        a += log(Lm[m + m * ldm]);
        c = fma(bet[m], bet[m], c);
    }
    for (int64_t n = threadIdx.x; n < N; n += 1024) {
        b = fma(yt[n], yt[n], b);
        d += log(ep[n]);
    }
    a = block_sum_1024(a, red);
    if (threadIdx.x == 0) S[S_LOGDIAG] = a;
    b = block_sum_1024(b, red);
    if (threadIdx.x == 0) S[S_YY] = b;
    c = block_sum_1024(c, red);
    if (threadIdx.x == 0) S[S_BB] = c;
    d = block_sum_1024(d, red);
    if (threadIdx.x == 0) S[S_LOGEP] = d;
}

// per sample (spgp.hpp:512-516, 557): r = y~ - mu, bigsum, and the sums of mu^T r, epc^T bigsum and bigsum ./ ep
__global__ void __launch_bounds__(1024) spgp_nvec_kernel(const double* __restrict__ yt, const double* __restrict__ mu,
    const double* __restrict__ bv, const double* __restrict__ sq_lmv, const double* __restrict__ ep, const double* __restrict__ sumvsq,
    const double* __restrict__ sq_lv, int64_t N, int64_t Np, double c, double sig, double del, double* __restrict__ r_out,
    double* __restrict__ big_out, double* __restrict__ S)
{
    __shared__ double red[32];
    double a = 0.0, b = 0.0, e = 0.0;
    for (int64_t n = threadIdx.x; n < Np; n += 1024) {
        if (n >= N) { r_out[n] = 0.0; big_out[n] = 0.0; continue; }
        const double y = yt[n], m = mu[n];
        const double big = y * bv[n] / sig - sq_lmv[n] / 2 - (y * y + m * m) / (2 * sig) + 0.5;
        const double epc = (c / ep[n] - sumvsq[n] - del * sq_lv[n]) / sig;
        r_out[n] = y - m;
        big_out[n] = big;
        a = fma(m, y - m, a);
        b = fma(epc, big, b);
        e += big / ep[n];
    }
    a = block_sum_1024(a, red);
    if (threadIdx.x == 0) S[S_MUR] = a;
    b = block_sum_1024(b, red);
    if (threadIdx.x == 0) S[S_EPCBIG] = b;
    e = block_sum_1024(e, red);
    if (threadIdx.x == 0) S[S_BIGEP] = e;
}

__global__ void spgp_scale_cols_kernel(const double* __restrict__ A, int64_t ld, int64_t ncols, const double* __restrict__ v,
    double* __restrict__ out)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= ld * ncols) return;
    out[i] = A[i] * v[i / ld];
}

struct PassArgs {
    const double* E0; const double* E1; const double* E2; const double* E3; int64_t ld; // MODE 0: K~, B1, invLV; 1: Q, invQ, invA, TT
    const double* b1; const double* r; const double* big;
    const double* xc; int64_t ldxc; // column coordinates (D x ldxc)
    const double* xr; int64_t ldxr; // row coordinates (D x ldxr)
    int64_t cols, strip;
    int D;
    double sig;
    double* rowpart; // [strip][D + 1][ldxr]: sum_n e x~c_dn, and the row sum at d = D
    double* blkpart; // MODE 0: [block][D] sums of e x~c_dn (x~r_dm - x~c_dn); MODE 1: [block][5] the dfc terms
};

// One thread per row, a strip of columns per block, D in sweeps of PASS_DC (e is recomputed per sweep).
template <int MODE>
__global__ void __launch_bounds__(128) spgp_pass_kernel(PassArgs a)
{
    __shared__ double red[4][PASS_DC];
    const int64_t m = blockIdx.x * (int64_t)128 + threadIdx.x;
    const int64_t n0 = blockIdx.y * a.strip, n1 = min(a.cols, n0 + a.strip);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int blk = blockIdx.y * gridDim.x + blockIdx.x;
    const double b1m = a.b1[m];
    const double two_sig = 2.0 / a.sig;
    auto elem = [&](int64_t n) {
        const int64_t i = m + n * a.ld;
        if (MODE == 0) return a.E0[i] * (a.E1[i] - b1m * a.r[n] / a.sig - two_sig * a.E2[i] * a.big[n]);
        return a.E0[i] * (a.E1[i] - a.sig * a.E2[i] - two_sig * a.E3[i] - b1m * a.b1[n]);
    };
    for (int d0 = 0; d0 < a.D; d0 += PASS_DC) {
        double R[PASS_DC], P[PASS_DC], xr[PASS_DC];
#pragma unroll
        for (int j = 0; j < PASS_DC; ++j) {
            R[j] = 0.0;
            P[j] = 0.0;
            xr[j] = (d0 + j < a.D) ? a.xr[(int64_t)(d0 + j) * a.ldxr + m] : 0.0;
        }
        double rs = 0.0, t_aq = 0.0, t_bqb = 0.0;
        for (int64_t n = n0; n < n1; ++n) {
            const double e = elem(n);
            if (d0 == 0) {
                rs += e;
                if (MODE == 1) {
                    const int64_t i = m + n * a.ld;
                    t_aq = fma(a.E2[i], a.E0[i], t_aq);
                    t_bqb = fma(b1m * a.E0[i], a.b1[n], t_bqb);
                }
            }
#pragma unroll
            for (int j = 0; j < PASS_DC; ++j) {
                if (d0 + j < a.D) {
                    const double xc = a.xc[(int64_t)(d0 + j) * a.ldxc + n];
                    R[j] = fma(e, xc, R[j]);
                    if (MODE == 0) P[j] = fma(e * xc, xr[j] - xc, P[j]);
                }
            }
        }
        const int64_t base = (int64_t)blockIdx.y * (a.D + 1);
#pragma unroll
        for (int j = 0; j < PASS_DC; ++j)
            if (d0 + j < a.D) a.rowpart[(base + d0 + j) * a.ldxr + m] = R[j];
        if (d0 == 0) {
            a.rowpart[(base + a.D) * a.ldxr + m] = rs;
            if (MODE == 1) {
                // diagonal terms of the dfc expression: trace(invQ), trace(invA), b1^T b1 (the thread's own row, if in the strip)
                double tq = 0.0, ta = 0.0, bb = 0.0;
                if (m >= n0 && m < n1) {
                    const int64_t i = m + m * a.ld;
                    tq = a.E1[i];
                    ta = a.E2[i];
                    bb = b1m * b1m;
                }
                double v[5] = {tq, ta, t_aq, t_bqb, bb};
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    const double s = lb_warp_sum(v[j]);
                    if (lane == 0) red[warp][j] = s;
                }
                __syncthreads();
                if (threadIdx.x < 5) a.blkpart[(int64_t)blk * 5 + threadIdx.x] = red[0][threadIdx.x] + red[1][threadIdx.x] + red[2][threadIdx.x] + red[3][threadIdx.x];
                __syncthreads();
            }
        }
        if (MODE == 0) {
#pragma unroll
            for (int j = 0; j < PASS_DC; ++j) {
                const double s = lb_warp_sum(P[j]);
                if (lane == 0) red[warp][j] = s;
            }
            __syncthreads();
            if (threadIdx.x < PASS_DC && d0 + threadIdx.x < a.D)
                a.blkpart[(int64_t)blk * a.D + d0 + threadIdx.x] = red[0][threadIdx.x] + red[1][threadIdx.x] + red[2][threadIdx.x] + red[3][threadIdx.x];
            __syncthreads();
        }
    }
}

// dfxb (spgp.hpp:536-546) from the row sums of both passes; writes -dfxb into grad (column-major flattening, :568) and the
// per-block sums of dfxb(:,i) x~b(:,i) for dfb (:549-551).  grid (ceil(M / 128), D).
__global__ void __launch_bounds__(128) spgp_dfxb_kernel(const double* __restrict__ rowG, int sG, const double* __restrict__ rowH, int sH,
    int64_t Mp, int M, int D, const double* __restrict__ xbt, const double* __restrict__ sb, double* __restrict__ grad, double* __restrict__ part)
{
    __shared__ double red[4];
    const int m = blockIdx.x * 128 + threadIdx.x;
    const int i = blockIdx.y;
    double v = 0.0;
    if (m < M) {
        double gx = 0.0, gs = 0.0, hx = 0.0, hs = 0.0;
        for (int s = 0; s < sG; ++s) {
            gx += rowG[((int64_t)s * (D + 1) + i) * Mp + m];
            gs += rowG[((int64_t)s * (D + 1) + D) * Mp + m];
        }
        for (int s = 0; s < sH; ++s) {
            hx += rowH[((int64_t)s * (D + 1) + i) * Mp + m];
            hs += rowH[((int64_t)s * (D + 1) + D) * Mp + m];
        }
        const double x = xbt[(int64_t)i * Mp + m];
        const double d = ((gx - x * gs) + (x * hs - hx)) * sb[i];
        grad[(int64_t)i * M + m] = -d;
        v = d * x;
    }
    v = lb_warp_sum(v);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) part[(int64_t)i * gridDim.x + blockIdx.x] = red[0] + red[1] + red[2] + red[3];
}

// f = -fw and the tail of the gradient, -[dfb, dfc, dfsig] (spgp.hpp:491, 546-564, 573-576).  One block of 64 threads.
__global__ void spgp_final_kernel(const double* __restrict__ S, const double* __restrict__ blkG, int nblkG, const double* __restrict__ blkH,
    int nblkH, const double* __restrict__ xpart, int nxb, const double* __restrict__ sb, int M, int D, double half_nm, double n, double sig,
    double del, int with_grad, double* __restrict__ f, double* __restrict__ grad)
{
    const int i = threadIdx.x;
    if (i == 0) {
        const double fw = S[S_LOGDIAG] + half_nm * log(sig) + (S[S_YY] - S[S_BB]) / (2 * sig) + S[S_LOGEP] / 2 + 0.5 * n * log(2 * M_PI);
        *f = -fw;
    }
    if (!with_grad) return;
    if (i < D) {
        double p = 0.0;
        for (int k = 0; k < nblkG; ++k) p += blkG[(int64_t)k * D + i];
        double xs = 0.0;
        for (int k = 0; k < nxb; ++k) xs += xpart[(int64_t)i * nxb + k];
        const double s = sb[i], b = s * s;
        double dfb = p / s;
        dfb += xs / b;
        dfb *= s / 2;
        grad[(int64_t)M * D + i] = -dfb;
    }
    if (i == 0) {
        double t[5] = {0, 0, 0, 0, 0};
        for (int k = 0; k < nblkH; ++k)
            for (int j = 0; j < 5; ++j) t[j] += blkH[(int64_t)k * 5 + j];
        const double trq = t[0], tra = t[1], aq = t[2], bqb = t[3], bb = t[4];
        const double dfc = (M + del * (trq - sig * tra) - sig * aq) / 2 - S[S_MUR] / sig + (bqb - del * bb) / 2 + S[S_EPCBIG];
        grad[(int64_t)(M + 1) * D] = -dfc;
        grad[(int64_t)(M + 1) * D + 1] = -S[S_BIGEP];
    }
}

// sigma^2 = c - |L^-1 k*|^2 + sig |Lm^-1 L^-1 k*|^2 (+ sig once optimised), spgp.hpp:608
__global__ void spgp_pred_kernel(const double* __restrict__ sq1, const double* __restrict__ sq2, int64_t n, double c, double sig, double add,
    double* __restrict__ s2)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) s2[i] = c - sq1[i] + sig * sq2[i] + add;
}

// r = lst - sig t over n entries, in place over t
__global__ void spgp_resid_kernel(const double* __restrict__ lst, double* __restrict__ t, int64_t n, double sig)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) t[i] = lst[i] - sig * t[i];
}

// Candidate gradients of one chunk, one CTA per candidate q: k = K*(:, q) (ld rows, zero below M), u = U(:, q), x~ = xqt(:, q).
// Every thread takes the pseudo-inputs m = tid + 128 j in a fixed order; the sums are reduced over the lanes, then over the warps
// in a fixed order, so a candidate's result is run-to-run identical and does not depend on the rest of the batch.  The difference
// x~_d - x~b_md is formed per term (x~_d sum_m w_m - sum_m w_m x~b_md cancels for candidates far from the origin).  mu0 / s2: the
// forward outputs of the chunk; out: the gradient outputs (D columns), its pointers from the chunk's first candidate.
__global__ void __launch_bounds__(GRAD_THREADS)
spgp_query_grad_kernel(const double* __restrict__ ks, const double* __restrict__ U, int64_t ld, int M, const double* __restrict__ b1,
    const double* __restrict__ xbt, const double* __restrict__ xqt, int64_t ldq, const double* __restrict__ sb, int D,
    const double* __restrict__ mu0, const double* __restrict__ s2, const LbGradOut out)
{
    __shared__ double sx[LB_MAX_D];
    __shared__ double red[2][GRAD_THREADS / 32][GRAD_DC];
    __shared__ double gsum[2][LB_MAX_D];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t q = blockIdx.x;
    for (int d = tid; d < D; d += GRAD_THREADS) sx[d] = xqt[(int64_t)d * ldq + q];
    __syncthreads();
    const double* kc = ks + q * ld;
    const double* uc = U + q * ld;
    for (int d0 = 0; d0 < D; d0 += GRAD_DC) {
        double am[GRAD_DC], aw[GRAD_DC];
#pragma unroll
        for (int j = 0; j < GRAD_DC; ++j) am[j] = aw[j] = 0.0;
        for (int m = tid; m < M; m += GRAD_THREADS) {
            const double k = kc[m];
            const double cb = k * b1[m], cu = k * uc[m];
#pragma unroll
            for (int j = 0; j < GRAD_DC; ++j)
                if (d0 + j < D) {
                    const double t = sx[d0 + j] - xbt[(int64_t)(d0 + j) * ld + m];
                    am[j] = fma(cb, t, am[j]);
                    aw[j] = fma(cu, t, aw[j]);
                }
        }
#pragma unroll
        for (int j = 0; j < GRAD_DC; ++j) {
            const double a = lb_warp_sum(am[j]), b = lb_warp_sum(aw[j]);
            if (lane == 0) {
                red[0][warp][j] = a;
                red[1][warp][j] = b;
            }
        }
        __syncthreads();
        if (tid < 2 * GRAD_DC) {
            const int k = tid / GRAD_DC, j = tid % GRAD_DC;
            double s = 0.0;
            for (int w = 0; w < GRAD_THREADS / 32; ++w) s += red[k][w][j];
            if (d0 + j < D) gsum[k][d0 + j] = s;
        }
        __syncthreads();
    }
    if (tid >= D) return;
    const int d = tid;
    const double gmu = -sb[d] * gsum[0][d], gs2 = 2.0 * sb[d] * gsum[1][d];
    const int64_t o = q * D + d;
    if (out.dmu) out.dmu[o] = gmu;
    if (out.ds2) out.ds2[o] = gs2;
    if (out.acq_id < 0) return;
    const double s = s2[q];
    const double mu = mu0[q] + (out.mean ? out.mean[q] : out.mean_const); // acq_kernel's sum, so the values are lb_spgp_acq_argmax's
    const double gm = out.mean_grad ? gmu + out.mean_grad[o] : gmu;
    const double g = lb_acq_grad_value(out.acq_id, mu, s, gm, gs2, out.p0, out.p1);
    if (out.grad) out.grad[o] = g;
    if (d == 0 && out.acq) out.acq[q] = lb_acq_value(out.acq_id, mu, s, out.p0, out.p1);
}

LbOncePerDevice g_attr_once;
int set_attrs()
{
    if (!g_attr_once.need()) return LB_OK;
    LB_CUDA(cudaFuncSetAttribute(spgp_gemm_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GC::PIPE_BYTES));
    LB_CUDA(cudaFuncSetAttribute(spgp_gemm_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GC::PIPE_BYTES));
    LB_CUDA(cudaFuncSetAttribute(spgp_gemm_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GC::PIPE_BYTES));
    return LB_OK;
}

inline int64_t round_up(int64_t v, int64_t q) { return (v + q - 1) / q * q; }
inline unsigned nblocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

} // namespace

struct lb_spgp {
    int device = 0;
    int sms = 132;
    lb_gp* q = nullptr; // Q = K(xb, xb) + del I: dL -> L, dLinv = L^-1, dKinv = Q^-1
    lb_gp* a = nullptr; // A = sig I + V~ V~^T: dL -> Lm, dLinv = Lm^-1
    cudaStream_t st = nullptr;
    std::mutex mu;
    long long launches = 0;

    int64_t N = 0, Np = 0;
    int D = 0;
    DevBuf<double> dX; // N x D row-major
    DevBuf<double> dY; // Np, zero padded

    int M = 0;
    int64_t Mp = 0;
    DevBuf<double> dXt, dXbt, dSb;
    DevBuf<double> dW;                    // w
    DevBuf<double> dK, dV, dP1, dP2, dP3; // Mp x Np
    DevBuf<double> dQ, dZ, dInvA, dTT;    // Mp x Mp
    DevBuf<double> dNv;   // N-vectors, 12 x Np
    DevBuf<double> dMv;   // M-vectors, 8 x Mp
    DevBuf<double> dS;    // scalars
    DevBuf<double> dOut;  // f, grad
    DevBuf<double> dWork; // split-K slices, row / block partials
    // prediction state (lb_spgp_compute)
    bool computed = false;
    bool b1_ready = false; // Mv row 6 holds b1 = L^-T Lm^-T bet of the current factors (candidate gradients)
    double c = 0, sig = 0;
    // query workspace
    DevBuf<double> dQx, dQxt, dMu, dS2; // dQx: the host entry points' candidates
    DevBuf<double> dGrad; // candidate gradients: the mean's input gradient, grad mu, grad sigma^2, the acquisition's, Mq x D each
    ArgmaxWs am; // acquisition values, means, argmax records
};

namespace {

// the inner handles' factor storage (raw: lb_gp's copy-on-write buffers, never shared here) and its inverses
void free_inner(lb_gp* h)
{
    lb_pool_free(h->dL);
    lb_pool_free(h->dInvD);
    h->dL = h->dInvD = nullptr;
    h->dLinv.release();
    h->dKinv.release();
    lb_factor_changed(h);
    h->Np = 0;
}

// callers synchronise s->st before Mp changes (ensure_state: the Mp-sized buffers are reallocated first)
int ensure_inner(lb_spgp* s, lb_gp* h, int64_t Mp, int M)
{
    if (h->Np != Mp) {
        free_inner(h);
        const int64_t T = Mp / LB_TILE;
        LB_ALLOC(h, h->dL, sizeof(double) * Mp * Mp);
        LB_ALLOC(h, h->dInvD, sizeof(double) * T * LB_TILE * LB_TILE);
        LB_CUDA(cudaMemsetAsync(h->dInvD, 0, sizeof(double) * T * LB_TILE * LB_TILE, s->st));
        h->Np = Mp;
    }
    h->N = M;
    lb_factor_changed(h); // a new factor invalidates the inverses
    return LB_OK;
}

int ensure_state(lb_spgp* s, int M)
{
    const int64_t Mp = round_up(M, LB_TILE), Np = s->Np;
    s->M = M;
    s->Mp = Mp;
    const size_t mn = sizeof(double) * Mp * Np, mm = sizeof(double) * Mp * Mp;
    const std::pair<DevBuf<double>*, size_t> bufs[] = {{&s->dXt, sizeof(double) * s->D * Np}, {&s->dXbt, sizeof(double) * s->D * Mp},
        {&s->dSb, sizeof(double) * LB_MAX_D}, {&s->dK, mn}, {&s->dV, mn}, {&s->dP1, mn}, {&s->dP2, mn}, {&s->dP3, mn}, {&s->dQ, mm},
        {&s->dZ, mm}, {&s->dInvA, mm}, {&s->dTT, mm}, {&s->dNv, sizeof(double) * 12 * Np}, {&s->dMv, sizeof(double) * 8 * Mp}};
    int rc;
    for (const auto& b : bufs)
        if ((rc = b.first->resize(s->device, s->st, b.second))) return rc;
    if ((rc = ensure_inner(s, s->q, Mp, M))) return rc;
    if ((rc = ensure_inner(s, s->a, Mp, M))) return rc;
    return LB_OK;
}

// C = op(A) op(B) over K; rows x cols multiples of 128 x 64.  Split-K (non-triangular products only) when the output has too
// few tiles to fill the SMs: the small-M SYRK and TT over K = Np.
template <bool A_KC, bool B_KC>
int gemm(lb_spgp* s, const double* A, int64_t lda, const double* B, int64_t ldb, double* C, int64_t ldc, int64_t rows, int64_t cols,
    int64_t K, int tri, double diag)
{
    const int mtiles = (int)(rows / lbg::BM), tiles = mtiles * (int)(cols / GC::BN);
    int splits = 1;
    int64_t kchunk = K;
    if (tri == 0 && ldc == rows && rows == cols) {
        const int want = (2 * s->sms + tiles - 1) / tiles;
        const int kmax = (int)(K / 512);
        splits = std::max(1, std::min(std::min(want, kmax), 64));
        kchunk = round_up((K + splits - 1) / splits, LB_TILE);
        splits = (int)((K + kchunk - 1) / kchunk);
    }
    double* out = C;
    if (splits > 1) {
        int rc = s->dWork.reserve(s->device, s->st, sizeof(double) * splits * rows * cols);
        if (rc) return rc;
        out = s->dWork.get();
    }
    spgp_gemm_kernel<A_KC, B_KC><<<dim3(tiles, splits), GC::THREADS, GC::PIPE_BYTES, s->st>>>(A, lda, B, ldb, out, splits > 1 ? rows : ldc,
        rows * cols, mtiles, (int)K, tri, (int)kchunk, diag);
    s->launches++;
    if (splits > 1) {
        spgp_split_reduce_kernel<<<nblocks(rows * cols, 256), 256, 0, s->st>>>(s->dWork.get(), splits, rows, ldc, C, diag);
        s->launches++;
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// number of column strips for a one-thread-per-row pass over rows x cols
int64_t pick_strip(const lb_spgp* s, int64_t rows, int64_t cols, int* nstrips)
{
    const int64_t rb = rows / 128;
    int64_t want = (8 * s->sms + rb - 1) / rb;
    want = std::max<int64_t>(1, std::min<int64_t>(want, (cols + 31) / 32));
    const int64_t strip = (cols + want - 1) / want;
    *nstrips = (int)((cols + strip - 1) / strip);
    return strip;
}

int check_w(const lb_spgp* s, int64_t M, int64_t n_w, const double* w)
{
    if (!w || M < 1 || M > s->N || M > INT32_MAX) return LB_ERR_ARG;
    if (n_w != (M + 1) * s->D + 2) return LB_ERR_ARG;
    for (int64_t i = 0; i < n_w; ++i)
        if (!std::isfinite(w[i])) return LB_ERR_ARG;
    return LB_OK;
}

int read_info(lb_spgp* s)
{
    int iq[2] = {0, 0}, ia[2] = {0, 0};
    LB_CUDA(cudaMemcpyAsync(iq, s->q->dInfo.get(), sizeof(iq), cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaMemcpyAsync(ia, s->a->dInfo.get(), sizeof(ia), cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaStreamSynchronize(s->st));
    if (iq[1] || ia[1]) return LB_ERR_TIMEOUT;
    if (iq[0] > 0) return iq[0];
    if (ia[0] > 0) return ia[0];
    return LB_OK;
}

// The forward part shared by _likelihood_wp (:456-488) and _compute (:389-407): leaves K~ (dK), V~ (dV), L^-1, Lm^-1,
// Lm^-1 V~ (dP1), bet, y~, ep and sumVsq on the device.  Nv rows: 0 ep, 1 y~, 2 sumVsq; Mv rows: 0 bet.
int forward(lb_spgp* s, int M, const double* w, double jitter, double* c_out, double* sig_out)
{
    int rc;
    if ((rc = set_attrs())) return rc;
    if ((rc = ensure_state(s, M))) return rc;
    const int D = s->D;
    const int64_t Mp = s->Mp, Np = s->Np, N = s->N;
    double sb[LB_MAX_D];
    for (int d = 0; d < D; ++d) sb[d] = sqrt(exp(w[(int64_t)M * D + d]));
    const double c = exp(w[(int64_t)(M + 1) * D]), sig = exp(w[(int64_t)(M + 1) * D + 1]);
    *c_out = c;
    *sig_out = sig;
    if ((rc = s->dW.reserve(s->device, s->st, sizeof(double) * ((M + 1) * D + 2)))) return rc;
    LB_CUDA(cudaMemcpyAsync(s->dSb.get(), sb, sizeof(double) * D, cudaMemcpyHostToDevice, s->st));
    LB_CUDA(cudaMemcpyAsync(s->dW.get(), w, sizeof(double) * ((M + 1) * D + 2), cudaMemcpyHostToDevice, s->st));
    double* ep = s->dNv.get();
    double* yt = s->dNv.get() + Np;
    double* sumvsq = s->dNv.get() + 2 * Np;
    double* bet = s->dMv.get();
    spgp_stage_kernel<<<dim3(nblocks(Np, 256), D), 256, 0, s->st>>>(s->dX.get(), N, D, s->dSb.get(), s->dXt.get(), Np);
    spgp_stage_xb_kernel<<<dim3(nblocks(Mp, 256), D), 256, 0, s->st>>>(s->dW.get(), M, s->dSb.get(), s->dXbt.get(), Mp);
    spgp_kmat_kernel<<<nblocks(Mp * Mp, 256), 256, 0, s->st>>>(s->dXbt.get(), Mp, M, s->dXbt.get(), Mp, M, D, c, s->dQ.get(), Mp, Mp, 1, jitter, s->q->dL);
    spgp_kmat_kernel<<<nblocks(Mp * Np, 256), 256, 0, s->st>>>(s->dXbt.get(), Mp, M, s->dXt.get(), Np, N, D, c, s->dK.get(), Mp, Np, 0, 0.0, nullptr);
    s->launches += 4;
    LB_CUDA(cudaGetLastError());
    // L = chol(Q), L^-1
    if ((rc = lb_launch_potrf(s->q))) return rc;
    if ((rc = lb_launch_linv(s->q))) return rc;
    // V = L^-1 K; ep; K~, V~, y~
    if ((rc = gemm<false, true>(s, s->q->dLinv.get(), Mp, s->dK.get(), Mp, s->dV.get(), Mp, Mp, Np, Mp, 1, 0.0))) return rc;
    spgp_ep_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dK.get(), s->dV.get(), Mp, N, Np, s->dY.get(), c, sig, ep, yt, sumvsq);
    s->launches++;
    // Lm = chol(sig I + V~ V~^T), Lm^-1
    if ((rc = gemm<false, false>(s, s->dV.get(), Mp, s->dV.get(), Mp, s->a->dL, Mp, Mp, Mp, Np, 0, sig))) return rc;
    if ((rc = lb_launch_potrf(s->a))) return rc;
    if ((rc = lb_launch_linv(s->a))) return rc;
    // invLmV = Lm^-1 V~, bet = invLmV y~
    if ((rc = gemm<false, true>(s, s->a->dLinv.get(), Mp, s->dV.get(), Mp, s->dP1.get(), Mp, Mp, Np, Mp, 1, 0.0))) return rc;
    int ns;
    const int64_t strip = pick_strip(s, Mp, N, &ns);
    if ((rc = s->dWork.reserve(s->device, s->st, sizeof(double) * ns * Mp))) return rc;
    spgp_rowdot_kernel<<<dim3((unsigned)(Mp / 128), ns), 128, 0, s->st>>>(s->dP1.get(), Mp, N, strip, yt, s->dWork.get());
    spgp_sum_parts_kernel<<<nblocks(Mp, 256), 256, 0, s->st>>>(s->dWork.get(), ns, Mp, bet);
    s->launches += 3;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int likelihood(lb_spgp* s, int M, const double* w, double jitter, double* f, double* grad)
{
    double c, sig;
    int rc = forward(s, M, w, jitter, &c, &sig);
    if (rc) return rc;
    const int D = s->D;
    const int64_t Mp = s->Mp, Np = s->Np, N = s->N;
    const int nw = (M + 1) * D + 2;
    if ((rc = s->dOut.reserve(s->device, s->st, sizeof(double) * (nw + 1))) || (rc = s->dS.reserve(s->device, s->st, sizeof(double) * 64)))
        return rc;
    double* ep = s->dNv.get();
    double* yt = s->dNv.get() + Np;
    double* sumvsq = s->dNv.get() + 2 * Np;
    double* mu = s->dNv.get() + 3 * Np;
    double* bv = s->dNv.get() + 4 * Np;
    double* sq_lmv = s->dNv.get() + 5 * Np;
    double* sq_lv = s->dNv.get() + 6 * Np;
    double* r = s->dNv.get() + 7 * Np;
    double* big = s->dNv.get() + 8 * Np;
    double* bet = s->dMv.get();
    double* u = s->dMv.get() + Mp;
    double* b1 = s->dMv.get() + 2 * Mp;
    const double half_nm = (double)((N - M) / 2); // spgp.hpp:491: (n - _m) / 2 in integer arithmetic
    spgp_value_kernel<<<1, 1024, 0, s->st>>>(s->a->dL, Mp, M, bet, yt, ep, N, s->dS.get());
    s->launches++;
    if (!grad) {
        spgp_final_kernel<<<1, 64, 0, s->st>>>(s->dS.get(), nullptr, 0, nullptr, 0, nullptr, 0, s->dSb.get(), M, D, half_nm, (double)N, sig, jitter, 0,
            s->dOut.get(), s->dOut.get() + 1);
        s->launches++;
        LB_CUDA(cudaGetLastError());
        if ((rc = read_info(s))) return rc;
        LB_CUDA(cudaMemcpy(f, s->dOut.get(), sizeof(double), cudaMemcpyDeviceToHost));
        return LB_OK;
    }
    // bet^T invLmV and colsum(invLmV^2); u = Lm^-T bet; b1 = L^-T u; mu = u^T V~  (spgp.hpp:503, 512, 516)
    spgp_coldot_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dP1.get(), Mp, Np, bet, bv, sq_lmv);
    spgp_coldot_kernel<<<nblocks(Mp, 8), 256, 0, s->st>>>(s->a->dLinv.get(), Mp, Mp, bet, u, nullptr);
    spgp_coldot_kernel<<<nblocks(Mp, 8), 256, 0, s->st>>>(s->q->dLinv.get(), Mp, Mp, u, b1, nullptr);
    spgp_coldot_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dV.get(), Mp, Np, u, mu, nullptr);
    s->launches += 4;
    // B1 = L^-T (Lm^-T invLmV) (:502), invLV = L^-T V~ (:505)
    if ((rc = gemm<true, true>(s, s->a->dLinv.get(), Mp, s->dP1.get(), Mp, s->dP2.get(), Mp, Mp, Np, Mp, 2, 0.0))) return rc;
    if ((rc = gemm<true, true>(s, s->q->dLinv.get(), Mp, s->dP2.get(), Mp, s->dP3.get(), Mp, Mp, Np, Mp, 2, 0.0))) return rc;
    if ((rc = gemm<true, true>(s, s->q->dLinv.get(), Mp, s->dV.get(), Mp, s->dP2.get(), Mp, Mp, Np, Mp, 2, 0.0))) return rc;
    spgp_coldot_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dP2.get(), Mp, Np, nullptr, nullptr, sq_lv);
    spgp_nvec_kernel<<<1, 1024, 0, s->st>>>(yt, mu, bv, sq_lmv, ep, sumvsq, sq_lv, N, Np, c, sig, jitter, r, big, s->dS.get());
    // TT = invLV diag(bigsum) invLV^T (:518)
    spgp_scale_cols_kernel<<<nblocks(Mp * Np, 256), 256, 0, s->st>>>(s->dP2.get(), Mp, Np, big, s->dP1.get());
    s->launches += 3;
    if ((rc = gemm<false, false>(s, s->dP2.get(), Mp, s->dP1.get(), Mp, s->dTT.get(), Mp, Mp, Mp, Np, 0, 0.0))) return rc;
    // invQ = L^-T L^-1 (:507), invA = Z^T Z with Z = Lm^-1 L^-1 (:508-509)
    if ((rc = lb_launch_kinv(s->q))) return rc;
    if ((rc = lb_launch_symmetrize(s->q, s->q->dKinv.get()))) return rc;
    if ((rc = gemm<false, true>(s, s->a->dLinv.get(), Mp, s->q->dLinv.get(), Mp, s->dZ.get(), Mp, Mp, Mp, Mp, 1, 0.0))) return rc;
    if ((rc = gemm<true, true>(s, s->dZ.get(), Mp, s->dZ.get(), Mp, s->dInvA.get(), Mp, Mp, Mp, Mp, 2, 0.0))) return rc;
    // the two weighted passes
    int nsG, nsH;
    const int64_t stripG = pick_strip(s, Mp, N, &nsG), stripH = pick_strip(s, Mp, M, &nsH);
    const int64_t mtb = Mp / 128;
    const size_t offH = (size_t)nsG * (D + 1) * Mp, offBG = offH + (size_t)nsH * (D + 1) * Mp;
    const size_t offBH = offBG + (size_t)nsG * mtb * D, offX = offBH + (size_t)nsH * mtb * 5;
    const int nxb = (M + 127) / 128;
    if ((rc = s->dWork.reserve(s->device, s->st, sizeof(double) * (offX + (size_t)D * nxb)))) return rc;
    PassArgs pa{};
    pa.E0 = s->dK.get(); pa.E1 = s->dP3.get(); pa.E2 = s->dP2.get(); pa.E3 = nullptr; pa.ld = Mp;
    pa.b1 = b1; pa.r = r; pa.big = big;
    pa.xc = s->dXt.get(); pa.ldxc = Np; pa.xr = s->dXbt.get(); pa.ldxr = Mp;
    pa.cols = N; pa.strip = stripG; pa.D = D; pa.sig = sig;
    pa.rowpart = s->dWork.get(); pa.blkpart = s->dWork.get() + offBG;
    spgp_pass_kernel<0><<<dim3((unsigned)mtb, nsG), 128, 0, s->st>>>(pa);
    PassArgs ph = pa;
    ph.E0 = s->dQ.get(); ph.E1 = s->q->dKinv.get(); ph.E2 = s->dInvA.get(); ph.E3 = s->dTT.get();
    ph.xc = s->dXbt.get(); ph.ldxc = Mp; ph.cols = M; ph.strip = stripH;
    ph.rowpart = s->dWork.get() + offH; ph.blkpart = s->dWork.get() + offBH;
    spgp_pass_kernel<1><<<dim3((unsigned)mtb, nsH), 128, 0, s->st>>>(ph);
    spgp_dfxb_kernel<<<dim3(nxb, D), 128, 0, s->st>>>(s->dWork.get(), nsG, s->dWork.get() + offH, nsH, Mp, M, D, s->dXbt.get(), s->dSb.get(), s->dOut.get() + 1,
        s->dWork.get() + offX);
    spgp_final_kernel<<<1, 64, 0, s->st>>>(s->dS.get(), s->dWork.get() + offBG, nsG * (int)mtb, s->dWork.get() + offBH, nsH * (int)mtb, s->dWork.get() + offX, nxb,
        s->dSb.get(), M, D, half_nm, (double)N, sig, jitter, 1, s->dOut.get(), s->dOut.get() + 1);
    s->launches += 4;
    LB_CUDA(cudaGetLastError());
    if ((rc = read_info(s))) return rc;
    LB_CUDA(cudaMemcpy(f, s->dOut.get(), sizeof(double), cudaMemcpyDeviceToHost));
    LB_CUDA(cudaMemcpy(grad, s->dOut.get() + 1, sizeof(double) * nw, cudaMemcpyDeviceToHost));
    return LB_OK;
}

// mu - mean and sigma^2 of Mq candidates (device row-major dXq) into dMu / dS2 (Mq each), in chunks of QCHUNK; with grad, also
// the candidate gradients of each chunk (b1 in Mv row 6, ensure_b1), whose outputs start at candidate 0.  The gradient products
// take one more Mp x Cp block behind the forward workspace, whose layout they leave as it is.
int predict(lb_spgp* s, int64_t Mq, const double* dXq, int optimized, double* dMu, double* dS2, const LbGradOut* grad = nullptr)
{
    const int D = s->D;
    const int64_t Mp = s->Mp;
    const int64_t Cp = round_up(std::min<int64_t>(Mq, QCHUNK), LB_TILE);
    int rc;
    if ((rc = set_attrs())) return rc;
    if ((rc = s->dQxt.reserve(s->device, s->st, sizeof(double) * ((grad ? 4 : 3) * Mp * Cp + (size_t)D * Cp + 2 * Cp)))) return rc;
    double* ks = s->dQxt.get() + (size_t)D * Cp;
    double* lst = ks + Mp * Cp;
    double* lmst = lst + Mp * Cp;
    double* sq1 = lmst + Mp * Cp;
    double* sq2 = sq1 + Cp;
    double* tb = sq2 + Cp; // gradients: Lm^-T lmst, then lst - sig Lm^-T lmst
    for (int64_t q0 = 0; q0 < Mq; q0 += QCHUNK) {
        const int64_t nq = std::min<int64_t>(QCHUNK, Mq - q0), nqp = round_up(nq, LB_TILE);
        spgp_stage_kernel<<<dim3(nblocks(nqp, 256), D), 256, 0, s->st>>>(dXq + q0 * D, nq, D, s->dSb.get(), s->dQxt.get(), nqp);
        spgp_kmat_kernel<<<nblocks(Mp * nqp, 256), 256, 0, s->st>>>(s->dXbt.get(), Mp, s->M, s->dQxt.get(), nqp, nq, D, s->c, ks, Mp, nqp, 0, 0.0, nullptr);
        s->launches += 2;
        if ((rc = gemm<false, true>(s, s->q->dLinv.get(), Mp, ks, Mp, lst, Mp, Mp, nqp, Mp, 1, 0.0))) return rc;
        if ((rc = gemm<false, true>(s, s->a->dLinv.get(), Mp, lst, Mp, lmst, Mp, Mp, nqp, Mp, 1, 0.0))) return rc;
        spgp_coldot_kernel<<<nblocks(nq, 8), 256, 0, s->st>>>(lmst, Mp, nq, s->dMv.get(), dMu + q0, sq2);
        spgp_coldot_kernel<<<nblocks(nq, 8), 256, 0, s->st>>>(lst, Mp, nq, nullptr, nullptr, sq1);
        spgp_pred_kernel<<<nblocks(nq, 256), 256, 0, s->st>>>(sq1, sq2, nq, s->c, s->sig, optimized ? s->sig : 0.0, dS2 + q0);
        s->launches += 3;
        LB_CUDA(cudaGetLastError());
        if (!grad) continue;
        // u = L^-T (lst - sig Lm^-T lmst) over lmst, which the forward reductions above have already read
        if ((rc = gemm<true, true>(s, s->a->dLinv.get(), Mp, lmst, Mp, tb, Mp, Mp, nqp, Mp, 2, 0.0))) return rc;
        spgp_resid_kernel<<<nblocks(Mp * nqp, 256), 256, 0, s->st>>>(lst, tb, Mp * nqp, s->sig);
        s->launches++;
        if ((rc = gemm<true, true>(s, s->q->dLinv.get(), Mp, tb, Mp, lmst, Mp, Mp, nqp, Mp, 2, 0.0))) return rc;
        LbGradOut o = *grad;
        o.mean = grad->mean ? grad->mean + q0 : nullptr;
        o.mean_grad = grad->mean_grad ? grad->mean_grad + q0 * D : nullptr;
        o.dmu = grad->dmu ? grad->dmu + q0 * D : nullptr;
        o.ds2 = grad->ds2 ? grad->ds2 + q0 * D : nullptr;
        o.acq = grad->acq ? grad->acq + q0 : nullptr;
        o.grad = grad->grad ? grad->grad + q0 * D : nullptr;
        spgp_query_grad_kernel<<<(unsigned)nq, GRAD_THREADS, 0, s->st>>>(ks, lmst, Mp, s->M, s->dMv.get() + 6 * Mp, s->dXbt.get(),
            s->dQxt.get(), nqp, s->dSb.get(), D, dMu + q0, dS2 + q0, o);
        s->launches++;
        LB_CUDA(cudaGetLastError());
    }
    return LB_OK;
}

// the outputs and argmax records of Mq candidates
int ensure_query_ws(lb_spgp* s, int64_t Mq)
{
    const size_t mq = sizeof(double) * Mq;
    int rc;
    for (DevBuf<double>* b : {&s->dMu, &s->dS2, &s->am.vals, &s->am.mean})
        if ((rc = b->reserve(s->device, s->st, mq))) return rc;
    return s->am.reserve(s->device, s->st, Mq);
}

// ensure_query_ws and the upload of Mq host candidates to dQx
int ensure_query(lb_spgp* s, int64_t Mq, const double* Xq)
{
    const size_t mq = sizeof(double) * Mq;
    int rc;
    if ((rc = ensure_query_ws(s, Mq)) || (rc = s->dQx.reserve(s->device, s->st, mq * s->D))) return rc;
    LB_CUDA(cudaMemcpyAsync(s->dQx.get(), Xq, mq * s->D, cudaMemcpyHostToDevice, s->st));
    return LB_OK;
}

// the fused UCB / EI and argmax of lb_spgp_acq_argmax over the Mq predictions in s->dMu / s->dS2 (dMean: device, NULL for none),
// values into dAcq (NULL: not kept)
int acq_score(lb_spgp* s, int acq_id, const double* acq_params, int64_t Mq, const double* dMean, double mean_const, double* dAcq,
    double* dBestVal, long long* dBestIdx)
{
    return lb_launch_acq_full(s->st, acq_id, acq_params[0], acq_params[1], Mq, s->dMu.get(), 1, dMean, mean_const, s->dS2.get(), dAcq,
        s->am.blk_val.get(), s->am.blk_idx.get(), dBestVal, dBestIdx, &s->launches);
}

// b1 = L^-T (Lm^-T bet) into Mv row 6 (row 5: Lm^-T bet), once per set of factors; the likelihood's own b1 (row 2) is not touched
int ensure_b1(lb_spgp* s)
{
    if (s->b1_ready) return LB_OK;
    const int64_t Mp = s->Mp;
    double* t = s->dMv.get() + 5 * Mp;
    spgp_coldot_kernel<<<nblocks(Mp, 8), 256, 0, s->st>>>(s->a->dLinv.get(), Mp, Mp, s->dMv.get(), t, nullptr);
    spgp_coldot_kernel<<<nblocks(Mp, 8), 256, 0, s->st>>>(s->q->dLinv.get(), Mp, Mp, t, s->dMv.get() + 6 * Mp, nullptr);
    s->launches += 2;
    LB_CUDA(cudaGetLastError());
    s->b1_ready = true;
    return LB_OK;
}

// lb_spgp_query_grad / lb_spgp_acq_grad (acq_id < 0: no acquisition): the arguments are checked by the callers
int grad_common(lb_spgp* s, int64_t Mq, const double* Xq, int optimized, int acq_id, const double* acq_params, const double* mean_at_q,
    double mean_const, const double* mean_grad, double* mu_out, double* s2_out, double* dmu_out, double* ds2_out, double* acq_out,
    double* grad_out)
{
    const int D = s->D;
    for (int64_t i = 0; i < Mq * D; ++i)
        if (!std::isfinite(Xq[i])) return LB_ERR_ARG;
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->computed) return LB_ERR_STATE;
    LB_DEVICE(s);
    int rc;
    if ((rc = ensure_query(s, Mq, Xq))) return rc;
    const size_t md = (size_t)Mq * D;
    if ((rc = s->dGrad.reserve(s->device, s->st, sizeof(double) * 4 * md))) return rc;
    double* g = s->dGrad.get();
    LbGradOut out{};
    out.acq_id = acq_id;
    out.p0 = acq_id >= 0 ? acq_params[0] : 0.0;
    out.p1 = acq_id == LB_ACQ_EI ? acq_params[1] : 0.0;
    out.mean_const = mean_const;
    if (mean_at_q) {
        LB_CUDA(cudaMemcpyAsync(s->am.mean.get(), mean_at_q, sizeof(double) * Mq, cudaMemcpyHostToDevice, s->st));
        out.mean = s->am.mean.get();
    }
    if (mean_grad) {
        LB_CUDA(cudaMemcpyAsync(g, mean_grad, sizeof(double) * md, cudaMemcpyHostToDevice, s->st));
        out.mean_grad = g;
    }
    out.dmu = dmu_out ? g + md : nullptr;
    out.ds2 = ds2_out ? g + 2 * md : nullptr;
    out.acq = acq_out ? s->am.vals.get() : nullptr;
    out.grad = grad_out ? g + 3 * md : nullptr;
    if ((rc = ensure_b1(s)) || (rc = predict(s, Mq, s->dQx.get(), optimized, s->dMu.get(), s->dS2.get(), &out))) return rc;
    const auto back = [&](double* dst, const double* src, size_t n) -> int {
        if (dst) LB_CUDA(cudaMemcpyAsync(dst, src, sizeof(double) * n, cudaMemcpyDeviceToHost, s->st));
        return LB_OK;
    };
    if ((rc = back(mu_out, s->dMu.get(), Mq)) || (rc = back(s2_out, s->dS2.get(), Mq)) || (rc = back(dmu_out, out.dmu, md))
        || (rc = back(ds2_out, out.ds2, md)) || (rc = back(acq_out, out.acq, Mq)) || (rc = back(grad_out, out.grad, md)))
        return rc;
    LB_CUDA(cudaStreamSynchronize(s->st));
    return LB_OK;
}

} // namespace

extern "C" {

int lb_spgp_create(lb_spgp** out, int device)
{
    if (!out) return LB_ERR_ARG;
    *out = nullptr;
    lb_spgp* s = new (std::nothrow) lb_spgp();
    if (!s) return LB_ERR_ALLOC;
    s->device = device;
    int rc = lb_create(&s->q, device, LB_PREC_FP64);
    if (!rc) rc = lb_create(&s->a, device, LB_PREC_FP64);
    if (rc) {
        lb_destroy(s->q);
        delete s;
        return rc;
    }
    DeviceGuard g(device);
    s->st = s->q->stream;
    if ((rc = lb_set_stream(s->a, s->st))) { // one stream for the whole evaluation (A's factor has its own side stream)
        lb_spgp_destroy(s);
        return rc;
    }
    cudaDeviceGetAttribute(&s->sms, cudaDevAttrMultiProcessorCount, device);
    *out = s;
    return LB_OK;
}

int lb_spgp_destroy(lb_spgp* s)
{
    if (!s) return LB_OK;
    DeviceGuard g(s->device);
    cudaStreamSynchronize(s->st);
    if (s->a) { lb_set_stream(s->a, nullptr); free_inner(s->a); lb_destroy(s->a); }
    if (s->q) { free_inner(s->q); lb_destroy(s->q); }
    delete s; // its buffers go back to the pool
    return LB_OK;
}

int lb_spgp_set_data(lb_spgp* s, int64_t N, int D, const double* X_rowmajor, const double* y_zm)
{
    if (!s || N < 1 || D < 1 || !X_rowmajor || !y_zm) return LB_ERR_ARG;
    if (D > LB_MAX_D) return LB_ERR_UNSUPPORTED;
    for (int64_t i = 0; i < N * D; ++i)
        if (!std::isfinite(X_rowmajor[i])) return LB_ERR_ARG;
    for (int64_t i = 0; i < N; ++i)
        if (!std::isfinite(y_zm[i])) return LB_ERR_ARG;
    std::lock_guard<std::mutex> lk(s->mu);
    LB_DEVICE(s);
    LB_CUDA(cudaStreamSynchronize(s->st));
    const int64_t Np = round_up(N, LB_TILE);
    int rc;
    if ((rc = s->dX.resize(s->device, s->st, sizeof(double) * Np * D)) || (rc = s->dY.resize(s->device, s->st, sizeof(double) * Np))) return rc;
    s->N = N;
    s->Np = Np;
    s->D = D;
    s->computed = false;
    s->b1_ready = false;
    LB_CUDA(cudaMemcpyAsync(s->dX.get(), X_rowmajor, sizeof(double) * N * D, cudaMemcpyHostToDevice, s->st));
    LB_CUDA(cudaMemsetAsync(s->dY.get(), 0, sizeof(double) * Np, s->st));
    LB_CUDA(cudaMemcpyAsync(s->dY.get(), y_zm, sizeof(double) * N, cudaMemcpyHostToDevice, s->st));
    LB_CUDA(cudaStreamSynchronize(s->st));
    return LB_OK;
}

int lb_spgp_lik(lb_spgp* s, int64_t M, int64_t n_w, const double* w, double jitter, double* f, double* grad)
{
    if (!s || !f || !std::isfinite(jitter)) return LB_ERR_ARG;
    if (s->N == 0) return LB_ERR_STATE;
    int rc = check_w(s, M, n_w, w);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(s->mu);
    LB_DEVICE(s);
    s->computed = false; // the factors now belong to this w
    s->b1_ready = false;
    return likelihood(s, (int)M, w, jitter, f, grad);
}

int lb_spgp_compute(lb_spgp* s, int64_t M, int64_t n_w, const double* w, double jitter)
{
    if (!s || !std::isfinite(jitter)) return LB_ERR_ARG;
    if (s->N == 0) return LB_ERR_STATE;
    int rc = check_w(s, M, n_w, w);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(s->mu);
    LB_DEVICE(s);
    s->computed = false;
    s->b1_ready = false;
    double c, sig;
    if ((rc = forward(s, (int)M, w, jitter, &c, &sig))) return rc;
    if ((rc = read_info(s))) return rc;
    s->c = c;
    s->sig = sig;
    s->computed = true;
    return LB_OK;
}

int lb_spgp_query(const lb_spgp* sc, int64_t Mq, const double* Xq_rowmajor, int optimized, double* mu_minus_mean, double* sigma2)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || Mq < 0 || (Mq > 0 && (!Xq_rowmajor || !mu_minus_mean || !sigma2))) return LB_ERR_ARG;
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->computed) return LB_ERR_STATE;
    if (Mq == 0) return LB_OK;
    LB_DEVICE(s);
    int rc;
    if ((rc = ensure_query(s, Mq, Xq_rowmajor))) return rc;
    if ((rc = predict(s, Mq, s->dQx.get(), optimized, s->dMu.get(), s->dS2.get()))) return rc;
    LB_CUDA(cudaMemcpyAsync(mu_minus_mean, s->dMu.get(), sizeof(double) * Mq, cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaMemcpyAsync(sigma2, s->dS2.get(), sizeof(double) * Mq, cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaStreamSynchronize(s->st));
    return LB_OK;
}

int lb_spgp_acq_argmax(const lb_spgp* sc, int acq_id, const double* acq_params, int64_t Mq, const double* Xq_rowmajor, int optimized,
    const double* mean_at_q, double mean_const, double* acq_out, double* best_val, int64_t* best_idx)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || !acq_params || Mq < 1 || !Xq_rowmajor || !best_val || !best_idx) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_ARG;
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->computed) return LB_ERR_STATE;
    LB_DEVICE(s);
    int rc;
    if ((rc = ensure_query(s, Mq, Xq_rowmajor))) return rc;
    if ((rc = predict(s, Mq, s->dQx.get(), optimized, s->dMu.get(), s->dS2.get()))) return rc;
    ArgmaxWs& am = s->am;
    const double* dMean = nullptr;
    if (mean_at_q) {
        LB_CUDA(cudaMemcpyAsync(am.mean.get(), mean_at_q, sizeof(double) * Mq, cudaMemcpyHostToDevice, s->st));
        dMean = am.mean.get();
    }
    if ((rc = acq_score(s, acq_id, acq_params, Mq, dMean, mean_const, am.vals.get(), am.best_val.get(), am.best_idx.get()))) return rc;
    return am.read_best(s->st, best_val, best_idx, acq_out, Mq);
}

int lb_spgp_query_dev(const lb_spgp* sc, int64_t Mq, const double* dXq_rowmajor, int optimized, double* dMu_minus_mean, double* dSigma2)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || Mq < 0 || (Mq > 0 && (!dXq_rowmajor || !dMu_minus_mean || !dSigma2))) return LB_ERR_ARG;
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->computed) return LB_ERR_STATE;
    if (Mq == 0) return LB_OK;
    LB_DEVICE(s);
    return predict(s, Mq, dXq_rowmajor, optimized, dMu_minus_mean, dSigma2);
}

int lb_spgp_acq_argmax_dev(const lb_spgp* sc, int acq_id, const double* acq_params, int64_t Mq, const double* dXq_rowmajor, int optimized,
    const double* dMean_at_q, double mean_const, double* dAcq_out, double* dBest_val, int64_t* dBest_idx)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || !acq_params || Mq < 1 || !dXq_rowmajor || !dBest_val || !dBest_idx) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_ARG;
    std::lock_guard<std::mutex> lk(s->mu);
    if (!s->computed) return LB_ERR_STATE;
    LB_DEVICE(s);
    int rc;
    if ((rc = ensure_query_ws(s, Mq)) || (rc = predict(s, Mq, dXq_rowmajor, optimized, s->dMu.get(), s->dS2.get()))) return rc;
    return acq_score(s, acq_id, acq_params, Mq, dMean_at_q, mean_const, dAcq_out, dBest_val, (long long*)dBest_idx);
}

int lb_spgp_acq_cmaes(const lb_spgp* sc, int acq_id, const double* acq_params, int optimized, double mean_const, const lb_cmaes_opts* opts,
    int64_t R, const double* starts_rowmajor, double* best_x, double* best_val, int64_t* n_evals)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || !acq_params) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_ARG;
    int rc = lb_cmaes_args(opts, R, starts_rowmajor, s->D, best_x, best_val, n_evals);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(s->mu); // the model stays the same for the whole search
    if (!s->computed) return LB_ERR_STATE;
    LB_DEVICE(s);
    const LbCmaesHost on{s->device, s->st, s->D, &s->launches, {nullptr, nullptr, nullptr}}; // fp64 only: no timeout word
    return lb_cmaes_search(
        on, opts, R, starts_rowmajor, [&](int64_t M) { return ensure_query_ws(s, M); },
        [&](const double* dCand, int64_t M, double* dVals, double* dBV, long long* dBI) {
            int e = predict(s, M, dCand, optimized, s->dMu.get(), s->dS2.get());
            return e ? e : acq_score(s, acq_id, acq_params, M, nullptr, mean_const, dVals, dBV, dBI);
        },
        best_x, best_val, n_evals);
}

int lb_spgp_query_grad(const lb_spgp* sc, int64_t Mq, const double* Xq_rowmajor, int optimized, double* mu_minus_mean, double* sigma2,
    double* dmu, double* dsigma2)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || Mq < 1 || !Xq_rowmajor) return LB_ERR_ARG;
    return grad_common(s, Mq, Xq_rowmajor, optimized, -1, nullptr, nullptr, 0.0, nullptr, mu_minus_mean, sigma2, dmu, dsigma2, nullptr,
        nullptr);
}

int lb_spgp_acq_grad(const lb_spgp* sc, int acq_id, const double* acq_params, int64_t Mq, const double* Xq_rowmajor, int optimized,
    const double* mean_at_q, double mean_const, const double* mean_grad_at_q, double* acq_out, double* grad_out)
{
    lb_spgp* s = const_cast<lb_spgp*>(sc);
    if (!s || !acq_params || Mq < 1 || !Xq_rowmajor) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_ARG;
    return grad_common(s, Mq, Xq_rowmajor, optimized, acq_id, acq_params, mean_at_q, mean_const, mean_grad_at_q, nullptr, nullptr,
        nullptr, nullptr, acq_out, grad_out);
}

long long lb_spgp_launch_count(const lb_spgp* s) { return s ? s->launches + s->q->launches + s->a->launches : 0; }

} // extern "C"
