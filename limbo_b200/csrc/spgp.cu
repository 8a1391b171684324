// limbo_b200/csrc/spgp.cu — Snelson and Ghahramani's pseudo-input sparse GP (FITC) with M learned pseudo-inputs:
// experimental::model::SPGP (src/limbo/experimental/model/spgp.hpp).
//
//   _likelihood / _likelihood_wp  spgp.hpp:446-580  -> lb_spgp_lik
//   _compute(false)               spgp.hpp:389-407  -> lb_spgp_compute
//   _predict                      spgp.hpp:582-610  -> lb_spgp_query / lb_spgp_acq_argmax
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
// Layout: M is padded to Mp = roundup(M, 128) and N to Np = roundup(N, 128); padded rows and columns of K are zero, so they
// contribute nothing, and the padded parts of Q and A factor as the identity resp. sig I.
#include "../../include/limbo_b200.h"
#include "gemm.cuh"
#include <algorithm>
#include <cmath>
#include <mutex>
#include <new>

int lb_launch_linv(lb_gp* h);                  // lml.cu
int lb_launch_symmetrize(lb_gp* h, double* dA); // lml.cu
int lb_launch_acq_full(cudaStream_t st, int acq_id, double p0, double p1, int64_t M, const double* dMu, int mu_stride,
    const double* dMeanAtQ, double mean_const, const double* dS2, double* dAcq, double* dBlkVal, long long* dBlkIdx,
    double* dBestVal, long long* dBestIdx, long long* launches); // query.cu

namespace {

using GC = lbg::CfgDual;
constexpr int PASS_DC = 8;    // input dimensions per sweep of spgp_pass_kernel
constexpr int QCHUNK = 8192;  // candidates per prediction chunk

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
    double* dX = nullptr; // N x D row-major
    double* dY = nullptr; // Np, zero padded

    int M = 0;
    int64_t Mp = 0, mp_alloc = 0, np_alloc = 0;
    double *dXt = nullptr, *dXbt = nullptr, *dSb = nullptr;
    double* dW = nullptr; size_t w_cap = 0; // w
    double *dK = nullptr, *dV = nullptr, *dP1 = nullptr, *dP2 = nullptr, *dP3 = nullptr; // Mp x Np
    double *dQ = nullptr, *dZ = nullptr, *dInvA = nullptr, *dTT = nullptr;               // Mp x Mp
    double* dNv = nullptr;  // N-vectors, 12 x Np
    double* dMv = nullptr;  // M-vectors, 8 x Mp
    double* dS = nullptr;   // scalars
    double* dOut = nullptr; size_t out_cap = 0; // f, grad
    double* dWork = nullptr; size_t work_cap = 0; // split-K slices, row / block partials
    // prediction state (lb_spgp_compute)
    bool computed = false;
    double c = 0, sig = 0;
    // query workspace
    double *dQx = nullptr, *dQxt = nullptr, *dKs = nullptr, *dLst = nullptr, *dLmst = nullptr, *dQv = nullptr; size_t q_cap = 0;
    double *dMu = nullptr, *dS2 = nullptr, *dAcq = nullptr, *dMeanQ = nullptr, *dBlk = nullptr; long long *dBlkIdx = nullptr, *dBestIdx = nullptr;
    double* dBest = nullptr;
    int64_t mq_cap = 0;
};

namespace {

void spfree(void*& p)
{
    lb_pool_free(p);
    p = nullptr;
}
#define SP_FREE(p) spfree(reinterpret_cast<void*&>(p))

template <typename T>
int spalloc(lb_spgp* s, T** p, size_t bytes)
{
    *p = static_cast<T*>(lb_pool_alloc(s->device, bytes));
    return *p ? LB_OK : LB_ERR_ALLOC;
}
#define SP_ALLOC(s, p, bytes)                           \
    do {                                                \
        int rc_ = spalloc((s), &(p), (bytes));          \
        if (rc_) return rc_;                            \
    } while (0)

void free_inner(lb_gp* h)
{
    void* all[] = {h->dL, h->dInvD, h->dLinv, h->dKinv};
    for (void* p : all) lb_pool_free(p);
    h->dL = h->dInvD = h->dLinv = h->dKinv = nullptr;
    h->linv_valid = h->kinv_valid = false;
    h->linv_levels = 0;
    h->Np = 0;
}

int ensure_inner(lb_spgp* s, lb_gp* h, int64_t Mp, int M)
{
    if (h->Np != Mp) {
        free_inner(h);
        const int64_t T = Mp / LB_TILE;
        SP_ALLOC(s, h->dL, sizeof(double) * Mp * Mp);
        SP_ALLOC(s, h->dInvD, sizeof(double) * T * LB_TILE * LB_TILE);
        LB_CUDA(cudaMemsetAsync(h->dInvD, 0, sizeof(double) * T * LB_TILE * LB_TILE, s->st));
        h->Np = Mp;
    }
    h->N = M;
    h->linv_valid = h->kinv_valid = false; // a new factor invalidates the inverses
    h->linv_levels = 0;
    return LB_OK;
}

void free_state(lb_spgp* s)
{
    SP_FREE(s->dXt); SP_FREE(s->dXbt); SP_FREE(s->dSb);
    SP_FREE(s->dK); SP_FREE(s->dV); SP_FREE(s->dP1); SP_FREE(s->dP2); SP_FREE(s->dP3);
    SP_FREE(s->dQ); SP_FREE(s->dZ); SP_FREE(s->dInvA); SP_FREE(s->dTT);
    SP_FREE(s->dNv); SP_FREE(s->dMv);
    s->mp_alloc = s->np_alloc = 0;
    s->computed = false;
}

int ensure_state(lb_spgp* s, int M)
{
    const int64_t Mp = round_up(M, LB_TILE), Np = s->Np;
    s->M = M;
    s->Mp = Mp;
    if (s->mp_alloc != Mp || s->np_alloc != Np) {
        cudaStreamSynchronize(s->st);
        free_state(s);
        const size_t mn = sizeof(double) * Mp * Np, mm = sizeof(double) * Mp * Mp;
        SP_ALLOC(s, s->dXt, sizeof(double) * s->D * Np);
        SP_ALLOC(s, s->dXbt, sizeof(double) * s->D * Mp);
        SP_ALLOC(s, s->dSb, sizeof(double) * LB_MAX_D);
        SP_ALLOC(s, s->dK, mn); SP_ALLOC(s, s->dV, mn); SP_ALLOC(s, s->dP1, mn); SP_ALLOC(s, s->dP2, mn); SP_ALLOC(s, s->dP3, mn);
        SP_ALLOC(s, s->dQ, mm); SP_ALLOC(s, s->dZ, mm); SP_ALLOC(s, s->dInvA, mm); SP_ALLOC(s, s->dTT, mm);
        SP_ALLOC(s, s->dNv, sizeof(double) * 12 * Np);
        SP_ALLOC(s, s->dMv, sizeof(double) * 8 * Mp);
        s->mp_alloc = Mp;
        s->np_alloc = Np;
    }
    int rc;
    if ((rc = ensure_inner(s, s->q, Mp, M))) return rc;
    if ((rc = ensure_inner(s, s->a, Mp, M))) return rc;
    return LB_OK;
}

int ensure_buf(lb_spgp* s, double** p, size_t* cap, size_t bytes)
{
    if (*cap >= bytes && *p) return LB_OK;
    cudaStreamSynchronize(s->st);
    SP_FREE(*p);
    *cap = 0;
    SP_ALLOC(s, *p, bytes);
    *cap = bytes;
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
        int rc = ensure_buf(s, &s->dWork, &s->work_cap, sizeof(double) * splits * rows * cols);
        if (rc) return rc;
        out = s->dWork;
    }
    spgp_gemm_kernel<A_KC, B_KC><<<dim3(tiles, splits), GC::THREADS, GC::PIPE_BYTES, s->st>>>(A, lda, B, ldb, out, splits > 1 ? rows : ldc,
        rows * cols, mtiles, (int)K, tri, (int)kchunk, diag);
    s->launches++;
    if (splits > 1) {
        spgp_split_reduce_kernel<<<nblocks(rows * cols, 256), 256, 0, s->st>>>(s->dWork, splits, rows, ldc, C, diag);
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
    LB_CUDA(cudaMemcpyAsync(iq, s->q->dInfo, sizeof(iq), cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaMemcpyAsync(ia, s->a->dInfo, sizeof(ia), cudaMemcpyDeviceToHost, s->st));
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
    if ((rc = ensure_buf(s, &s->dW, &s->w_cap, sizeof(double) * ((M + 1) * D + 2)))) return rc;
    LB_CUDA(cudaMemcpyAsync(s->dSb, sb, sizeof(double) * D, cudaMemcpyHostToDevice, s->st));
    LB_CUDA(cudaMemcpyAsync(s->dW, w, sizeof(double) * ((M + 1) * D + 2), cudaMemcpyHostToDevice, s->st));
    double* ep = s->dNv;
    double* yt = s->dNv + Np;
    double* sumvsq = s->dNv + 2 * Np;
    double* bet = s->dMv;
    spgp_stage_kernel<<<dim3(nblocks(Np, 256), D), 256, 0, s->st>>>(s->dX, N, D, s->dSb, s->dXt, Np);
    spgp_stage_xb_kernel<<<dim3(nblocks(Mp, 256), D), 256, 0, s->st>>>(s->dW, M, s->dSb, s->dXbt, Mp);
    spgp_kmat_kernel<<<nblocks(Mp * Mp, 256), 256, 0, s->st>>>(s->dXbt, Mp, M, s->dXbt, Mp, M, D, c, s->dQ, Mp, Mp, 1, jitter, s->q->dL);
    spgp_kmat_kernel<<<nblocks(Mp * Np, 256), 256, 0, s->st>>>(s->dXbt, Mp, M, s->dXt, Np, N, D, c, s->dK, Mp, Np, 0, 0.0, nullptr);
    s->launches += 4;
    LB_CUDA(cudaGetLastError());
    // L = chol(Q), L^-1
    if ((rc = lb_launch_potrf(s->q))) return rc;
    if ((rc = lb_launch_linv(s->q))) return rc;
    // V = L^-1 K; ep; K~, V~, y~
    if ((rc = gemm<false, true>(s, s->q->dLinv, Mp, s->dK, Mp, s->dV, Mp, Mp, Np, Mp, 1, 0.0))) return rc;
    spgp_ep_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dK, s->dV, Mp, N, Np, s->dY, c, sig, ep, yt, sumvsq);
    s->launches++;
    // Lm = chol(sig I + V~ V~^T), Lm^-1
    if ((rc = gemm<false, false>(s, s->dV, Mp, s->dV, Mp, s->a->dL, Mp, Mp, Mp, Np, 0, sig))) return rc;
    if ((rc = lb_launch_potrf(s->a))) return rc;
    if ((rc = lb_launch_linv(s->a))) return rc;
    // invLmV = Lm^-1 V~, bet = invLmV y~
    if ((rc = gemm<false, true>(s, s->a->dLinv, Mp, s->dV, Mp, s->dP1, Mp, Mp, Np, Mp, 1, 0.0))) return rc;
    int ns;
    const int64_t strip = pick_strip(s, Mp, N, &ns);
    if ((rc = ensure_buf(s, &s->dWork, &s->work_cap, sizeof(double) * ns * Mp))) return rc;
    spgp_rowdot_kernel<<<dim3((unsigned)(Mp / 128), ns), 128, 0, s->st>>>(s->dP1, Mp, N, strip, yt, s->dWork);
    spgp_sum_parts_kernel<<<nblocks(Mp, 256), 256, 0, s->st>>>(s->dWork, ns, Mp, bet);
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
    if ((rc = ensure_buf(s, &s->dOut, &s->out_cap, sizeof(double) * (nw + 1)))) return rc;
    if (!s->dS) SP_ALLOC(s, s->dS, sizeof(double) * 64);
    double* ep = s->dNv;
    double* yt = s->dNv + Np;
    double* sumvsq = s->dNv + 2 * Np;
    double* mu = s->dNv + 3 * Np;
    double* bv = s->dNv + 4 * Np;
    double* sq_lmv = s->dNv + 5 * Np;
    double* sq_lv = s->dNv + 6 * Np;
    double* r = s->dNv + 7 * Np;
    double* big = s->dNv + 8 * Np;
    double* bet = s->dMv;
    double* u = s->dMv + Mp;
    double* b1 = s->dMv + 2 * Mp;
    const double half_nm = (double)((N - M) / 2); // spgp.hpp:491: (n - _m) / 2 in integer arithmetic
    spgp_value_kernel<<<1, 1024, 0, s->st>>>(s->a->dL, Mp, M, bet, yt, ep, N, s->dS);
    s->launches++;
    if (!grad) {
        spgp_final_kernel<<<1, 64, 0, s->st>>>(s->dS, nullptr, 0, nullptr, 0, nullptr, 0, s->dSb, M, D, half_nm, (double)N, sig, jitter, 0,
            s->dOut, s->dOut + 1);
        s->launches++;
        LB_CUDA(cudaGetLastError());
        if ((rc = read_info(s))) return rc;
        LB_CUDA(cudaMemcpy(f, s->dOut, sizeof(double), cudaMemcpyDeviceToHost));
        return LB_OK;
    }
    // bet^T invLmV and colsum(invLmV^2); u = Lm^-T bet; b1 = L^-T u; mu = u^T V~  (spgp.hpp:503, 512, 516)
    spgp_coldot_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dP1, Mp, Np, bet, bv, sq_lmv);
    spgp_coldot_kernel<<<nblocks(Mp, 8), 256, 0, s->st>>>(s->a->dLinv, Mp, Mp, bet, u, nullptr);
    spgp_coldot_kernel<<<nblocks(Mp, 8), 256, 0, s->st>>>(s->q->dLinv, Mp, Mp, u, b1, nullptr);
    spgp_coldot_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dV, Mp, Np, u, mu, nullptr);
    s->launches += 4;
    // B1 = L^-T (Lm^-T invLmV) (:502), invLV = L^-T V~ (:505)
    if ((rc = gemm<true, true>(s, s->a->dLinv, Mp, s->dP1, Mp, s->dP2, Mp, Mp, Np, Mp, 2, 0.0))) return rc;
    if ((rc = gemm<true, true>(s, s->q->dLinv, Mp, s->dP2, Mp, s->dP3, Mp, Mp, Np, Mp, 2, 0.0))) return rc;
    if ((rc = gemm<true, true>(s, s->q->dLinv, Mp, s->dV, Mp, s->dP2, Mp, Mp, Np, Mp, 2, 0.0))) return rc;
    spgp_coldot_kernel<<<nblocks(Np, 8), 256, 0, s->st>>>(s->dP2, Mp, Np, nullptr, nullptr, sq_lv);
    spgp_nvec_kernel<<<1, 1024, 0, s->st>>>(yt, mu, bv, sq_lmv, ep, sumvsq, sq_lv, N, Np, c, sig, jitter, r, big, s->dS);
    // TT = invLV diag(bigsum) invLV^T (:518)
    spgp_scale_cols_kernel<<<nblocks(Mp * Np, 256), 256, 0, s->st>>>(s->dP2, Mp, Np, big, s->dP1);
    s->launches += 3;
    if ((rc = gemm<false, false>(s, s->dP2, Mp, s->dP1, Mp, s->dTT, Mp, Mp, Mp, Np, 0, 0.0))) return rc;
    // invQ = L^-T L^-1 (:507), invA = Z^T Z with Z = Lm^-1 L^-1 (:508-509)
    if ((rc = lb_launch_kinv(s->q))) return rc;
    if ((rc = lb_launch_symmetrize(s->q, s->q->dKinv))) return rc;
    if ((rc = gemm<false, true>(s, s->a->dLinv, Mp, s->q->dLinv, Mp, s->dZ, Mp, Mp, Mp, Mp, 1, 0.0))) return rc;
    if ((rc = gemm<true, true>(s, s->dZ, Mp, s->dZ, Mp, s->dInvA, Mp, Mp, Mp, Mp, 2, 0.0))) return rc;
    // the two weighted passes
    int nsG, nsH;
    const int64_t stripG = pick_strip(s, Mp, N, &nsG), stripH = pick_strip(s, Mp, M, &nsH);
    const int64_t mtb = Mp / 128;
    const size_t offH = (size_t)nsG * (D + 1) * Mp, offBG = offH + (size_t)nsH * (D + 1) * Mp;
    const size_t offBH = offBG + (size_t)nsG * mtb * D, offX = offBH + (size_t)nsH * mtb * 5;
    const int nxb = (M + 127) / 128;
    if ((rc = ensure_buf(s, &s->dWork, &s->work_cap, sizeof(double) * (offX + (size_t)D * nxb)))) return rc;
    PassArgs pa{};
    pa.E0 = s->dK; pa.E1 = s->dP3; pa.E2 = s->dP2; pa.E3 = nullptr; pa.ld = Mp;
    pa.b1 = b1; pa.r = r; pa.big = big;
    pa.xc = s->dXt; pa.ldxc = Np; pa.xr = s->dXbt; pa.ldxr = Mp;
    pa.cols = N; pa.strip = stripG; pa.D = D; pa.sig = sig;
    pa.rowpart = s->dWork; pa.blkpart = s->dWork + offBG;
    spgp_pass_kernel<0><<<dim3((unsigned)mtb, nsG), 128, 0, s->st>>>(pa);
    PassArgs ph = pa;
    ph.E0 = s->dQ; ph.E1 = s->q->dKinv; ph.E2 = s->dInvA; ph.E3 = s->dTT;
    ph.xc = s->dXbt; ph.ldxc = Mp; ph.cols = M; ph.strip = stripH;
    ph.rowpart = s->dWork + offH; ph.blkpart = s->dWork + offBH;
    spgp_pass_kernel<1><<<dim3((unsigned)mtb, nsH), 128, 0, s->st>>>(ph);
    spgp_dfxb_kernel<<<dim3(nxb, D), 128, 0, s->st>>>(s->dWork, nsG, s->dWork + offH, nsH, Mp, M, D, s->dXbt, s->dSb, s->dOut + 1,
        s->dWork + offX);
    spgp_final_kernel<<<1, 64, 0, s->st>>>(s->dS, s->dWork + offBG, nsG * (int)mtb, s->dWork + offBH, nsH * (int)mtb, s->dWork + offX, nxb,
        s->dSb, M, D, half_nm, (double)N, sig, jitter, 1, s->dOut, s->dOut + 1);
    s->launches += 4;
    LB_CUDA(cudaGetLastError());
    if ((rc = read_info(s))) return rc;
    LB_CUDA(cudaMemcpy(f, s->dOut, sizeof(double), cudaMemcpyDeviceToHost));
    LB_CUDA(cudaMemcpy(grad, s->dOut + 1, sizeof(double) * nw, cudaMemcpyDeviceToHost));
    return LB_OK;
}

// mu - mean and sigma^2 of Mq candidates (device row-major dQx) into s->dMu / s->dS2, in chunks of QCHUNK
int predict(lb_spgp* s, int64_t Mq, int optimized)
{
    const int D = s->D;
    const int64_t Mp = s->Mp;
    const int64_t Cp = round_up(std::min<int64_t>(Mq, QCHUNK), LB_TILE);
    int rc;
    if ((rc = set_attrs())) return rc;
    if ((rc = ensure_buf(s, &s->dQxt, &s->q_cap, sizeof(double) * (3 * Mp * Cp + (size_t)D * Cp + 2 * Cp)))) return rc;
    double* ks = s->dQxt + (size_t)D * Cp;
    double* lst = ks + Mp * Cp;
    double* lmst = lst + Mp * Cp;
    double* sq1 = lmst + Mp * Cp;
    double* sq2 = sq1 + Cp;
    for (int64_t q0 = 0; q0 < Mq; q0 += QCHUNK) {
        const int64_t nq = std::min<int64_t>(QCHUNK, Mq - q0), nqp = round_up(nq, LB_TILE);
        spgp_stage_kernel<<<dim3(nblocks(nqp, 256), D), 256, 0, s->st>>>(s->dQx + q0 * D, nq, D, s->dSb, s->dQxt, nqp);
        spgp_kmat_kernel<<<nblocks(Mp * nqp, 256), 256, 0, s->st>>>(s->dXbt, Mp, s->M, s->dQxt, nqp, nq, D, s->c, ks, Mp, nqp, 0, 0.0, nullptr);
        s->launches += 2;
        if ((rc = gemm<false, true>(s, s->q->dLinv, Mp, ks, Mp, lst, Mp, Mp, nqp, Mp, 1, 0.0))) return rc;
        if ((rc = gemm<false, true>(s, s->a->dLinv, Mp, lst, Mp, lmst, Mp, Mp, nqp, Mp, 1, 0.0))) return rc;
        spgp_coldot_kernel<<<nblocks(nq, 8), 256, 0, s->st>>>(lmst, Mp, nq, s->dMv, s->dMu + q0, sq2);
        spgp_coldot_kernel<<<nblocks(nq, 8), 256, 0, s->st>>>(lst, Mp, nq, nullptr, nullptr, sq1);
        spgp_pred_kernel<<<nblocks(nq, 256), 256, 0, s->st>>>(sq1, sq2, nq, s->c, s->sig, optimized ? s->sig : 0.0, s->dS2 + q0);
        s->launches += 3;
        LB_CUDA(cudaGetLastError());
    }
    return LB_OK;
}

int ensure_query(lb_spgp* s, int64_t Mq, const double* Xq)
{
    if (Mq > s->mq_cap) {
        cudaStreamSynchronize(s->st);
        SP_FREE(s->dQx); SP_FREE(s->dMu); SP_FREE(s->dS2); SP_FREE(s->dAcq); SP_FREE(s->dMeanQ); SP_FREE(s->dBlk); SP_FREE(s->dBlkIdx); SP_FREE(s->dBest);
        SP_FREE(s->dBestIdx);
        s->mq_cap = 0;
        const int64_t nblk = (Mq + 255) / 256;
        SP_ALLOC(s, s->dQx, sizeof(double) * Mq * s->D);
        SP_ALLOC(s, s->dMu, sizeof(double) * Mq);
        SP_ALLOC(s, s->dS2, sizeof(double) * Mq);
        SP_ALLOC(s, s->dAcq, sizeof(double) * Mq);
        SP_ALLOC(s, s->dMeanQ, sizeof(double) * Mq);
        SP_ALLOC(s, s->dBlk, sizeof(double) * nblk);
        SP_ALLOC(s, s->dBlkIdx, sizeof(long long) * nblk);
        SP_ALLOC(s, s->dBest, sizeof(double));
        SP_ALLOC(s, s->dBestIdx, sizeof(long long));
        s->mq_cap = Mq;
    }
    LB_CUDA(cudaMemcpyAsync(s->dQx, Xq, sizeof(double) * Mq * s->D, cudaMemcpyHostToDevice, s->st));
    return LB_OK;
}

struct SpDevice {
    int prev = -1;
    bool ok = true;
    explicit SpDevice(int dev)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~SpDevice()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};
#define SP_DEVICE(s)                  \
    SpDevice sp_dev__((s)->device);   \
    if (!sp_dev__.ok) return LB_ERR_CUDA

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
    SpDevice g(device);
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
    {
        SpDevice g(s->device);
        cudaStreamSynchronize(s->st);
        free_state(s);
        SP_FREE(s->dX); SP_FREE(s->dY); SP_FREE(s->dW); SP_FREE(s->dS); SP_FREE(s->dOut); SP_FREE(s->dWork); SP_FREE(s->dQxt);
        SP_FREE(s->dQx); SP_FREE(s->dMu); SP_FREE(s->dS2); SP_FREE(s->dAcq); SP_FREE(s->dMeanQ); SP_FREE(s->dBlk); SP_FREE(s->dBlkIdx); SP_FREE(s->dBest);
        SP_FREE(s->dBestIdx);
        if (s->a) { lb_set_stream(s->a, nullptr); free_inner(s->a); lb_destroy(s->a); }
        if (s->q) { free_inner(s->q); lb_destroy(s->q); }
    }
    delete s;
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
    SP_DEVICE(s);
    LB_CUDA(cudaStreamSynchronize(s->st));
    const int64_t Np = round_up(N, LB_TILE);
    if (Np != s->Np || D != s->D) {
        free_state(s);
        SP_FREE(s->dX); SP_FREE(s->dY);
        SP_ALLOC(s, s->dX, sizeof(double) * Np * D);
        SP_ALLOC(s, s->dY, sizeof(double) * Np);
    }
    s->N = N;
    s->Np = Np;
    s->D = D;
    s->computed = false;
    LB_CUDA(cudaMemcpyAsync(s->dX, X_rowmajor, sizeof(double) * N * D, cudaMemcpyHostToDevice, s->st));
    LB_CUDA(cudaMemsetAsync(s->dY, 0, sizeof(double) * Np, s->st));
    LB_CUDA(cudaMemcpyAsync(s->dY, y_zm, sizeof(double) * N, cudaMemcpyHostToDevice, s->st));
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
    SP_DEVICE(s);
    s->computed = false; // the factors now belong to this w
    return likelihood(s, (int)M, w, jitter, f, grad);
}

int lb_spgp_compute(lb_spgp* s, int64_t M, int64_t n_w, const double* w, double jitter)
{
    if (!s || !std::isfinite(jitter)) return LB_ERR_ARG;
    if (s->N == 0) return LB_ERR_STATE;
    int rc = check_w(s, M, n_w, w);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(s->mu);
    SP_DEVICE(s);
    s->computed = false;
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
    SP_DEVICE(s);
    int rc;
    if ((rc = ensure_query(s, Mq, Xq_rowmajor))) return rc;
    if ((rc = predict(s, Mq, optimized))) return rc;
    LB_CUDA(cudaMemcpyAsync(mu_minus_mean, s->dMu, sizeof(double) * Mq, cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaMemcpyAsync(sigma2, s->dS2, sizeof(double) * Mq, cudaMemcpyDeviceToHost, s->st));
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
    SP_DEVICE(s);
    int rc;
    if ((rc = ensure_query(s, Mq, Xq_rowmajor))) return rc;
    if ((rc = predict(s, Mq, optimized))) return rc;
    const double* dMean = nullptr;
    if (mean_at_q) {
        LB_CUDA(cudaMemcpyAsync(s->dMeanQ, mean_at_q, sizeof(double) * Mq, cudaMemcpyHostToDevice, s->st));
        dMean = s->dMeanQ;
    }
    if ((rc = lb_launch_acq_full(s->st, acq_id, acq_params[0], acq_params[1], Mq, s->dMu, 1, dMean, mean_const, s->dS2, s->dAcq, s->dBlk,
             s->dBlkIdx, s->dBest, s->dBestIdx, &s->launches)))
        return rc;
    long long idx = 0;
    LB_CUDA(cudaMemcpyAsync(best_val, s->dBest, sizeof(double), cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaMemcpyAsync(&idx, s->dBestIdx, sizeof(long long), cudaMemcpyDeviceToHost, s->st));
    if (acq_out) LB_CUDA(cudaMemcpyAsync(acq_out, s->dAcq, sizeof(double) * Mq, cudaMemcpyDeviceToHost, s->st));
    LB_CUDA(cudaStreamSynchronize(s->st));
    *best_idx = idx;
    return LB_OK;
}

long long lb_spgp_launch_count(const lb_spgp* s) { return s ? s->launches + s->q->launches + s->a->launches : 0; }

} // extern "C"
