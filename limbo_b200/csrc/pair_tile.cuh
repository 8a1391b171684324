// limbo_b200/csrc/pair_tile.cuh — squared distances over a 128 x 128 tile of point pairs, shared by the K build
// (kbuild.cu), K* (query.cu) and the likelihood gradient (lml.cu).
//
// Both point sets are dimension-major (one 128-point block of one dimension is a contiguous 1 KB run).  A pass stages
// DCH dimensions of the tile's 128 rows and 128 columns into shared memory with 1-D bulk copies behind one mbarrier,
// which the caller initialises (count 1, lb_fence_barrier_init) and publishes with a __syncthreads before the first pass.
//
// Thread-to-element mapping (256 threads, 8 warps): a thread owns rows 16 * warp + 2 * (lane & 7) + {0, 1} and, in
// column pass h of 8 * NC columns, columns h * 8NC + 8c + 2 * (lane >> 3) + {0, 1} for c < NC; z[c][e] is the pair
// (row + (e & 1), column + (e >> 1)).
#pragma once
#include "common.cuh"

constexpr int DCH = 16; // input dimensions staged per pass

// t-th lower-triangular tile, rows first: (0,0), (1,0), (1,1), (2,0), ...
__device__ __forceinline__ void tile_from_index(int t, int& bi, int& bj)
{
    int r = (int)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
    while ((int64_t)(r + 1) * (r + 2) / 2 <= t) ++r;
    while ((int64_t)r * (r + 1) / 2 > t) --r;
    bi = r;
    bj = t - r * (r + 1) / 2;
}

// Stage pass `pass` (dimensions pass * DCH ..) of the rows i0.. of A (leading dimension lda) into sa and of the columns
// j0.. of B (leading dimension ldb) into sb; returns once every thread sees the data.  Flips phase; returns the number
// of dimensions staged.
__device__ __forceinline__ int pair_stage(const double* __restrict__ A, int64_t lda, int64_t i0, const double* __restrict__ B,
    int64_t ldb, int64_t j0, int D, int pass, double (*sa)[LB_TILE], double (*sb)[LB_TILE], uint64_t* bar, uint32_t& phase)
{
    const int d0 = pass * DCH;
    const int dc = min(DCH, D - d0);
    __syncthreads(); // previous readers done before the copies overwrite
    if (threadIdx.x == 0) {
        lb_fence_proxy_async();
        lb_mbar_expect_tx(bar, (uint32_t)(2 * dc * LB_TILE * sizeof(double)));
        for (int d = 0; d < dc; ++d) {
            lb_bulk_g2s(&sa[d][0], A + (int64_t)(d0 + d) * lda + i0, LB_TILE * sizeof(double), bar);
            lb_bulk_g2s(&sb[d][0], B + (int64_t)(d0 + d) * ldb + j0, LB_TILE * sizeof(double), bar);
        }
    }
    lb_mbar_wait(bar, phase);
    phase ^= 1;
    return dc;
}

// z[c][e] = sum_d (a_d - b_d)^2 over the D dimensions for column pass h (mapping above), one fma per dimension in ascending
// order.  When one pass holds every dimension, column passes h >= 1 reuse what h = 0 staged.
template <int NC>
__device__ __forceinline__ void pair_distances(const double* __restrict__ A, int64_t lda, int64_t i0, const double* __restrict__ B,
    int64_t ldb, int64_t j0, int D, double (*sa)[LB_TILE], double (*sb)[LB_TILE], uint64_t* bar, uint32_t& phase, int h,
    double (&z)[NC][4])
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int li = lane & 7, lj = lane >> 3;
    const int r0 = warp * 16 + 2 * li;
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
        for (int e = 0; e < 4; ++e) z[c][e] = 0.0;
    const int npass = (D + DCH - 1) / DCH;
    for (int pass = 0; pass < npass; ++pass) {
        const int dc = min(DCH, D - pass * DCH);
        if (!(npass == 1 && h >= 1)) pair_stage(A, lda, i0, B, ldb, j0, D, pass, sa, sb, bar, phase);
        for (int d = 0; d < dc; ++d) {
            const double2 xi = *reinterpret_cast<const double2*>(&sa[d][r0]);
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                const double2 xj = *reinterpret_cast<const double2*>(&sb[d][h * 8 * NC + c * 8 + 2 * lj]);
                double q;
                q = xi.x - xj.x; z[c][0] = fma(q, q, z[c][0]);
                q = xi.y - xj.x; z[c][1] = fma(q, q, z[c][1]);
                q = xi.x - xj.y; z[c][2] = fma(q, q, z[c][2]);
                q = xi.y - xj.y; z[c][3] = fma(q, q, z[c][3]);
            }
        }
    }
}
