// limbo_b200/csrc/kbuild.cu — N x N kernel-matrix build (HBM-write bound).
//
// Replaces GP::_compute_full_kernel's double loop + mirror (model/gp.hpp:552-562)
// and BaseKernel::operator() (kernel/kernel.hpp:81-84) for SquaredExpARD
// (squared_exp_ard.hpp:138-151, k = 0), MaternFiveHalves
// (matern_five_halves.hpp:104-113), MaternThreeHalves and Exp.
//
// One CTA per lower-triangular 128 x 128 tile.  The two 128-point blocks of X
// (dimension-major, pre-scaled by 1/ell_d for SE-ARD) are staged into shared
// memory with TMA 1-D bulk copies (cp.async.bulk + mbarrier), every kernel
// value is evaluated once and written twice (tile and mirrored tile) with
// 16-byte stores; noise + 1e-8 is fused on the diagonal; the padding region is
// the identity.
#include "pair_tile.cuh"

namespace {

__global__ void scale_x_kernel(const double* __restrict__ X, double* __restrict__ Xs, int64_t Np, KernParams kp)
{
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int d = blockIdx.y;
    if (i >= Np) return;
    // squared_exp_ard.hpp:148: (x1 - x2).cwiseQuotient(_ell); we scale x once
    // by 1/ell_d instead (<= 2 ulp difference on z, see DESIGN.md §6); Lambda columns: common.cuh lb_staged_coord
    Xs[d * Np + i] = lb_staged_coord(kp, d, [&](int r) { return X[r * Np + i]; });
}

// KID: kernel id (compile time, so only one functor is inlined); EDGE: the tile touches the diagonal or the identity
// padding (noise / padding predicates); interior tiles (the vast majority) skip every per-element test.
// NC: 8-column chunks per pass (8: two passes of 64 columns, 128 registers, two CTAs per SM; 4: four passes of 32 columns, fewer
// live accumulators -> three CTAs per SM: the kernels whose per-element arithmetic is long (Matern, Exp: ~45 fp64 instructions)
// are bound by latency / issue, not by HBM, and want the extra warps)
template <int KID, bool EDGE, int NC>
__device__ __forceinline__ void kbuild_tile(const double* __restrict__ Xs, double* __restrict__ K, int64_t N, int64_t Np,
    const KernParams& kp, int bi, int bj, double (*sxi)[LB_TILE], double (*sxj)[LB_TILE], uint64_t* bar)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int li = lane & 7, lj = lane >> 3;
    const int64_t i0 = (int64_t)bi * LB_TILE, j0 = (int64_t)bj * LB_TILE;
    const int r0 = warp * 16 + 2 * li; // local rows r0, r0+1
    const bool diag_tile = (bi == bj);

    if (tid == 0) {
        lb_mbar_init(bar, 1);
        lb_fence_barrier_init();
    }
    __syncthreads();
    uint32_t phase = 0;

    constexpr int NH = 16 / NC, HW = 8 * NC; // passes over the 128 columns, columns per pass
    for (int h = 0; h < NH; ++h) {
        double z[NC][4];
        pair_distances<NC>(Xs, Np, i0, Xs, Np, j0, kp.D, sxi, sxj, bar, phase, h, z);

        const int64_t gi = i0 + r0; // global rows gi, gi+1
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int64_t gj = j0 + h * HW + c * 8 + 2 * lj; // global cols gj, gj+1
            double v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                double k = lb_kernel_from_z(KID, z[c][e], kp);
                if (EDGE) {
                    const int64_t ii = gi + (e & 1), jj = gj + (e >> 1);
                    if (ii == jj) k += kp.noise + 1e-8; // kernel.hpp:83
                    if (ii >= N || jj >= N) k = (ii == jj) ? 1.0 : 0.0; // identity padding
                }
                v[e] = k;
            }
            // tile (rows gi.., col gj / gj+1): two consecutive rows per store
            *reinterpret_cast<double2*>(&K[gi + gj * Np]) = make_double2(v[0], v[1]);
            *reinterpret_cast<double2*>(&K[gi + (gj + 1) * Np]) = make_double2(v[2], v[3]);
            if (!diag_tile) { // mirrored tile, gp.hpp:560-562
                *reinterpret_cast<double2*>(&K[gj + gi * Np]) = make_double2(v[0], v[2]);
                *reinterpret_cast<double2*>(&K[gj + (gi + 1) * Np]) = make_double2(v[1], v[3]);
            }
        }
    }
}

template <int KID>
__global__ void __launch_bounds__(256, (KID == LB_K_SE_ARD) ? 2 : 3)
kbuild_kernel(const double* __restrict__ Xs, double* __restrict__ K, int64_t N, int64_t Np, KernParams kp)
{
    __shared__ __align__(128) double sxi[DCH][LB_TILE];
    __shared__ __align__(128) double sxj[DCH][LB_TILE];
    __shared__ __align__(8) uint64_t bar;
    int bi, bj;
    tile_from_index(blockIdx.x, bi, bj);
    const bool edge = (bi == bj) || ((int64_t)(bi + 1) * LB_TILE > N);
    constexpr int NC = (KID == LB_K_SE_ARD) ? 8 : 4;
    if (edge) kbuild_tile<KID, true, NC>(Xs, K, N, Np, kp, bi, bj, sxi, sxj, &bar);
    else kbuild_tile<KID, false, NC>(Xs, K, N, Np, kp, bi, bj, sxi, sxj, &bar);
}

} // namespace

int lb_launch_scale_x(lb_gp* h)
{
    dim3 grid((unsigned)((h->Np + 255) / 256), (unsigned)h->kp.D);
    scale_x_kernel<<<grid, 256, 0, h->stream>>>(h->dX, h->dXs, h->Np, h->kp);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_kbuild(lb_gp* h, double* dK)
{
    const int64_t T = h->Np / LB_TILE;
    const int64_t tiles = T * (T + 1) / 2;
    LbProfScope ps(h, h->stream, LB_PC_KBUILD);
    switch (h->kp.id) {
    case LB_K_SE_ARD: kbuild_kernel<LB_K_SE_ARD><<<(unsigned)tiles, 256, 0, h->stream>>>(h->dXs, dK, h->N, h->Np, h->kp); break;
    case LB_K_MATERN52: kbuild_kernel<LB_K_MATERN52><<<(unsigned)tiles, 256, 0, h->stream>>>(h->dXs, dK, h->N, h->Np, h->kp); break;
    case LB_K_MATERN32: kbuild_kernel<LB_K_MATERN32><<<(unsigned)tiles, 256, 0, h->stream>>>(h->dXs, dK, h->N, h->Np, h->kp); break;
    default: kbuild_kernel<LB_K_EXP><<<(unsigned)tiles, 256, 0, h->stream>>>(h->dXs, dK, h->N, h->Np, h->kp); break;
    }
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
