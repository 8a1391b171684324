// limbo_b200/csrc/trsv.cu — blocked triangular solves with few right-hand sides
// (HBM-read bound: every byte of the lower triangle of L is read once per
// direction).
//
// Replaces GP::_compute_alpha (model/gp.hpp:605-611):
//     alpha = L^-1 obs_mean ; alpha = L^-T alpha
// One persistent launch per direction: CTA i owns the 128-row block i,
// accumulates  b_i - sum_j L[i,j] x_j  as the x_j become available, then applies
// the pre-inverted diagonal block.  Block ids are handed out by an atomic ticket,
// so a CTA only ever waits on CTAs that started before it (no deadlock; the spin
// is bounded: on timeout info[1] is set and LB_ERR_TIMEOUT returned).
//
// The dependency chain (T sequential blocks) is what bounds these kernels, not
// HBM.  A flag per block (poll flag -> barrier -> load x_j) would cost two L2 round
// trips per step, and fetching the diagonal-block inverse only after the last x_j
// had arrived would add a third.  Instead
//   * the solution is published through a scratch vector pre-filled with a
//     sentinel: consumers poll the 8-byte VALUES themselves (one round trip, no
//     ordering between elements needed);
//   * inv(L_ii) is staged into shared memory with cp.async while the CTA works
//     through its row, so the last step of the chain touches no global memory
//     except the x_j it waits for.
#include "common.cuh"

namespace {

constexpr int NR = 2; // right-hand sides per launch
constexpr long long SPIN_LIMIT = 1LL << 22;
constexpr unsigned long long SENTINEL = 0xFFFFFFFFFFFFFFFFull; // a NaN no arithmetic produces (results carry the canonical quiet NaN)
constexpr size_t TRSV_SMEM = (size_t)LB_TILE * LB_TILE * sizeof(double);

__device__ __forceinline__ unsigned long long ld_poll(const double* p)
{
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_publish(double* p, double v)
{
    asm volatile("st.relaxed.gpu.global.f64 [%0], %1;\n" ::"l"(p), "d"(v) : "memory");
}

// one element of x_j, as soon as its producer has stored it
__device__ __forceinline__ double wait_value(const double* p, int* info)
{
    unsigned long long v = ld_poll(p);
    long long spins = 0;
    while (v == SENTINEL) {
        __nanosleep(20);
        v = ld_poll(p);
        if (++spins > SPIN_LIMIT) {
            atomicExch(info + 1, 1);
            return 0.0;
        }
    }
    return __longlong_as_double((long long)v);
}

__device__ __forceinline__ void stage_invd(double* sInv, const double* __restrict__ Di)
{
    for (int idx = threadIdx.x; idx < LB_TILE * LB_TILE / 2; idx += 256) lb_cp_async16(sInv + 2 * idx, Di + 2 * idx);
    lb_cp_async_commit();
}

// forward: solve L x = b in place (B: Np x nr, column-major, ld = ldb); X: scratch Np x nr, sentinel-filled
__global__ void __launch_bounds__(256, 1)
trsv_fwd_kernel(const double* __restrict__ L, int64_t ld, const double* __restrict__ invD, double* __restrict__ B,
    int64_t ldb, int nr, int T, double* __restrict__ X, int* __restrict__ ticket, int* __restrict__ info)
{
    extern __shared__ __align__(16) double sInv[]; // inv(L_ii), column-major 128 x 128
    __shared__ double xs[NR][LB_TILE];
    __shared__ double part[2][NR][LB_TILE];
    __shared__ int s_i;
    const int tid = threadIdx.x;
    if (tid == 0) s_i = atomicAdd(ticket, 1);
    __syncthreads();
    const int i = s_i;
    stage_invd(sInv, invD + (int64_t)i * LB_TILE * LB_TILE);
    const int r = tid & 127, q = tid >> 7;
    double acc[NR];
#pragma unroll
    for (int p = 0; p < NR; ++p) acc[p] = 0.0;
    // this block's right-hand side, fetched now (off the dependency chain)
    double bi = 0.0;
    if (tid < nr * LB_TILE) bi = B[(int64_t)i * LB_TILE + (tid & 127) + (int64_t)(tid >> 7) * ldb];

    for (int j = 0; j < i; ++j) {
        // issue the loads of L[i,j] before waiting on x_j
        const double* Lt = L + (int64_t)i * LB_TILE + r + ((int64_t)j * LB_TILE + q * 64) * ld;
        double lv[64];
#pragma unroll
        for (int c = 0; c < 64; ++c) lv[c] = __ldcs(Lt + (int64_t)c * ld);
        if (tid < nr * LB_TILE) {
            const int p = tid >> 7, c = tid & 127;
            xs[p][c] = wait_value(X + (int64_t)j * LB_TILE + c + (int64_t)p * ldb, info);
        }
        __syncthreads();
#pragma unroll
        for (int p = 0; p < NR; ++p) {
            if (p < nr) {
                double s = acc[p];
#pragma unroll
                for (int c = 0; c < 64; ++c) s = fma(lv[c], xs[p][q * 64 + c], s);
                acc[p] = s;
            }
        }
        __syncthreads(); // xs reused next iteration
    }
#pragma unroll
    for (int p = 0; p < NR; ++p) part[q][p][r] = acc[p];
    lb_cp_async_wait<0>();
    __syncthreads();
    // rhs block: b_i - sum
    if (tid < nr * LB_TILE) {
        const int p = tid >> 7, c = tid & 127;
        xs[p][c] = bi - (part[0][p][c] + part[1][p][c]);
    }
    __syncthreads();
    // x_i = invD_i * rhs (from shared memory)
#pragma unroll
    for (int p = 0; p < NR; ++p) acc[p] = 0.0;
    const double* Di = sInv + r + (q * 64) * LB_TILE;
#pragma unroll 16
    for (int c = 0; c < 64; ++c) {
        const double dv = Di[c * LB_TILE];
#pragma unroll
        for (int p = 0; p < NR; ++p)
            if (p < nr) acc[p] = fma(dv, xs[p][q * 64 + c], acc[p]);
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < NR; ++p) part[q][p][r] = acc[p];
    __syncthreads();
    for (int idx = tid; idx < nr * LB_TILE; idx += 256) {
        int p = idx >> 7, c = idx & 127;
        const double v = part[0][p][c] + part[1][p][c];
        st_publish(X + (int64_t)i * LB_TILE + c + (int64_t)p * ldb, v); // consumers poll these
        B[(int64_t)i * LB_TILE + c + (int64_t)p * ldb] = v;
    }
}

// backward: solve L^T x = y in place
__global__ void __launch_bounds__(256, 1)
trsv_bwd_kernel(const double* __restrict__ L, int64_t ld, const double* __restrict__ invD, double* __restrict__ B,
    int64_t ldb, int nr, int T, double* __restrict__ X, int* __restrict__ ticket, int* __restrict__ info)
{
    extern __shared__ __align__(16) double sInv[];
    __shared__ double xs[NR][LB_TILE];
    __shared__ double red[NR][LB_TILE];
    __shared__ int s_i;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_i = T - 1 - atomicAdd(ticket, 1);
    __syncthreads();
    const int i = s_i;
    stage_invd(sInv, invD + (int64_t)i * LB_TILE * LB_TILE);
    // warp w owns columns c = w + 8*cc (cc = 0..15) of the block column i
    double acc[NR][16];
#pragma unroll
    for (int p = 0; p < NR; ++p)
#pragma unroll
        for (int cc = 0; cc < 16; ++cc) acc[p][cc] = 0.0;
    double bi = 0.0; // this block's right-hand side, fetched off the dependency chain
    if (tid < nr * LB_TILE) bi = B[(int64_t)i * LB_TILE + (tid & 127) + (int64_t)(tid >> 7) * ldb];

    for (int j = T - 1; j > i; --j) {
        const double* Lt = L + (int64_t)j * LB_TILE + lane + ((int64_t)i * LB_TILE + warp) * ld;
        double lv[16][4];
#pragma unroll
        for (int cc = 0; cc < 16; ++cc)
#pragma unroll
            for (int s = 0; s < 4; ++s) lv[cc][s] = __ldcs(Lt + 32 * s + (int64_t)(8 * cc) * ld);
        if (tid < nr * LB_TILE) {
            const int p = tid >> 7, c = tid & 127;
            xs[p][c] = wait_value(X + (int64_t)j * LB_TILE + c + (int64_t)p * ldb, info);
        }
        __syncthreads();
#pragma unroll
        for (int p = 0; p < NR; ++p) {
            if (p < nr) {
                double xv[4];
#pragma unroll
                for (int s = 0; s < 4; ++s) xv[s] = xs[p][lane + 32 * s];
#pragma unroll
                for (int cc = 0; cc < 16; ++cc)
#pragma unroll
                    for (int s = 0; s < 4; ++s) acc[p][cc] = fma(lv[cc][s], xv[s], acc[p][cc]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int p = 0; p < NR; ++p)
#pragma unroll
        for (int cc = 0; cc < 16; ++cc) {
            double s = lb_warp_sum(acc[p][cc]);
            if (lane == 0) red[p][warp + 8 * cc] = s;
        }
    lb_cp_async_wait<0>();
    __syncthreads();
    if (tid < nr * LB_TILE) {
        const int p = tid >> 7, c = tid & 127;
        xs[p][c] = bi - red[p][c];
    }
    __syncthreads();
    // x_i = invD_i^T * rhs : column dot products over the staged block
#pragma unroll
    for (int p = 0; p < NR; ++p) {
        if (p < nr) {
            for (int cc = 0; cc < 16; ++cc) {
                const int c = warp + 8 * cc;
                double s = 0.0;
#pragma unroll
                for (int k = 0; k < 4; ++k) s = fma(sInv[lane + 32 * k + c * LB_TILE], xs[p][lane + 32 * k], s);
                s = lb_warp_sum(s);
                if (lane == 0) red[p][c] = s;
            }
        }
    }
    __syncthreads();
    for (int idx = tid; idx < nr * LB_TILE; idx += 256) {
        int p = idx >> 7, c = idx & 127;
        const double v = red[p][c];
        st_publish(X + (int64_t)i * LB_TILE + c + (int64_t)p * ldb, v);
        B[(int64_t)i * LB_TILE + c + (int64_t)p * ldb] = v;
    }
}

LbOncePerDevice g_attr_once;

} // namespace

// Solve with the factor held by h, in place on dB (Np x nrhs, ld = Np).
int lb_launch_trsv(lb_gp* h, double* dB, int nrhs, bool forward)
{
    if (g_attr_once.need()) {
        LB_CUDA(cudaFuncSetAttribute(trsv_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TRSV_SMEM));
        LB_CUDA(cudaFuncSetAttribute(trsv_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TRSV_SMEM));
    }
    const int T = (int)(h->Np / LB_TILE);
    // scratch: the published solution blocks (NR columns of Np doubles), sentinel-filled per launch
    int rc = h->dTrsvX.resize(h, sizeof(double) * NR * h->Np);
    if (rc) return rc;
    for (int p0 = 0; p0 < nrhs; p0 += NR) {
        const int nr = (nrhs - p0 < NR) ? (nrhs - p0) : NR;
        LB_CUDA(cudaMemsetAsync(h->dFlags.get(), 0, (T + 1) * sizeof(int), h->stream));
        LB_CUDA(cudaMemsetAsync(h->dTrsvX.get(), 0xFF, sizeof(double) * NR * h->Np, h->stream));
        LbProfScope ps(h, h->stream, LB_PC_TRSV);
        if (forward)
            trsv_fwd_kernel<<<T, 256, TRSV_SMEM, h->stream>>>(h->dL, h->Np, h->dInvD, dB + (int64_t)p0 * h->Np, h->Np, nr, T, h->dTrsvX.get(),
                h->dFlags.get() + T, h->dInfo.get());
        else
            trsv_bwd_kernel<<<T, 256, TRSV_SMEM, h->stream>>>(h->dL, h->Np, h->dInvD, dB + (int64_t)p0 * h->Np, h->Np, nr, T, h->dTrsvX.get(),
                h->dFlags.get() + T, h->dInfo.get());
        h->launches++;
    }
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_launch_solve_alpha(lb_gp* h)
{
    // alpha = obs_mean ; L^-1 ; L^-T      (gp.hpp:608-610)
    LB_CUDA(cudaMemcpyAsync(h->dAlpha, h->dY, sizeof(double) * h->Np * h->P, cudaMemcpyDeviceToDevice, h->stream));
    int rc = lb_launch_trsv(h, h->dAlpha, h->P, true);
    if (rc) return rc;
    return lb_launch_trsv(h, h->dAlpha, h->P, false);
}
