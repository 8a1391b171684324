// limbo_b200/csrc/sparsify.cu — density-based sparsification of a sample set
// (model::SparsifiedGP::_sparsify, model/sparsified_gp.hpp:121-183).
//
// The reference builds the N x N distance matrix, then removes the densest point
// (smallest sum of its k = D nearest distances, _get_most_dense_point) until
// max_points remain, re-sorting every row after every removal.  Here:
//   * init: one thread per row keeps its k nearest live points as (s, j) pairs,
//     s = squared distance, sorted lexicographically (s first, then j), in k x N
//     device arrays: O(N k) memory, O(N^2 D) work, X staged in 128-point tiles;
//   * greedy loop: ONE persistent cooperative launch, three grid barriers per
//     removal, no host round trip:
//       A. rows whose list held the last winner p take the replacement found in C
//          and recompute their score; then every CTA's argmin over its rows;
//       B. every CTA reduces the per-CTA minima to the same winner p, marks it
//          dead and collects the live rows whose list contains p;
//       C. for each such row r, the whole grid looks for the smallest live pair
//          (s_rj, j) above r's old k-th pair.  The other k - 1 entries are still
//          r's nearest, so that pair completes the new list.  Rows without p
//          keep their lists: removing a non-member cannot change the k smallest.
// Distances are s = sum_d t_d * t_d in ascending d from 0.0, every product and sum
// rounded (the stand-in's squaredNorm(), Eigen/Core:105), scores the rounded
// sqrt(s) of the list summed in ascending order from 0.0 (sparsified_gp.hpp:139-143).
// Ties: the winner is the lowest index among equal scores (the sequential par::loop).
// Every grid barrier wait is bounded (WAIT_NS); on timeout the error flag is raised
// and every CTA leaves the loop.
#include "common.cuh"
#include <cfloat>

namespace {

constexpr int INIT_THREADS = 128;
constexpr int LOOP_THREADS = 512;
constexpr int NO_IDX = 0x7fffffff; // sorts after every real index: empty list slots are (+inf, NO_IDX)
constexpr unsigned long long WAIT_NS = 4000000000ull; // bound of one grid-barrier wait (4 s)
enum { CTL_BAR_COUNT = 0, CTL_BAR_GEN = 1, CTL_AFF0 = 2, CTL_ERR = 4, CTL_WORDS = 8 };
enum { SP_ERR_TIMEOUT = 1, SP_ERR_NONFINITE = 2 };

__device__ __forceinline__ bool pair_less(double a, int ia, double b, int ib) { return a < b || (a == b && ia < ib); }

// squared distance between point a (stride sa) and point b (stride sb), in the reference's rounding
__device__ __forceinline__ double dist2(const double* a, int64_t sa, const double* b, int64_t sb, int D)
{
    double s = 0.0;
    for (int d = 0; d < D; ++d) {
        const double t = __dsub_rn(a[d * sa], b[d * sb]);
        s = __dadd_rn(s, __dmul_rn(t, t));
    }
    return s;
}

__device__ __forceinline__ double row_score(const double* nbr_s, int64_t N, int64_t r, int k)
{
    double sum = 0.0;
    for (int i = 0; i < k; ++i) sum = __dadd_rn(sum, __dsqrt_rn(__ldcg(nbr_s + i * N + r)));
    return sum;
}

// lexicographic (s, i) minimum over the CTA; every thread returns the result
__device__ __forceinline__ void block_min_pair(double& s, int& i, double* sh_s, int* sh_i)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, s, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (pair_less(os, oi, s, i)) { s = os; i = oi; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads(); // sh_* may still be read by the previous call
    if (lane == 0) { sh_s[warp] = s; sh_i[warp] = i; }
    __syncthreads();
    s = lane < nw ? sh_s[lane] : __longlong_as_double(0x7ff0000000000000LL);
    i = lane < nw ? sh_i[lane] : NO_IDX;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double os = __shfl_xor_sync(0xffffffffu, s, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (pair_less(os, oi, s, i)) { s = os; i = oi; }
    }
}

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p)
{
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Grid-wide barrier for a cooperative launch (all CTAs co-resident).  Returns false once the error flag is up: the wait
// timed out here or anywhere else, and the caller leaves its loop.
__device__ bool grid_barrier(unsigned* ctl)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        int* err = (int*)(ctl + CTL_ERR);
        const unsigned gen = ld_acquire(ctl + CTL_BAR_GEN);
        __threadfence();
        if (atomicAdd(ctl + CTL_BAR_COUNT, 1u) == gridDim.x - 1) {
            atomicExch(ctl + CTL_BAR_COUNT, 0u);
            __threadfence();
            atomicAdd(ctl + CTL_BAR_GEN, 1u);
        }
        else {
            const unsigned long long t0 = global_ns();
            unsigned spins = 0;
            while (ld_acquire(ctl + CTL_BAR_GEN) == gen) {
                __nanosleep(32);
                if ((++spins & 255) == 0 && (*(volatile int*)err || global_ns() - t0 > WAIT_NS)) {
                    atomicOr(err, SP_ERR_TIMEOUT);
                    break;
                }
            }
        }
        __threadfence();
    }
    __syncthreads();
    return *(volatile int*)(ctl + CTL_ERR) == 0;
}

// row-major N x D -> dimension-major D x N (the layout lb_set_data stores)
__global__ void sparsify_soa_kernel(const double* __restrict__ src, int64_t N, int D, double* __restrict__ dst)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < N) for (int d = 0; d < D; ++d) dst[(int64_t)d * N + i] = src[i * D + d];
}

// k nearest (s, j) pairs of every row, sorted, and the row's score.  X: D x N.  Flags non-finite coordinates.
__global__ void __launch_bounds__(INIT_THREADS) sparsify_knn_init_kernel(const double* __restrict__ X, int64_t N, int D, int k,
    double* __restrict__ nbr_s, int* __restrict__ nbr_j, double* __restrict__ score, int* __restrict__ alive, unsigned* __restrict__ ctl)
{
    extern __shared__ double sm[];
    double* sT = sm;                       // D x 128 tile of candidates
    double* sR = sm + D * INIT_THREADS;    // D x 128 the CTA's own rows
    const int tid = threadIdx.x;
    const int64_t r = blockIdx.x * (int64_t)INIT_THREADS + tid;
    const bool own = r < N;
    for (int d = 0; d < D; ++d) sR[d * INIT_THREADS + tid] = own ? X[(int64_t)d * N + r] : 0.0;
    if (own)
        for (int i = 0; i < k; ++i) { nbr_s[i * N + r] = __longlong_as_double(0x7ff0000000000000LL); nbr_j[i * N + r] = NO_IDX; }
    double worst = __longlong_as_double(0x7ff0000000000000LL);
    int worst_j = NO_IDX;
    bool bad = false;
    for (int64_t j0 = 0; j0 < N; j0 += INIT_THREADS) {
        const int nj = (int)(N - j0 < INIT_THREADS ? N - j0 : INIT_THREADS);
        __syncthreads();
        for (int idx = tid; idx < D * INIT_THREADS; idx += INIT_THREADS) {
            const int d = idx / INIT_THREADS, jj = idx % INIT_THREADS;
            const double v = jj < nj ? X[(int64_t)d * N + j0 + jj] : 0.0;
            bad |= !isfinite(v);
            sT[idx] = v;
        }
        __syncthreads();
        if (!own) continue;
        for (int jj = 0; jj < nj; ++jj) {
            const int j = (int)(j0 + jj);
            if (j == r) continue;
            const double s = dist2(sR + tid, INIT_THREADS, sT + jj, INIT_THREADS, D);
            if (!pair_less(s, j, worst, worst_j)) continue;
            int pos = k - 1; // insertion into the sorted list (rare: O(k log(N / k)) times per row)
            while (pos > 0) {
                const double ps = nbr_s[(pos - 1) * N + r];
                const int pj = nbr_j[(pos - 1) * N + r];
                if (!pair_less(s, j, ps, pj)) break;
                nbr_s[pos * N + r] = ps;
                nbr_j[pos * N + r] = pj;
                --pos;
            }
            nbr_s[pos * N + r] = s;
            nbr_j[pos * N + r] = j;
            worst = nbr_s[(k - 1) * N + r];
            worst_j = nbr_j[(k - 1) * N + r];
        }
    }
    if (bad) atomicOr((int*)(ctl + CTL_ERR), SP_ERR_NONFINITE);
    if (own) {
        score[r] = row_score(nbr_s, N, r, k);
        alive[r] = 1;
    }
}

__global__ void __launch_bounds__(LOOP_THREADS, 1) sparsify_greedy_kernel(const double* __restrict__ X, int64_t N, int D, int k,
    int64_t max_points, double* __restrict__ nbr_s, int* __restrict__ nbr_j, double* __restrict__ score, int* __restrict__ alive,
    int* __restrict__ aff, int* __restrict__ aff_best, double* __restrict__ part_s, int* __restrict__ part_i, unsigned* __restrict__ ctl,
    long long* __restrict__ removed, double* __restrict__ removed_score, long long* __restrict__ n_removed)
{
    __shared__ double sh_s[32];
    __shared__ int sh_i[32];
    __shared__ double sXr[LB_MAX_D];
    const int tid = threadIdx.x, b = blockIdx.x, G = gridDim.x;
    if (*(volatile int*)(ctl + CTL_ERR)) return; // non-finite input (init kernel)
    const int64_t rows = (N + G - 1) / G, row0 = b * rows < N ? b * rows : N,
                  row1 = row0 + rows < N ? row0 + rows : N;
    const double INF = __longlong_as_double(0x7ff0000000000000LL);
    int p = -1, A_prev = 0;
    for (int64_t t = 0, n = N; n > max_points; ++t, --n) {
        // ---- A: refresh the rows of this CTA that lost p, then this CTA's argmin (strict < from DBL_MAX, lowest index) ----
        for (int a = tid; a < A_prev; a += LOOP_THREADS) {
            const int r = __ldcg(aff + a);
            if (r < row0 || r >= row1) continue;
            int i = 0;
            while (i < k - 1 && __ldcg(nbr_j + i * N + r) != p) ++i;
            for (; i < k - 1; ++i) {
                nbr_s[i * N + r] = __ldcg(nbr_s + (i + 1) * N + r);
                nbr_j[i * N + r] = __ldcg(nbr_j + (i + 1) * N + r);
            }
            const int j = __ldcg(aff_best + a);
            nbr_s[(k - 1) * N + r] = j >= 0 ? dist2(X + r, N, X + j, N, D) : INF;
            nbr_j[(k - 1) * N + r] = j >= 0 ? j : NO_IDX;
            score[r] = row_score(nbr_s, N, r, k);
        }
        __syncthreads();
        double bs = DBL_MAX;
        int bi = NO_IDX;
        for (int64_t r = row0 + tid; r < row1; r += LOOP_THREADS) {
            if (!__ldcg(alive + r)) continue;
            const double s = __ldcg(score + r);
            if (s < DBL_MAX && pair_less(s, (int)r, bs, bi)) { bs = s; bi = (int)r; }
        }
        block_min_pair(bs, bi, sh_s, sh_i);
        if (tid == 0) { part_s[b] = bs; part_i[b] = bi; }
        if (!grid_barrier(ctl)) return;

        // ---- B: the winner, and the live rows whose list holds it ----
        bs = DBL_MAX;
        bi = NO_IDX;
        for (int c = tid; c < G; c += LOOP_THREADS) {
            const double s = __ldcg(part_s + c);
            const int i = __ldcg(part_i + c);
            if (pair_less(s, i, bs, bi)) { bs = s; bi = i; }
        }
        block_min_pair(bs, bi, sh_s, sh_i);
        if (bi == NO_IDX) return; // no score < DBL_MAX: the reference's k < 0 break
        p = bi;
        unsigned* cnt = ctl + CTL_AFF0 + (t & 1);
        if (b == 0 && tid == 0) {
            alive[p] = 0;
            removed[t] = p;
            removed_score[t] = bs;
            *n_removed = t + 1;
        }
        for (int64_t r = (int64_t)b * LOOP_THREADS + tid; r < N; r += (int64_t)G * LOOP_THREADS) {
            if (r == p || !__ldcg(alive + r)) continue;
            for (int i = 0; i < k; ++i)
                if (__ldcg(nbr_j + i * N + r) == p) {
                    const unsigned a = atomicAdd(cnt, 1u);
                    aff[a] = (int)r;
                    aff_best[a] = -1;
                    break;
                }
        }
        if (!grid_barrier(ctl)) return;

        // ---- C: replacement of each such row, split over the grid (A rows x nchunk chunks of the points) ----
        const int A = (int)__ldcg(cnt);
        const int64_t per_row = G / (A > 0 ? A : 1), full = (N + LOOP_THREADS - 1) / LOOP_THREADS;
        const int64_t nchunk = per_row < 1 ? 1 : (per_row < full ? per_row : full);
        for (int64_t u = b; u < (int64_t)A * nchunk; u += G) {
            const int a = (int)(u / nchunk);
            const int64_t c = u % nchunk;
            const int r = __ldcg(aff + a);
            __syncthreads();
            if (tid < D) sXr[tid] = X[(int64_t)tid * N + r];
            __syncthreads();
            const double thr_s = __ldcg(nbr_s + (k - 1) * N + r);
            const int thr_j = __ldcg(nbr_j + (k - 1) * N + r);
            const int64_t c0 = c * N / nchunk, c1 = (c + 1) * N / nchunk;
            bs = INF;
            bi = NO_IDX;
            for (int64_t j = c0 + tid; j < c1; j += LOOP_THREADS) {
                if (j == r || j == p || !__ldcg(alive + j)) continue;
                const double s = dist2(sXr, 1, X + j, N, D);
                if (pair_less(thr_s, thr_j, s, (int)j) && pair_less(s, (int)j, bs, bi)) { bs = s; bi = (int)j; }
            }
            block_min_pair(bs, bi, sh_s, sh_i);
            if (tid == 0 && bi != NO_IDX) { // lock-free minimum on the row's slot; the slot's pair is recomputed from its index
                int cur = __ldcg(aff_best + a);
                while (true) {
                    if (cur >= 0 && !pair_less(bs, bi, dist2(sXr, 1, X + cur, N, D), cur)) break;
                    const int prev = atomicCAS(aff_best + a, cur, bi);
                    if (prev == cur) break;
                    cur = prev;
                }
            }
        }
        if (b == 0 && tid == 0) ctl[CTL_AFF0 + ((t + 1) & 1)] = 0;
        if (!grid_barrier(ctl)) return;
        A_prev = A;
    }
}

// kept = the live indices in ascending order (one CTA)
__global__ void __launch_bounds__(1024) sparsify_compact_kernel(const int* __restrict__ alive, int64_t N, long long* __restrict__ kept,
    long long* __restrict__ n_kept)
{
    __shared__ int wsum[32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    long long base = 0;
    for (int64_t c0 = 0; c0 < N; c0 += 1024) {
        const int64_t idx = c0 + tid;
        const bool f = idx < N && alive[idx];
        const unsigned ballot = __ballot_sync(0xffffffffu, f);
        if (lane == 0) wsum[warp] = __popc(ballot);
        __syncthreads();
        int off = 0, total = 0;
        for (int w = 0; w < 32; ++w) {
            off += w < warp ? wsum[w] : 0;
            total += wsum[w];
        }
        if (f) kept[base + off + __popc(ballot & ((1u << lane) - 1u))] = idx;
        __syncthreads();
        base += total;
    }
    if (tid == 0) *n_kept = base;
}

struct DebugTiming {
    bool on = false;
    float ms[2] = {0.f, 0.f};
} g_timing;

} // namespace

extern "C" {
// tools/bench_sparsify.py: device-event times of the k-NN init and of the greedy loop of the next lb_sparsify* calls
int lb_debug_sparsify_timing(int on)
{
    g_timing.on = on != 0;
    return LB_OK;
}
int lb_debug_sparsify_last_ms(double* ms2)
{
    if (!ms2) return LB_ERR_ARG;
    ms2[0] = g_timing.ms[0];
    ms2[1] = g_timing.ms[1];
    return LB_OK;
}
}

// Sparsify N > max_points points (dX: row-major N x D on the device, 1 <= D <= LB_MAX_D, D <= max_points) on stream st.
// Writes dKept (n_kept ascending indices), dRemoved / dRemovedScore (N - n_kept entries, may be NULL) and *n_kept (host).
// Synchronises st.  LB_ERR_ARG for a non-finite coordinate, LB_ERR_TIMEOUT when a grid barrier wait timed out.
int lb_run_sparsify(const lb_gp* h, cudaStream_t st, int64_t N, int D, const double* dX, int64_t max_points, long long* dKept,
    int64_t* n_kept, long long* dRemoved, double* dRemovedScore, long long* launches)
{
    const int k = D;
    int dev = 0, nsm = 0, per_sm = 0;
    LB_CUDA(cudaGetDevice(&dev));
    LB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev));
    LB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sparsify_greedy_kernel, LOOP_THREADS, 0));
    if (per_sm < 1) return LB_ERR_UNSUPPORTED;
    const int G = nsm;
    double *Xs = nullptr, *nbr_s = nullptr, *score = nullptr, *part_s = nullptr, *rs = nullptr;
    int *nbr_j = nullptr, *alive = nullptr, *aff = nullptr, *aff_best = nullptr, *part_i = nullptr;
    unsigned* ctl = nullptr;
    long long *cnt = nullptr, *rm = nullptr;
    int rc = LB_OK;
    auto release = [&]() {
        cudaStreamSynchronize(st);
        void* all[] = {Xs, nbr_s, score, part_s, nbr_j, alive, aff, aff_best, part_i, ctl, cnt, dRemoved ? nullptr : rm,
            dRemovedScore ? nullptr : rs};
        for (void* q : all) lb_pool_free(q);
    };
#define SP_ALLOC(ptr, bytes)                                 \
    if ((rc = lb_dalloc(h, &(ptr), (bytes)))) { release(); return rc; }
    SP_ALLOC(Xs, sizeof(double) * D * N);
    SP_ALLOC(nbr_s, sizeof(double) * k * N);
    SP_ALLOC(nbr_j, sizeof(int) * k * N);
    SP_ALLOC(score, sizeof(double) * N);
    SP_ALLOC(alive, sizeof(int) * N);
    SP_ALLOC(aff, sizeof(int) * N);
    SP_ALLOC(aff_best, sizeof(int) * N);
    SP_ALLOC(part_s, sizeof(double) * G);
    SP_ALLOC(part_i, sizeof(int) * G);
    SP_ALLOC(ctl, sizeof(unsigned) * CTL_WORDS);
    SP_ALLOC(cnt, sizeof(long long) * 2); // n_removed, n_kept
    rm = dRemoved;
    rs = dRemovedScore;
    if (!rm) SP_ALLOC(rm, sizeof(long long) * N);
    if (!rs) SP_ALLOC(rs, sizeof(double) * N);
#undef SP_ALLOC
    auto fail = [&](cudaError_t e, int line) {
        lb_set_last_cuda_error(e, __FILE__, line);
        release();
        return LB_ERR_CUDA;
    };
    cudaError_t e;
    if ((e = cudaMemsetAsync(ctl, 0, sizeof(unsigned) * CTL_WORDS, st)) != cudaSuccess) return fail(e, __LINE__);
    if ((e = cudaMemsetAsync(cnt, 0, sizeof(long long) * 2, st)) != cudaSuccess) return fail(e, __LINE__);
    cudaEvent_t ev[3] = {};
    if (g_timing.on)
        for (cudaEvent_t& x : ev) cudaEventCreate(&x);
    sparsify_soa_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(dX, N, D, Xs);
    if (ev[0]) cudaEventRecord(ev[0], st);
    const size_t init_smem = sizeof(double) * 2 * D * INIT_THREADS;
    static LbOncePerDevice attr_once;
    if (attr_once.need() &&
        (e = cudaFuncSetAttribute(sparsify_knn_init_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
             (int)(sizeof(double) * 2 * LB_MAX_D * INIT_THREADS))) != cudaSuccess)
        return fail(e, __LINE__);
    sparsify_knn_init_kernel<<<(unsigned)((N + INIT_THREADS - 1) / INIT_THREADS), INIT_THREADS, init_smem, st>>>(Xs, N, D, k, nbr_s,
        nbr_j, score, alive, ctl);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail(e, __LINE__);
    if (ev[1]) cudaEventRecord(ev[1], st);
    const double* cXs = Xs;
    int64_t cN = N, cmax = max_points;
    int cD = D, ck = k;
    void* args[] = {(void*)&cXs, &cN, &cD, &ck, &cmax, &nbr_s, &nbr_j, &score, &alive, &aff, &aff_best, &part_s, &part_i, &ctl, &rm, &rs,
        &cnt};
    if ((e = cudaLaunchCooperativeKernel((const void*)sparsify_greedy_kernel, dim3(G), dim3(LOOP_THREADS), args, 0, st)) != cudaSuccess)
        return fail(e, __LINE__);
    if (ev[2]) cudaEventRecord(ev[2], st);
    sparsify_compact_kernel<<<1, 1024, 0, st>>>(alive, N, dKept, cnt + 1);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail(e, __LINE__);
    *launches += 4;
    long long hc[2] = {0, 0};
    int herr = 0;
    if ((e = cudaMemcpyAsync(hc, cnt, sizeof(hc), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return fail(e, __LINE__);
    if ((e = cudaMemcpyAsync(&herr, ctl + CTL_ERR, sizeof(int), cudaMemcpyDeviceToHost, st)) != cudaSuccess) return fail(e, __LINE__);
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return fail(e, __LINE__);
    if (ev[0]) {
        cudaEventElapsedTime(&g_timing.ms[0], ev[0], ev[1]);
        cudaEventElapsedTime(&g_timing.ms[1], ev[1], ev[2]);
        for (cudaEvent_t x : ev) cudaEventDestroy(x);
    }
    release();
    if (herr & SP_ERR_NONFINITE) return LB_ERR_ARG;
    if (herr & SP_ERR_TIMEOUT) return LB_ERR_TIMEOUT;
    *n_kept = hc[1];
    return hc[0] + hc[1] == N ? LB_OK : LB_ERR_STATE;
}
