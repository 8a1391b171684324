// limbo_b200/csrc/abi.cu — extern "C" boundary (include/limbo_b200.h) and the
// host-side orchestration of the device pipeline.  No torch types, no CPU
// fallback: every numerical result below comes from the CUDA kernels in this
// directory.
#include "../../include/limbo_b200.h"
#include "common.cuh"
#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <cstdio>
#include <mutex>
#include <new>
#include <string>

static thread_local std::string g_last_cuda_error;
void lb_set_last_cuda_error(cudaError_t e, const char* file, int line)
{
    char buf[512];
    snprintf(buf, sizeof(buf), "%s (%s) at %s:%d", cudaGetErrorName(e), cudaGetErrorString(e), file, line);
    g_last_cuda_error = buf;
    cudaGetLastError(); // clear sticky-less errors
}

#include <vector>
struct Profiler {
    struct Rec { cudaEvent_t a, b; int cls; };
    std::vector<Rec> recs;
    std::vector<cudaEvent_t> pool;
    cudaEvent_t cur[LB_PC_COUNT] = {};
    double ms[LB_PC_COUNT] = {};
    long long n[LB_PC_COUNT] = {};
    std::mutex mu;
    cudaEvent_t get()
    {
        if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
        cudaEvent_t e; cudaEventCreate(&e); return e;
    }
};
void lb_prof_begin(const lb_gp* h, cudaStream_t st, int cls)
{
    Profiler* p = (Profiler*)h->prof;
    std::lock_guard<std::mutex> lk(p->mu);
    cudaEvent_t e = p->get();
    cudaEventRecord(e, st);
    p->cur[cls] = e;
}
void lb_prof_end(const lb_gp* h, cudaStream_t st, int cls)
{
    Profiler* p = (Profiler*)h->prof;
    std::lock_guard<std::mutex> lk(p->mu);
    cudaEvent_t e = p->get();
    cudaEventRecord(e, st);
    p->recs.push_back({p->cur[cls], e, cls});
}

namespace {

struct QueryWs { // per-handle query workspace (guarded by qmutex)
    DevBuf<double> dQraw;  // M x D row-major staging
    DevBuf<double> dQs;    // D x Mp
    DevBuf<double> dV;     // Np x Mc
    DevBuf<double> dMu;    // M x P
    DevBuf<double> dS2;    // M
    ArgmaxWs am;           // acquisition values (M), host means uploaded (M), argmax records
    DevBuf<double> dCols;  // lb_acq_argmax_cols: the q x 2 acquisition parameters, then the q mean constants
    DevBuf<double> dFront; // lb_ehvi_argmax: the front sorted by f[0] (k x 2); lb_ehvi3d_argmax: ehvi.cu's Front3 (9 k)
    DevBuf<double> dEhvi3; // lb_ehvi3d_argmax: the front pass's planes and the partial sums (lb_ehvi3d_ws_doubles; 271 MB at k = 256)
    DevBuf<double> dGrad;  // two-model gradients (lb_eci_grad, lb_ehvi_grad): grad mu (M x D), then grad sigma^2 (M x D)
    DevBuf<float> dKt;     // TF32 path: K*^T chunk (Mc x Np fp32)
    DevBuf<float> dNorm2;
    DevBuf<double> dBias;  // reduced-precision path: rounding-bias weight per candidate
    DevBuf<int> dErr;
};

struct Extra {
    std::mutex qmutex;
    QueryWs ws;
    DevBuf<double> dMisc; // small scalars (loglik outputs, grad)
    cudaStream_t own = nullptr; // the handle's own stream (h->stream may point at a caller's stream)
    double lambda_host[LB_MAX_D * LB_MAX_LAMBDA] = {}; // host mirror of dLambda (lb_set_kernel compares against it)
    long long n_append = 0; // incremental updates actually taken (tests)
    double* hPoint = nullptr;  // pinned, mapped host buffer for the one-point query (mu[P], sigma^2)
    double* dPoint = nullptr;  // its device alias
    int point_cap = 0;
    cudaEvent_t ev_pair[2] = {}; // pair_locked's fork / join events, created on first use (the events of h->ev belong to the fit)
};

} // namespace

// The Extra block is stored behind the public struct.
struct lb_gp_full : lb_gp {
    Extra ex;
};
static inline lb_gp_full* full(const lb_gp* h) { return static_cast<lb_gp_full*>(const_cast<lb_gp*>(h)); }
static inline int n_outputs(const lb_gp* h) { return h->P > 0 ? h->P : 1; } // columns of mu (a handle without observations: 1)

namespace {

// handle workspaces grow with 256 bytes of slack
template <typename T>
int ensure(const lb_gp* h, DevBuf<T>& b, size_t bytes)
{
    return b.reserve(h, bytes, 256);
}

// Make *p private to h before h writes it (copy-on-write for buffers lb_clone shares).  preserve = keep the contents;
// otherwise the caller overwrites the whole buffer and the copy is skipped.  A missing buffer is allocated.
template <typename T>
int make_unique(lb_gp* h, T** p, size_t bytes, bool preserve, bool* fresh = nullptr)
{
    if (fresh) *fresh = false;
    if (*p && !lb_pool_shared(*p)) return LB_OK;
    T* n = nullptr;
    LB_ALLOC(h, n, bytes);
    if (fresh) *fresh = true;
    if (*p) {
        if (preserve) {
            LB_CUDA(cudaMemcpyAsync(n, *p, bytes, cudaMemcpyDeviceToDevice, h->stream));
            LB_CUDA(cudaStreamSynchronize(h->stream)); // the other holder may write the buffer once it is its sole owner
        }
        lb_pool_free(*p);
    }
    *p = n;
    return LB_OK;
}

// row-major (n x D) -> dimension-major (D x np) with optional per-dimension scale, zero padded
__global__ void pack_soa_kernel(const double* __restrict__ src, int64_t n, int D, double* __restrict__ dst, int64_t np,
    KernParams kp, int scaled)
{
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int d = blockIdx.y;
    if (i >= np) return;
    // D = row length of src; grid.y = D (raw copy) or kp.D (staged for the kernel: x/ell and the Lambda projections)
    double v = 0.0;
    if (i < n) v = scaled ? lb_staged_coord(kp, d, [&](int r) { return src[i * D + r]; }) : src[i * D + d];
    dst[(int64_t)d * np + i] = v;
}

__global__ void pad_cols_kernel(const double* __restrict__ src, int64_t n, int P, double* __restrict__ dst, int64_t np)
{
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int p = blockIdx.y;
    if (i >= np) return;
    dst[(int64_t)p * np + i] = (i < n) ? src[(int64_t)p * n + i] : 0.0;
}

__global__ void fill_kernel(double* __restrict__ p, int64_t n, double v)
{
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// identity on the padding region rows/cols [n0, np)
__global__ void identity_pad_kernel(double* __restrict__ A, int64_t np, int64_t n0)
{
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t tot = np * np;
    for (; idx < tot; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx % np, c = idx / np;
        if (r >= n0 || c >= n0) A[idx] = (r == c) ? 1.0 : 0.0;
    }
}

__global__ void identity_blocks_kernel(double* __restrict__ invD, int b0, int b1)
{
    int b = b0 + blockIdx.x;
    if (b >= b1) return;
    double* p = invD + (int64_t)b * LB_TILE * LB_TILE;
    for (int idx = threadIdx.x; idx < LB_TILE * LB_TILE; idx += blockDim.x) p[idx] = ((idx & 127) == (idx >> 7)) ? 1.0 : 0.0;
}

// copy the N x N leading block of a column-major Np matrix, zeroing the strict upper part if asked
__global__ void extract_kernel(const double* __restrict__ A, int64_t np, int64_t n, double* __restrict__ dst, int lower_only)
{
    int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t tot = n * n;
    for (; idx < tot; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx % n, c = idx / n;
        double v = A[r + c * np];
        if (lower_only && r < c) v = 0.0;
        dst[idx] = v;
    }
}

// k(x_i, x_new) for i < n (no noise), zero beyond: kernel.hpp:81-84 with i != j
__global__ void krow_kernel(const double* __restrict__ Xs, int64_t np, int64_t n, int64_t inew, KernParams kp,
    double* __restrict__ out)
{
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= np) return;
    double z = 0.0;
    for (int d = 0; d < kp.D; ++d) {
        double q = Xs[(int64_t)d * np + i] - Xs[(int64_t)d * np + inew];
        z = fma(q, q, z);
    }
    out[i] = (i < n) ? lb_kernel_from_z(kp.id, z, kp) : 0.0;
}

// finish the incremental row (gp.hpp:591-597): L[n, 0:n] = l^T ; L[n,n] = sqrt(k_nn - l.l)
__global__ void append_row_kernel(double* __restrict__ L, int64_t np, int64_t n, const double* __restrict__ lvec, double knn,
    int* __restrict__ info)
{
    __shared__ double red[8];
    double s = 0.0;
    for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
        double v = lvec[j];
        L[n + j * np] = v;
        s = fma(v, v, s);
    }
    s = lb_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += red[w];
        double d = knn - t;
        if (!(d > 0.0)) atomicCAS(info, 0, (int)(n + 1));
        L[n + n * np] = sqrt(d);
    }
}

// byte sizes of the six buffers lb_clone shares, for a model of padded order Np (invD: Np / LB_TILE blocks of LB_TILE x LB_TILE)
struct SharedBytes { size_t X, Xs, Y, L, InvD, Alpha; };
SharedBytes shared_bytes(int64_t Np, int D, int P)
{
    const size_t row = sizeof(double) * Np;
    return {row * D, row * (D + LB_MAX_LAMBDA), row * P, row * Np, row * LB_TILE, row * P};
}
SharedBytes shared_bytes(const lb_gp* h) { return shared_bytes(h->Np, h->D, h->P); }

// callers synchronise the handle's stream first
void free_model(lb_gp* h)
{
    void* shared[] = {h->dX, h->dXs, h->dY, h->dL, h->dInvD, h->dAlpha};
    for (void* p : shared) lb_pool_free(p); // buffers lb_clone shares only lose this handle's reference
    h->dX = h->dXs = h->dY = h->dL = h->dInvD = h->dAlpha = nullptr;
    // the private buffers sized by Np
    h->dLinv.release(); h->dKinv.release(); h->dFlags.release(); h->dLinv32.release(); h->dWork.release(); h->dLinvW.release();
    h->dTrsvX.release();
    h->linv32_valid = false;
    h->Np = 0;
}

// What every (re)factorisation starts with.  Private Xs / L / invD / alpha: allocated when missing, replaced without a copy when
// still shared with a clone (every byte is rewritten by the fit); then the samples staged for the kernel in Xs.
int stage_fit(lb_gp* h)
{
    const SharedBytes sz = shared_bytes(h);
    int rc;
    bool fresh = false;
    if ((rc = make_unique(h, &h->dXs, sz.Xs, false))) return rc;
    if ((rc = make_unique(h, &h->dL, sz.L, false))) return rc;
    if ((rc = make_unique(h, &h->dAlpha, sz.Alpha, false))) return rc;
    if ((rc = make_unique(h, &h->dInvD, sz.InvD, false, &fresh))) return rc;
    if (fresh) // the panel kernels only write the lower part of every block; consumers read whole blocks
        LB_CUDA(cudaMemsetAsync(h->dInvD, 0, sz.InvD, h->stream));
    return lb_launch_scale_x(h);
}

int check_info(lb_gp* h)
{
    int info[2] = {0, 0};
    LB_CUDA(cudaMemcpyAsync(info, h->dInfo.get(), sizeof(info), cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    if (info[1]) return LB_ERR_TIMEOUT;
    if (info[0] > 0) return info[0];
    return LB_OK;
}

// lb_fit without the final host sync / info read
int fit_enqueue(lb_gp* h)
{
    int rc;
    if ((rc = stage_fit(h))) return rc;
    if ((rc = lb_launch_kbuild(h, h->dL))) return rc;
    if ((rc = lb_launch_potrf(h))) return rc;
    h->fitted = true;
    lb_factor_changed(h);
    return lb_launch_solve_alpha(h);
}

// The M candidates Xq (row-major M x D) on the device: Xq itself when dev, otherwise a copy in h's dQraw, uploaded on h->stream.
int candidates_on_device(lb_gp_full* h, const double* Xq, int64_t M, bool dev, const double** out)
{
    *out = Xq;
    if (dev) return LB_OK;
    QueryWs& w = h->ex.ws;
    int rc = ensure(h, w.dQraw, sizeof(double) * M * h->D);
    if (rc) return rc;
    LB_CUDA(cudaMemcpyAsync(w.dQraw.get(), Xq, sizeof(double) * M * h->D, cudaMemcpyHostToDevice, h->stream));
    *out = w.dQraw.get();
    return LB_OK;
}

// The candidate-chunk loop of every query path: sizes h's dQs for De x Mc and dV for the path's v_doubles of scratch, and per chunk of
// at most Mc candidates stages it for the kernel in dQs (De x mcp, mcp = mc rounded up to `granule`, zero padded) and calls body(m0, mc, mcp).
template <typename Body>
int for_each_chunk(lb_gp_full* h, const double* dQraw, int64_t M, int64_t Mc, int64_t granule, size_t v_doubles, Body&& body)
{
    DevBuf<double>& dQs = h->ex.ws.dQs;
    const int D = h->D, De = h->kp.D; // raw / staged input dimension
    int rc;
    if ((rc = ensure(h, dQs, sizeof(double) * De * Mc)) || (rc = ensure(h, h->ex.ws.dV, sizeof(double) * v_doubles))) return rc;
    for (int64_t m0 = 0; m0 < M; m0 += Mc) {
        const int64_t mc = std::min(Mc, M - m0);
        const int64_t mcp = (mc + granule - 1) / granule * granule;
        dim3 g1((unsigned)((mcp + 255) / 256), (unsigned)De);
        pack_soa_kernel<<<g1, 256, 0, h->stream>>>(dQraw + m0 * D, mc, D, dQs.get(), mcp, h->kp, 1);
        h->launches++;
        if ((rc = body(m0, mc, mcp))) return rc;
    }
    return LB_OK;
}

// The host ends of one call on one stream.  Host mode: in() gives a device copy of a host array, out() a device temporary whose
// contents finish() copies back to the caller's array before it synchronises the stream once.  Device mode: the caller's pointers
// pass through, and finish() neither copies nor waits.  NULL stays NULL.
class Staging {
public:
    StreamTemps tmp;
    Staging(int device, cudaStream_t st, bool dev) : tmp(device, st), st_(st), dev_(dev) {}
    template <typename T>
    int in(const T* src, size_t n, const T** out)
    {
        *out = src;
        if (!src || dev_) return LB_OK;
        T* p = nullptr;
        int rc = tmp.alloc(sizeof(T) * n, &p);
        if (rc) return rc;
        LB_CUDA(cudaMemcpyAsync(p, src, sizeof(T) * n, cudaMemcpyHostToDevice, st_));
        *out = p;
        return LB_OK;
    }
    template <typename T>
    int out(T* dst, size_t n, T** out)
    {
        *out = dst;
        if (!dst || dev_) return LB_OK;
        int rc = tmp.alloc(sizeof(T) * n, out);
        if (rc) return rc;
        back_.push_back({dst, *out, sizeof(T) * n});
        return LB_OK;
    }
    int finish()
    {
        if (dev_) return LB_OK;
        for (const Back& b : back_) LB_CUDA(cudaMemcpyAsync(b.dst, b.src, b.bytes, cudaMemcpyDeviceToHost, st_));
        LB_CUDA(cudaStreamSynchronize(st_));
        return LB_OK;
    }

private:
    struct Back { void* dst; const void* src; size_t bytes; };
    cudaStream_t st_;
    bool dev_;
    std::vector<Back> back_;
};

// false for a non-finite coordinate of the M x D host candidates; device candidates are not read
bool coordinates_finite(const double* Xq, int64_t M, int D, bool dev)
{
    if (!dev)
        for (int64_t i = 0; i < M * D; ++i)
            if (!std::isfinite(Xq[i])) return false;
    return true;
}

// n zeros into dst (NULL: nothing), on st when dst is a device array
template <typename T>
int zero_fill(T* dst, int64_t n, bool dev, cudaStream_t st)
{
    if (!dst) return LB_OK;
    if (dev) LB_CUDA(cudaMemsetAsync(dst, 0, sizeof(T) * n, st));
    else std::fill(dst, dst + n, T(0));
    return LB_OK;
}

// The layout of n_hparams log-hyper-parameters of kernel kernel_id (0 to 3) over Draw inputs: the number of SE-ARD Lambda columns
// (0 for the other kernels), or LB_ERR_ARG for a count that fits no layout, LB_ERR_UNSUPPORTED beyond LB_MAX_LAMBDA / LB_MAX_D.
int hparam_klam(int kernel_id, int Draw, int n_hparams)
{
    if (kernel_id != LB_K_SE_ARD) return n_hparams == 2 ? 0 : LB_ERR_ARG;
    const int rest = n_hparams - 1 - Draw; // [log ell (D), A columns (D each, k of them), log sigma_f]  squared_exp_ard.hpp:91,96-105
    if (rest < 0 || rest % Draw != 0) return LB_ERR_ARG;
    const int klam = rest / Draw;
    if (klam > LB_MAX_LAMBDA || Draw + klam > LB_MAX_D) return LB_ERR_UNSUPPORTED;
    return klam;
}

// The kernel state of the log-hyper-parameters p (layout from hparam_klam) and the noise, written over kp.  kp.lambda is left NULL:
// the Lambda columns, p[Draw ..] column-major, stay with the caller.  Every kernel build reads what this derives, so the single path
// (lb_set_kernel) and the batched likelihood (lb_lml_grad_batch) see the same K.
void kernel_state(KernParams& kp, int kernel_id, int Draw, int klam, const double* p, int n_hparams, double noise)
{
    kp.id = kernel_id;
    kp.Draw = Draw;
    kp.klam = klam;
    kp.D = Draw + klam;
    kp.lambda = nullptr;
    kp.noise = noise;
    if (kernel_id == LB_K_SE_ARD) {
        for (int d = 0; d < Draw; ++d) kp.inv_ell[d] = 1.0 / std::exp(p[d]);
        kp.sf2 = std::exp(2.0 * p[n_hparams - 1]);
        kp.l = 1.0;
    }
    else { // matern_five_halves.hpp:97-102 and siblings
        kp.l = std::exp(p[0]);
        kp.sf2 = std::exp(2.0 * p[1]);
    }
    kp.c1 = kp.c2 = 0.0;
    if (kernel_id == LB_K_MATERN52) { kp.c1 = std::sqrt(5.0) / kp.l; kp.c2 = 5.0 / (3.0 * (kp.l * kp.l)); }
    else if (kernel_id == LB_K_MATERN32) kp.c1 = std::sqrt(3.0) / kp.l;
    else if (kernel_id == LB_K_EXP) kp.c1 = 1.0 / (kp.l * kp.l);
}

} // namespace

int lb_ensure_scratch(lb_gp* h, size_t bytes)
{
    return ensure(h, h->dScratch, bytes);
}

extern "C" {
int lb_profile_enable(lb_gp* h, int on);

// Streams and events of destroyed handles are kept for the next lb_create on the same device: a likelihood
// evaluation clones and destroys one handle (kernel_lf_opt.hpp:79), and stream / event creation is not free either.
struct Shell { cudaStream_t own = nullptr, side = nullptr; cudaEvent_t ev[LB_NEV] = {}; };
static std::mutex g_shell_mu;
static std::vector<Shell> g_shells[64];

int lb_create(lb_gp** out, int device, int precision)
{
    if (!out) return LB_ERR_ARG;
    if (precision != LB_PREC_FP64 && precision != LB_PREC_TF32 && precision != LB_PREC_FP16 && precision != LB_PREC_FP16X3) return LB_ERR_UNSUPPORTED;
    int ndev = 0;
    LB_CUDA(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev || device >= 64) return LB_ERR_ARG;
    lb_gp_full* h = new (std::nothrow) lb_gp_full();
    if (!h) return LB_ERR_ALLOC;
    h->device = device;
    DeviceGuard guard(device);
    if (!guard.ok) { delete h; return LB_ERR_CUDA; }
    h->precision = precision;
    Shell sh;
    bool cached = false;
    {
        std::lock_guard<std::mutex> lk(g_shell_mu);
        if (!g_shells[device].empty()) { sh = g_shells[device].back(); g_shells[device].pop_back(); cached = true; }
    }
    if (!cached) {
        if (cudaStreamCreateWithFlags(&sh.own, cudaStreamNonBlocking) != cudaSuccess) {
            delete h;
            return LB_ERR_CUDA;
        }
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        if (cudaStreamCreateWithPriority(&sh.side, cudaStreamNonBlocking, hi) != cudaSuccess) sh.side = nullptr;
        for (int i = 0; i < LB_NEV; ++i) cudaEventCreateWithFlags(&sh.ev[i], cudaEventDisableTiming);
    }
    h->ex.own = sh.own;
    h->stream = sh.own;
    h->own_stream = true;
    h->side = sh.side;
    for (int i = 0; i < LB_NEV; ++i) h->ev[i] = sh.ev[i];
    if (h->dInfo.resize(h, 4 * sizeof(int)) || h->ex.dMisc.resize(h, (LB_MAX_HPARAMS + 16) * sizeof(double))) {
        lb_destroy(h);
        return LB_ERR_ALLOC;
    }
    cudaMemsetAsync(h->dInfo.get(), 0, 4 * sizeof(int), h->stream);
    h->kp.id = LB_K_SE_ARD;
    *out = h;
    return LB_OK;
}

int lb_destroy(lb_gp* hh)
{
    if (!hh) return LB_OK;
    lb_gp_full* h = full(hh);
    DeviceGuard guard(h->device);
    cudaStreamSynchronize(h->stream);
    if (h->ex.own && h->ex.own != h->stream) cudaStreamSynchronize(h->ex.own);
    if (h->side) cudaStreamSynchronize(h->side);
    lb_profile_enable(h, 0);
    free_model(h);
    h->ex.ws = QueryWs{}; // the remaining private buffers go back with the handle (delete h)
    if (h->ex.hPoint) cudaFreeHost(h->ex.hPoint);
    for (cudaEvent_t e : h->ex.ev_pair) if (e) cudaEventDestroy(e);
    for (cudaStream_t& s : h->group)
        if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); s = nullptr; }
    Shell sh;
    sh.own = h->ex.own; sh.side = h->side;
    for (int i = 0; i < LB_NEV; ++i) sh.ev[i] = h->ev[i];
    bool kept = false;
    if (sh.own && h->device >= 0 && h->device < 64) {
        std::lock_guard<std::mutex> lk(g_shell_mu);
        if (g_shells[h->device].size() < 64) { g_shells[h->device].push_back(sh); kept = true; }
    }
    if (!kept) {
        if (sh.own) cudaStreamDestroy(sh.own);
        if (sh.side) cudaStreamDestroy(sh.side);
        for (int i = 0; i < LB_NEV; ++i) if (sh.ev[i]) cudaEventDestroy(sh.ev[i]);
    }
    delete h;
    return LB_OK;
}

int lb_set_stream(lb_gp* h, void* s)
{
    if (!h) return LB_ERR_ARG;
    LB_DEVICE(h);
    lb_gp_full* f = full(h);
    LB_CUDA(cudaStreamSynchronize(f->stream));
    f->stream = s ? (cudaStream_t)s : f->ex.own;
    return LB_OK;
}

int lb_sync(lb_gp* h)
{
    if (!h) return LB_ERR_ARG;
    LB_DEVICE(h);
    LB_CUDA(cudaStreamSynchronize(h->stream));
    // device-side wait timeouts of the reduced-precision scoring path, for callers of the *_dev entry points (which
    // return before the kernels have run)
    lb_gp_full* f = full(h);
    if (f->ex.ws.dErr) {
        int herr = 0;
        LB_CUDA(cudaMemcpy(&herr, f->ex.ws.dErr.get(), sizeof(int), cudaMemcpyDeviceToHost));
        if (herr) {
            LB_CUDA(cudaMemset(f->ex.ws.dErr.get(), 0, sizeof(int)));
            return LB_ERR_TIMEOUT;
        }
    }
    return LB_OK;
}

long long lb_launch_count(const lb_gp* h) { return h ? h->launches : 0; }
int64_t lb_nb_samples(const lb_gp* h) { return h ? h->N : 0; }

static int set_data_common(lb_gp* h, int64_t N, int D, int P, const double* X, const double* Y, bool dev)
{
    if (!h || N < 0 || D < 1 || D > LB_MAX_D || P < 1) return LB_ERR_ARG;
    if (N > 0 && (!X || !Y)) return LB_ERR_ARG;
    LB_DEVICE(h);
    const int64_t Np = std::max<int64_t>(LB_TILE, (N + LB_TILE - 1) / LB_TILE * LB_TILE);
    const bool reshape = Np != h->Np || D != h->D || P != h->P;
    if (reshape) {
        LB_CUDA(cudaStreamSynchronize(h->stream));
        free_model(h);
    }
    // X and Y, rewritten in place unless a clone still reads them; Xs, L, invD, alpha: stage_fit (a clone that refits never needs its source's)
    const SharedBytes sz = shared_bytes(Np, D, P);
    int rc;
    if ((rc = make_unique(h, &h->dX, sz.X, false)) || (rc = make_unique(h, &h->dY, sz.Y, false))) return rc;
    if (reshape && (rc = h->dFlags.resize(h, sizeof(int) * (Np / LB_TILE + 8)))) return rc;
    h->Np = Np;
    if (D != h->D) h->kp.klam = 0; // the Lambda matrix belongs to the previous input dimension
    h->N = N; h->D = D; h->P = P;
    h->kp.Draw = D;
    h->kp.D = D + h->kp.klam;
    h->fitted = false;
    lb_factor_changed(h);
    const double* dXr = X;
    const double* dYr = Y;
    if (!dev && N > 0) {
        int rc = lb_ensure_scratch(h, sizeof(double) * (size_t)N * (D + P));
        if (rc) return rc;
        LB_CUDA(cudaMemcpyAsync(h->dScratch.get(), X, sizeof(double) * N * D, cudaMemcpyHostToDevice, h->stream));
        LB_CUDA(cudaMemcpyAsync(h->dScratch.get() + N * D, Y, sizeof(double) * N * P, cudaMemcpyHostToDevice, h->stream));
        dXr = h->dScratch.get();
        dYr = h->dScratch.get() + N * D;
    }
    dim3 g1((unsigned)((Np + 255) / 256), (unsigned)D), g2((unsigned)((Np + 255) / 256), (unsigned)P);
    pack_soa_kernel<<<g1, 256, 0, h->stream>>>(dXr, N, D, h->dX, Np, h->kp, 0);
    pad_cols_kernel<<<g2, 256, 0, h->stream>>>(dYr, N, P, h->dY, Np);
    h->launches += 2;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Samples only (multi-GPU Cholesky, potrf.cu lb_dchol_*): stages X without allocating the N x N factor storage of
// this handle; the handle can then only serve lb_set_kernel and the lb_dchol_* calls.
int lb_dchol_set_points(lb_gp* h, int64_t N, int D, const double* X)
{
    if (!h || N <= 0 || D < 1 || D > LB_MAX_D || !X) return LB_ERR_ARG;
    LB_DEVICE(h);
    LB_CUDA(cudaStreamSynchronize(h->stream));
    free_model(h);
    const int64_t Np = (N + LB_TILE - 1) / LB_TILE * LB_TILE;
    LB_ALLOC(h, h->dX, shared_bytes(Np, D, 0).X);
    LB_ALLOC(h, h->dXs, shared_bytes(Np, D, 0).Xs);
    h->Np = Np;
    if (D != h->D) h->kp.klam = 0;
    h->N = N; h->D = D; h->P = 0;
    h->kp.Draw = D;
    h->kp.D = D + h->kp.klam;
    h->fitted = false;
    lb_factor_changed(h);
    int rc = lb_ensure_scratch(h, sizeof(double) * (size_t)N * D);
    if (rc) return rc;
    LB_CUDA(cudaMemcpyAsync(h->dScratch.get(), X, sizeof(double) * N * D, cudaMemcpyHostToDevice, h->stream));
    dim3 g1((unsigned)((Np + 255) / 256), (unsigned)D);
    pack_soa_kernel<<<g1, 256, 0, h->stream>>>(h->dScratch.get(), N, D, h->dX, Np, h->kp, 0);
    h->launches++;
    LB_CUDA(cudaStreamSynchronize(h->stream));
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_set_data(lb_gp* h, int64_t N, int D, int P, const double* X, const double* Y)
{
    return set_data_common(h, N, D, P, X, Y, false);
}
int lb_set_data_dev(lb_gp* h, int64_t N, int D, int P, const double* dX, const double* dY)
{
    return set_data_common(h, N, D, P, dX, dY, true);
}

int lb_set_kernel(lb_gp* h, int kernel_id, const double* p, int n_hparams, double noise)
{
    if (!h || !p) return LB_ERR_ARG;
    if (kernel_id < 0 || kernel_id > 3) return LB_ERR_UNSUPPORTED;
    if (h->D <= 0) return LB_ERR_STATE; // need the input dimension first (lb_set_data)
    const int klam = hparam_klam(kernel_id, h->D, n_hparams);
    if (klam < 0) return klam;
    LB_DEVICE(h);
    bool lambda_same = true;
    const KernParams old = h->kp;
    const bool was_set = h->kernel_set;
    const int old_nh = h->n_hparams;
    KernParams& kp = h->kp;
    kernel_state(kp, kernel_id, h->D, klam, p, n_hparams, noise);
    if (klam > 0) { // _A(i, j) = p((j + 1) * D + i): already column-major
        int rc = h->dLambda.reserve(h, sizeof(double) * LB_MAX_D * LB_MAX_LAMBDA);
        if (rc) return rc;
        double* lh = full(h)->ex.lambda_host;
        lambda_same = (old.klam == klam) && std::memcmp(lh, p + h->D, sizeof(double) * h->D * klam) == 0;
        std::memcpy(lh, p + h->D, sizeof(double) * h->D * klam);
        LB_CUDA(cudaMemcpyAsync(h->dLambda.get(), p + h->D, sizeof(double) * h->D * klam, cudaMemcpyHostToDevice, h->stream));
        LB_CUDA(cudaStreamSynchronize(h->stream));
        kp.lambda = h->dLambda.get();
    }
    h->n_hparams = n_hparams;
    h->kernel_set = true;
    // The same functor state again (add_sample pushes the kernel before every lb_append, gp.hpp:126-152 never touches
    // it): the factor stays valid.
    bool same = was_set && old_nh == n_hparams && klam == old.klam && lambda_same && old.id == kp.id && old.D == kp.D && old.Draw == kp.Draw
        && old.sf2 == kp.sf2 && old.l == kp.l && old.noise == kp.noise && old.c1 == kp.c1 && old.c2 == kp.c2;
    if (same && kernel_id == LB_K_SE_ARD)
        for (int d = 0; d < h->D; ++d) same = same && (old.inv_ell[d] == kp.inv_ell[d]);
    if (!same) {
        h->fitted = false;
        lb_factor_changed(h);
    }
    return LB_OK;
}

int lb_fit(lb_gp* h)
{
    if (!h) return LB_ERR_ARG;
    if (!h->kernel_set || h->Np == 0 || !h->dX) return LB_ERR_STATE;
    LB_DEVICE(h);
    if (h->N == 0) return LB_ERR_STATE; // gp.hpp:90 assert(samples.size() != 0)
    int rc = fit_enqueue(h);
    return rc ? rc : check_info(h);
}

int lb_fit_async(lb_gp* h) // same as lb_fit without the final host sync / info read (bench "value" leg)
{
    if (!h) return LB_ERR_ARG;
    if (!h->kernel_set || h->Np == 0 || h->N == 0 || !h->dX) return LB_ERR_STATE;
    LB_DEVICE(h);
    return fit_enqueue(h);
}

int lb_check_info(lb_gp* h)
{
    if (!h) return LB_ERR_ARG;
    LB_DEVICE(h);
    return check_info(h);
}
int lb_debug_potf2(lb_gp* h, int k, long long* out, int n)
{
    if (!h) return LB_ERR_ARG;
    LB_DEVICE(h);
    return lb_debug_potf2_clocks(h, k, out, n);
}
// testing hook: how many times lb_append took the incremental path on this handle
long long lb_debug_append_count(const lb_gp* h) { return h ? full(h)->ex.n_append : 0; }
// testing hook: force the multi-launch (unfused) query path
int lb_debug_force_unfused_query(lb_gp* h, int on) { if (!h) return LB_ERR_ARG; h->force_unfused = on != 0; return LB_OK; }

// stage timers for bench.py: run only one stage (inputs must already be in place)
int lb_stage_kbuild(lb_gp* h)
{
    if (!h || !h->kernel_set || h->N == 0) return LB_ERR_STATE;
    LB_DEVICE(h);
    int rc = stage_fit(h);
    if (rc) return rc;
    h->fitted = false;
    return lb_launch_kbuild(h, h->dL);
}
int lb_stage_potrf(lb_gp* h)
{
    if (!h || h->N == 0 || !h->dL) return LB_ERR_STATE;
    LB_DEVICE(h);
    int rc = lb_launch_potrf(h);
    if (!rc) h->fitted = true;
    return rc;
}
int lb_stage_alpha(lb_gp* h)
{
    if (!h || !h->fitted) return LB_ERR_STATE;
    LB_DEVICE(h);
    return lb_launch_solve_alpha(h);
}

// GP::load(archive, recompute = false) (gp.hpp:505-509): take a stored factor and alpha instead of refactorising.
// Data and kernel must already be set (lb_set_data / lb_set_kernel); the diagonal-block inverses are rebuilt.
int lb_load_factor(lb_gp* h, const double* L_colmajor, const double* alpha_colmajor)
{
    if (!h || !L_colmajor || !alpha_colmajor) return LB_ERR_ARG;
    if (!h->kernel_set || h->N == 0 || h->Np == 0) return LB_ERR_STATE;
    LB_DEVICE(h);
    const int64_t N = h->N, Np = h->Np;
    const int T = (int)(Np / LB_TILE);
    int rc;
    if ((rc = stage_fit(h))) return rc;
    LB_CUDA(cudaMemsetAsync(h->dL, 0, sizeof(double) * Np * Np, h->stream));
    LB_CUDA(cudaMemcpy2DAsync(h->dL, Np * 8, L_colmajor, N * 8, N * 8, N, cudaMemcpyHostToDevice, h->stream));
    identity_pad_kernel<<<1024, 256, 0, h->stream>>>(h->dL, Np, N);
    LB_CUDA(cudaMemsetAsync(h->dAlpha, 0, sizeof(double) * Np * h->P, h->stream));
    LB_CUDA(cudaMemcpy2DAsync(h->dAlpha, Np * 8, alpha_colmajor, N * 8, N * 8, h->P, cudaMemcpyHostToDevice, h->stream));
    LB_CUDA(cudaMemsetAsync(h->dInfo.get(), 0, 2 * sizeof(int), h->stream));
    h->launches++;
    for (int k = 0; k < T; ++k)
        if ((rc = lb_launch_potf2_block(h, k, 0))) return rc;
    h->fitted = true;
    lb_factor_changed(h);
    return check_info(h);
}

int lb_refit_alpha(lb_gp* h, const double* Y)
{
    if (!h || !Y) return LB_ERR_ARG;
    if (!h->fitted) return LB_ERR_STATE;
    LB_DEVICE(h);
    int rc = lb_ensure_scratch(h, sizeof(double) * (size_t)h->N * h->P);
    if (rc) return rc;
    if ((rc = make_unique(h, &h->dY, shared_bytes(h).Y, false))) return rc;
    if ((rc = make_unique(h, &h->dAlpha, shared_bytes(h).Alpha, false))) return rc;
    LB_CUDA(cudaMemcpyAsync(h->dScratch.get(), Y, sizeof(double) * h->N * h->P, cudaMemcpyHostToDevice, h->stream));
    dim3 g2((unsigned)((h->Np + 255) / 256), (unsigned)h->P);
    pad_cols_kernel<<<g2, 256, 0, h->stream>>>(h->dScratch.get(), h->N, h->P, h->dY, h->Np);
    h->launches++;
    if ((rc = lb_launch_solve_alpha(h))) return rc;
    return check_info(h);
}

int lb_append(lb_gp* h, const double* x, const double* Yall)
{
    if (!h || !x || !Yall) return LB_ERR_ARG;
    if (!h->kernel_set) return LB_ERR_STATE;
    LB_DEVICE(h);
    if (h->N == 0 || !h->fitted) return LB_ERR_STATE; // first sample goes through lb_set_data + lb_fit
    const int64_t n = h->N;
    const int D = h->D, P = h->P;
    if (n + 1 > h->Np) { // grow by one tile, keep the factor
        const int64_t oldNp = h->Np, newNp = oldNp + LB_TILE;
        const int64_t oldT = oldNp / LB_TILE, newT = newNp / LB_TILE;
        const SharedBytes sz = shared_bytes(newNp, D, P);
        double *nX, *nXs, *nY, *nA, *nL, *nI;
        LB_CUDA(cudaStreamSynchronize(h->stream));
        LB_ALLOC(h, nX, sz.X);
        LB_ALLOC(h, nXs, sz.Xs);
        LB_ALLOC(h, nY, sz.Y);
        LB_ALLOC(h, nA, sz.Alpha);
        LB_ALLOC(h, nL, sz.L);
        LB_ALLOC(h, nI, sz.InvD);
        int rc = h->dFlags.resize(h, sizeof(int) * (newT + 8));
        if (rc) return rc;
        LB_CUDA(cudaMemsetAsync(nX, 0, sz.X, h->stream));
        LB_CUDA(cudaMemsetAsync(nY, 0, sz.Y, h->stream));
        LB_CUDA(cudaMemcpy2DAsync(nX, newNp * 8, h->dX, oldNp * 8, oldNp * 8, D, cudaMemcpyDeviceToDevice, h->stream));
        LB_CUDA(cudaMemcpy2DAsync(nL, newNp * 8, h->dL, oldNp * 8, oldNp * 8, oldNp, cudaMemcpyDeviceToDevice, h->stream));
        LB_CUDA(cudaMemcpyAsync(nI, h->dInvD, shared_bytes(oldNp, D, P).InvD, cudaMemcpyDeviceToDevice, h->stream));
        identity_pad_kernel<<<1024, 256, 0, h->stream>>>(nL, newNp, oldNp);
        identity_blocks_kernel<<<(unsigned)(newT - oldT), 256, 0, h->stream>>>(nI, (int)oldT, (int)newT);
        h->launches += 2;
        LB_CUDA(cudaStreamSynchronize(h->stream));
        lb_pool_free(h->dX); lb_pool_free(h->dXs); lb_pool_free(h->dY); lb_pool_free(h->dAlpha); lb_pool_free(h->dL); lb_pool_free(h->dInvD);
        h->dX = nX; h->dXs = nXs; h->dY = nY; h->dAlpha = nA; h->dL = nL; h->dInvD = nI;
        h->dLinv.release(); h->dKinv.release();
        h->Np = newNp;
    }
    const int64_t Np = h->Np;
    int rc = lb_ensure_scratch(h, sizeof(double) * (size_t)((n + 1) * P + D + Np));
    if (rc) return rc;
    { // copy-on-write: a clone may still read these (the row update keeps the rest of X, L, invD)
        const SharedBytes sz = shared_bytes(h);
        if ((rc = make_unique(h, &h->dX, sz.X, true))) return rc;
        if ((rc = make_unique(h, &h->dL, sz.L, true))) return rc;
        if ((rc = make_unique(h, &h->dInvD, sz.InvD, true))) return rc;
        if ((rc = make_unique(h, &h->dY, sz.Y, false))) return rc;
        if ((rc = make_unique(h, &h->dXs, sz.Xs, false))) return rc;
        if ((rc = make_unique(h, &h->dAlpha, sz.Alpha, false))) return rc;
    }
    full(h)->ex.n_append++;
    double* dYs = h->dScratch.get();
    double* dx = dYs + (n + 1) * P;
    double* dk = dx + D;
    LB_CUDA(cudaMemcpyAsync(dYs, Yall, sizeof(double) * (n + 1) * P, cudaMemcpyHostToDevice, h->stream));
    LB_CUDA(cudaMemcpyAsync(dx, x, sizeof(double) * D, cudaMemcpyHostToDevice, h->stream));
    // X[:, n] = x  (strided D writes)
    LB_CUDA(cudaMemcpy2DAsync(h->dX + n, Np * 8, dx, 8, 8, D, cudaMemcpyDeviceToDevice, h->stream));
    h->N = n + 1;
    dim3 g2((unsigned)((Np + 255) / 256), (unsigned)P);
    pad_cols_kernel<<<g2, 256, 0, h->stream>>>(dYs, n + 1, P, h->dY, Np);
    h->launches++;
    if ((rc = lb_launch_scale_x(h))) return rc;
    // new kernel row (gp.hpp:583-586), forward solve against the existing factor (gp.hpp:591-594)
    krow_kernel<<<(unsigned)((Np + 255) / 256), 256, 0, h->stream>>>(h->dXs, Np, n, n, h->kp, dk);
    h->launches++;
    if ((rc = lb_launch_trsv(h, dk, 1, true))) return rc;
    const double knn = h->kp.sf2 + h->kp.noise + 1e-8; // kernel(x,x) with i == j, kernel.hpp:83
    append_row_kernel<<<1, 256, 0, h->stream>>>(h->dL, Np, n, dk, knn, h->dInfo.get());
    h->launches++;
    if ((rc = lb_launch_potf2_block(h, (int)(n / LB_TILE), 0))) return rc;
    lb_factor_changed(h);
    if ((rc = lb_launch_solve_alpha(h))) return rc;
    return check_info(h);
}

// Batches of at least this many candidates take the panel path.  The slab kernel keeps the
// one-point / small-batch latency, but its time does not shrink with the batch: every CTA streams all of L through L2 whatever
// its slab width, while the panel path scales with the number of 128-candidate column tiles.  Measured on an H100 SXM at a 400 W
// power limit, N = 16384, ms per batch of 32 / 64 / 128 / 256 / 512 candidates: slab path 86.1 for every size, panel path
// 5.7 / 5.7 / 5.7 / 5.8 / 6.1: at this N the panel path wins from the smallest batch.  The default of 256 is not re-tuned:
// batches at small N (the reference's own regime) have not been measured on H100, and below the threshold a batch is bit-identical
// to one-point queries (query_point_kernel runs the slab body).
static int64_t g_query_panel_min = 0; // 0: the default
static int64_t query_panel_min() { return g_query_panel_min > 0 ? g_query_panel_min : 256; }
// testing hook: batch size from which lb_query / lb_acq_argmax take the panel path (<= 0 restores the default)
extern "C" int lb_debug_set_query_panel_min(long long m)
{
    g_query_panel_min = m > 0 ? (int64_t)m : 0;
    return LB_OK;
}

// The path a batch of M candidates takes on h.  host_point: the call has the shape of the one-point kernel (the candidate and the
// results on the host, no acquisition); lb_query of one point then always takes that kernel, whatever the panel threshold.
enum QueryPath { QP_PRIOR, QP_POINT, QP_REDUCED, QP_PANEL, QP_SLAB, QP_MULTI };
static QueryPath query_path(const lb_gp* h, int64_t M, bool host_point = false)
{
    if (h->N == 0 || !h->fitted) return QP_PRIOR;
    if (h->precision != LB_PREC_FP64) return QP_REDUCED;
    if (h->force_unfused) return QP_MULTI;
    const bool fused = lb_query_fused_supported(h);
    if (host_point && M == 1 && fused) return QP_POINT;
    if (M >= query_panel_min()) return QP_PANEL;
    return fused ? QP_SLAB : QP_MULTI;
}

// Widest candidate chunk, a multiple of the tile, whose V (Np x Mc doubles) stays within `bytes`; no wider than the padded batch
static int64_t v_chunk(const lb_gp* h, int64_t M, int64_t bytes)
{
    const int64_t Mp = (M + LB_TILE - 1) / LB_TILE * LB_TILE;
    return std::min(Mp, std::max<int64_t>(LB_TILE, bytes / (8 * h->Np) / LB_TILE * LB_TILE));
}
// the panel path and the gradients: candidate chunks bounded so that V (Np x Mc) stays <= ~6 GiB
static int64_t panel_chunk(const lb_gp* h, int64_t M) { return v_chunk(h, M, (int64_t)6 << 30); }
// the multi-launch path: candidate chunks bounded so that V (Np x Mc) stays <= ~4 GiB
static int64_t multi_chunk(const lb_gp* h, int64_t M) { return v_chunk(h, M, (int64_t)4 << 30); }
// The reduced-precision path: candidate chunks of k x (SMs x 128 candidates), whole waves of the persistent wgmma GEMM (one
// 128-candidate tile per CTA per wave); K*^T chunk <= 4 GiB.
static int64_t reduced_chunk(const lb_gp* h, int64_t M, int sms)
{
    const int64_t CH = 2 * LB_TILE, wave = (int64_t)(sms / 2) * CH;
    const int64_t cap = std::max<int64_t>(CH, ((int64_t)4 << 30) / (4 * h->Np) / CH * CH);
    return std::min((M + CH - 1) / CH * CH, (cap >= wave) ? cap / wave * wave : cap);
}

// The fills of query_fill, one per path: h's dMu (M x P) and dS2 (M) from the row-major device candidates dQraw, on h->stream.
// The prior, gp.hpp:161-163: mu = mean(v) (added by the caller), sigma2 = k(v,v) + noise
static int fill_prior(lb_gp_full* h, int64_t M)
{
    LB_CUDA(cudaMemsetAsync(h->ex.ws.dMu.get(), 0, sizeof(double) * M * n_outputs(h), h->stream));
    fill_kernel<<<(unsigned)((M + 255) / 256), 256, 0, h->stream>>>(h->ex.ws.dS2.get(), M, h->kp.sf2 + h->kp.noise);
    h->launches++;
    return LB_OK;
}

// reduced-precision variance on wgmma (tf32_query.cu); mu is accumulated in fp64 from the fp64 kernel values
static int fill_reduced(lb_gp_full* h, int64_t M, const double* dQraw)
{
    QueryWs& w = h->ex.ws;
    cudaStream_t st = h->stream;
    const int P = n_outputs(h);
    int rc, sms = 132;
    if ((rc = lb_tf32_prepare(h))) return rc;
    LB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
    const int64_t Mc = reduced_chunk(h, M, sms);
    if ((rc = ensure(h, w.dKt, sizeof(float) * (size_t)Mc * h->Np))) return rc;
    if ((rc = ensure(h, w.dNorm2, sizeof(double) * (size_t)Mc))) return rc; // Mc floats (split mode: Mc doubles)
    if ((rc = ensure(h, w.dBias, sizeof(double) * Mc))) return rc;
    if ((rc = w.dErr.reserve(h, sizeof(int)))) return rc;
    LB_CUDA(cudaMemsetAsync(w.dErr.get(), 0, sizeof(int), st));
    const size_t partials = (size_t)(P + 1) * (h->Np / LB_TILE) * Mc; // dV: mean (+ bias) partials per training tile
    return for_each_chunk(h, dQraw, M, Mc, 2 * LB_TILE, partials, [&](int64_t m0, int64_t mc, int64_t mcp) {
        double* dBias = (h->precision == LB_PREC_FP16X3) ? nullptr : w.dBias.get(); // 22-bit operands: no rounding-bias term
        int rc = lb_launch_kstar_tf32(h, st, mc, w.dQs.get(), mcp, w.dKt.get(), w.dV.get(), w.dMu.get() + m0 * P, dBias, &h->launches);
        if (rc) return rc;
        return lb_launch_sigma_tf32(h, st, mc, mcp, w.dKt.get(), w.dNorm2.get(), w.dErr.get(), dBias, w.dS2.get() + m0, &h->launches);
    });
}

// large batches: blocked solve over 2048-row super-blocks on the GEMM core (query.cu, namespace panel)
static int fill_panel(lb_gp_full* h, int64_t M, const double* dQraw)
{
    QueryWs& w = h->ex.ws;
    const int64_t Mc = panel_chunk(h, M);
    return for_each_chunk(h, dQraw, M, Mc, LB_TILE, lb_query_panel_scratch_doubles(h, Mc), [&](int64_t m0, int64_t mc, int64_t mcp) {
        return lb_launch_query_panel(h, h->stream, mc, w.dQs.get(), mcp, w.dV.get(), w.dMu.get() + m0 * n_outputs(h), w.dS2.get() + m0,
            &h->launches);
    });
}

// fused persistent path: one CTA per candidate slab, private V scratch per CTA; the whole padded batch is one chunk
static int fill_slab(lb_gp_full* h, int64_t M, const double* dQraw)
{
    QueryWs& w = h->ex.ws;
    int sms = 0;
    LB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->device));
    const int grid = (int)std::min<int64_t>(sms, (M + 7) / 8);
    const int64_t Mp = (M + LB_TILE - 1) / LB_TILE * LB_TILE;
    return for_each_chunk(h, dQraw, M, Mp, LB_TILE, lb_query_fused_scratch_doubles(h, grid), [&](int64_t, int64_t mc, int64_t mcp) {
        return lb_launch_query_fused(h, h->stream, mc, w.dQs.get(), mcp, w.dV.get(), grid, w.dMu.get(), w.dS2.get(), &h->launches);
    });
}

// one launch per step of the solve (query.cu): the only path for D > DMAXF or P > PMAXF, and the tests' reference
static int fill_multi(lb_gp_full* h, int64_t M, const double* dQraw)
{
    QueryWs& w = h->ex.ws;
    const int64_t Mc = multi_chunk(h, M);
    return for_each_chunk(h, dQraw, M, Mc, LB_TILE, (size_t)h->Np * Mc, [&](int64_t m0, int64_t mc, int64_t mcp) {
        return lb_launch_query(h, h->stream, mc, w.dQs.get(), mcp, w.dV.get(), w.dMu.get() + m0 * n_outputs(h), w.dS2.get() + m0, &h->launches);
    });
}

// Fills h's query workspace, w.dMu.get() (M x P, k^T alpha) and w.dS2.get() (M), for M candidates on h->stream, on the path
// query_path chooses.  Xq is row-major M x D, a device pointer when xq_dev.  The caller holds h->ex.qmutex and has checked the
// handle's state.  A reduced-precision fill leaves its timeout flag in w.dErr (query_timed_out).
static int query_fill(lb_gp_full* h, int64_t M, const double* Xq, bool xq_dev)
{
    QueryWs& w = h->ex.ws;
    int rc;
    if ((rc = ensure(h, w.dMu, sizeof(double) * M * n_outputs(h)))) return rc;
    if ((rc = ensure(h, w.dS2, sizeof(double) * M))) return rc;
    const QueryPath path = query_path(h, M);
    if (path == QP_PRIOR) return h->N != 0 ? LB_ERR_STATE : fill_prior(h, M);
    const double* dQraw = nullptr;
    if ((rc = candidates_on_device(h, Xq, M, xq_dev, &dQraw))) return rc;
    switch (path) {
    case QP_REDUCED: return fill_reduced(h, M, dQraw);
    case QP_PANEL: return fill_panel(h, M, dQraw);
    case QP_SLAB: return fill_slab(h, M, dQraw);
    default: return fill_multi(h, M, dQraw);
    }
}

// A device copy of mean_at_q (M values) on h's stream, or mean_at_q itself when it already is a device pointer (or NULL)
static int mean_on_device(lb_gp_full* h, cudaStream_t st, const double* mean_at_q, int64_t M, bool dev, const double** out)
{
    *out = mean_at_q;
    if (!mean_at_q || dev) return LB_OK;
    DevBuf<double>& mean = h->ex.ws.am.mean;
    int rc = ensure(h, mean, sizeof(double) * M);
    if (rc) return rc;
    LB_CUDA(cudaMemcpyAsync(mean.get(), mean_at_q, sizeof(double) * M, cudaMemcpyHostToDevice, st));
    *out = mean.get();
    return LB_OK;
}

// LB_ERR_TIMEOUT when the last reduced-precision fill of h marked its results invalid (synchronises h->stream)
static int query_timed_out(lb_gp_full* h)
{
    if (h->precision == LB_PREC_FP64 || h->N == 0 || !h->ex.ws.dErr) return LB_OK; // N == 0: the prior, no flag written
    int herr = 0;
    LB_CUDA(cudaMemcpyAsync(&herr, h->ex.ws.dErr.get(), sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    return herr ? LB_ERR_TIMEOUT : LB_OK;
}

// The per-column acquisition of lb_acq_argmax_cols / lb_acq_cmaes_cols (query.cu: acq_cols_kernel) over the handle's P columns:
// acq_params holds P x 2 parameters, mean_at_q M x P means (or NULL), mean_const P constants, and best_val / best_idx P records.
// dParams: the parameters then the constants on the device (3 P doubles), or NULL to upload acq_params and mean_const (host) into
// the query workspace.  dInstCol (device, one column per CMA-ES instance of lam candidates): each candidate scored in its instance's
// column only, M values and one record.
struct AcqCols {
    const double* mean_const;
    const double* dParams;
    const int* dInstCol;
    int lam;
};

static int query_common(const lb_gp* hc, int64_t M, const double* Xq, bool xq_dev, double* mu_out, double* s2_out,
    bool out_dev, int acq_id, const double* acq_params, const double* mean_at_q, double mean_const, double* acq_out,
    double* best_val, int64_t* best_idx, bool with_acq, bool lock_held = false, const AcqCols* cols = nullptr)
{
    if (!hc || M < 0) return LB_ERR_ARG;
    if (M == 0) return LB_OK;
    if (!Xq) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    if (h->D <= 0 || !h->kernel_set) return LB_ERR_STATE;
    LB_DEVICE(h);
    std::unique_lock<std::mutex> lock(h->ex.qmutex, std::defer_lock); // lock_held: the caller holds it (lb_acq_cmaes)
    if (!lock_held) lock.lock();
    QueryWs& w = h->ex.ws;
    cudaStream_t st = h->stream;
    const int De = h->kp.D, P = n_outputs(h);
    int rc;
    if (query_path(h, M, !xq_dev && !out_dev && !with_acq) == QP_POINT) {
        // one launch, one synchronisation (query.cu: query_point_kernel)
        Extra& ex = h->ex;
        if (ex.point_cap < P + 1) {
            if (ex.hPoint) cudaFreeHost(ex.hPoint);
            ex.hPoint = ex.dPoint = nullptr;
            LB_CUDA(cudaHostAlloc((void**)&ex.hPoint, sizeof(double) * (P + 1 + 7), cudaHostAllocMapped));
            LB_CUDA(cudaHostGetDevicePointer((void**)&ex.dPoint, ex.hPoint, 0));
            ex.point_cap = P + 1 + 7;
        }
        if ((rc = ensure(h, w.dQs, sizeof(double) * De * LB_TILE))) return rc;
        if ((rc = ensure(h, w.dV, sizeof(double) * lb_query_fused_scratch_doubles(h, 1)))) return rc;
        if ((rc = lb_launch_query_point(h, st, Xq, w.dQs.get(), w.dV.get(), ex.dPoint, &h->launches))) return rc;
        LB_CUDA(cudaStreamSynchronize(st));
        if (mu_out) std::memcpy(mu_out, ex.hPoint, sizeof(double) * P);
        if (s2_out) *s2_out = ex.hPoint[P];
        return LB_OK;
    }
    if ((rc = query_fill(h, M, Xq, xq_dev))) return rc;
    if (!out_dev && (rc = query_timed_out(h))) return rc;
    if (with_acq) {
        const int nrec = (cols && !cols->dInstCol) ? P : 1;
        const int64_t nvals = M * nrec;
        if ((rc = w.am.reserve(h->device, st, M, nrec))) return rc;
        const double* dMean = nullptr;
        if ((rc = mean_on_device(h, st, mean_at_q, nvals, out_dev, &dMean))) return rc;
        double* dAcq = nullptr;
        if (acq_out) {
            if (out_dev) dAcq = acq_out;
            else {
                if ((rc = ensure(h, w.am.vals, sizeof(double) * nvals))) return rc;
                dAcq = w.am.vals.get();
            }
        }
        double* dBV = out_dev ? best_val : w.am.best_val.get();
        long long* dBI = out_dev ? (long long*)best_idx : w.am.best_idx.get();
        if (cols) {
            const double* dParams = cols->dParams;
            if (!dParams) {
                if ((rc = ensure(h, w.dCols, sizeof(double) * 3 * P))) return rc;
                LB_CUDA(cudaMemcpyAsync(w.dCols.get(), acq_params, sizeof(double) * 2 * P, cudaMemcpyHostToDevice, st));
                LB_CUDA(cudaMemcpyAsync(w.dCols.get() + 2 * P, cols->mean_const, sizeof(double) * P, cudaMemcpyHostToDevice, st));
                dParams = w.dCols.get();
            }
            rc = lb_launch_acq_cols(st, acq_id, dParams, M, w.dMu.get(), P, dMean, dParams + 2 * P, w.dS2.get(), cols->dInstCol, cols->lam,
                dAcq, w.am.blk_val.get(), w.am.blk_idx.get(), dBV, dBI, &h->launches);
        } else {
            const double p0 = acq_params ? acq_params[0] : 0.0;
            const double p1 = (acq_params && acq_id == LB_ACQ_EI) ? acq_params[1] : 0.0;
            rc = lb_launch_acq_full(st, acq_id, p0, p1, M, w.dMu.get(), P, dMean, mean_const, w.dS2.get(), dAcq, w.am.blk_val.get(),
                w.am.blk_idx.get(), dBV, dBI, &h->launches);
        }
        if (rc) return rc;
        if (!out_dev && (rc = w.am.read_best(st, best_val, best_idx, acq_out, nvals, nrec))) return rc;
    }
    if (mu_out) {
        LB_CUDA(cudaMemcpyAsync(mu_out, w.dMu.get(), sizeof(double) * M * P, out_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    }
    if (s2_out) {
        LB_CUDA(cudaMemcpyAsync(s2_out, w.dS2.get(), sizeof(double) * M, out_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, st));
    }
    if (!out_dev) LB_CUDA(cudaStreamSynchronize(st));
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_query(const lb_gp* h, int64_t M, const double* Xq, double* mu, double* s2)
{
    return query_common(h, M, Xq, false, mu, s2, false, 0, nullptr, nullptr, 0.0, nullptr, nullptr, nullptr, false);
}
int lb_query_dev(const lb_gp* h, int64_t M, const double* dXq, double* dMu, double* dS2)
{
    return query_common(h, M, dXq, true, dMu, dS2, true, 0, nullptr, nullptr, 0.0, nullptr, nullptr, nullptr, false);
}

int lb_acq_argmax(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* Xq, const double* mean_at_q,
    double mean_const, double* acq_out, double* best_val, int64_t* best_idx)
{
    if (!best_val || !best_idx || !acq_params || M <= 0) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_UNSUPPORTED;
    return query_common(h, M, Xq, false, nullptr, nullptr, false, acq_id, acq_params, mean_at_q, mean_const, acq_out, best_val,
        best_idx, true);
}
int lb_acq_argmax_dev(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* dXq,
    const double* dMean_at_q, double mean_const, double* dAcq_out, double* dBest_val, int64_t* dBest_idx)
{
    if (!dBest_val || !dBest_idx || !acq_params || M <= 0) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_UNSUPPORTED;
    return query_common(h, M, dXq, true, nullptr, nullptr, true, acq_id, acq_params, dMean_at_q, mean_const, dAcq_out,
        dBest_val, dBest_idx, true);
}

// lb_acq_argmax_cols and _dev: one query of the M candidates, scored in each of the handle's q = P columns
static int acq_cols_common(const lb_gp* h, int acq_id, int64_t q, const double* acq_params, int64_t M, const double* Xq, bool dev,
    const double* mean_at_q, const double* mean_const, double* acq_out, double* best_val, int64_t* best_idx)
{
    if (!h || !best_val || !best_idx || !acq_params || !mean_const || M <= 0) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_UNSUPPORTED;
    if (h->precision != LB_PREC_FP64) return LB_ERR_UNSUPPORTED;
    if (q != n_outputs(h)) return LB_ERR_ARG;
    if (q > LB_ACQ_MAX_COLS) return LB_ERR_UNSUPPORTED; // one grid row per column
    const AcqCols cols{mean_const, nullptr, nullptr, 0};
    return query_common(h, M, Xq, dev, nullptr, nullptr, dev, acq_id, acq_params, mean_at_q, 0.0, acq_out, best_val, best_idx, true, false,
        &cols);
}
int lb_acq_argmax_cols(const lb_gp* h, int acq_id, int64_t q, const double* acq_params, int64_t M, const double* Xq, const double* mean_at_q,
    const double* mean_const, double* acq_out, double* best_val, int64_t* best_idx)
{
    return acq_cols_common(h, acq_id, q, acq_params, M, Xq, false, mean_at_q, mean_const, acq_out, best_val, best_idx);
}
int lb_acq_argmax_cols_dev(const lb_gp* h, int acq_id, int64_t q, const double* acq_params, int64_t M, const double* dXq,
    const double* dMean_at_q, const double* mean_const, double* dAcq_out, double* dBest_val, int64_t* dBest_idx)
{
    return acq_cols_common(h, acq_id, q, acq_params, M, dXq, true, dMean_at_q, mean_const, dAcq_out, dBest_val, dBest_idx);
}

// One handle's gradient pass on h->stream: mu (w.dMu, M x P), sigma^2 (w.dS2, M) and the outputs of `out`, whose pointers start at
// candidate 0, for the M row-major device candidates dQraw.  The prior (gp.hpp:161-163: mu = mean(v), added by the caller, sigma^2 =
// k(v, v) + noise, both constant in v: zero gradients) or query_fill's panel chunks, so that mu, sigma^2 and the values are
// bit-identical to that path.  The caller holds h's qmutex and has checked that a handle with samples is fitted.
static int grad_fill(lb_gp_full* h, int64_t M, const double* dQraw, const LbGradOut& out)
{
    QueryWs& w = h->ex.ws;
    cudaStream_t st = h->stream;
    const int D = h->D, P = n_outputs(h);
    int rc;
    if ((rc = ensure(h, w.dMu, sizeof(double) * M * P))) return rc;
    if ((rc = ensure(h, w.dS2, sizeof(double) * M))) return rc;
    if (query_path(h, M) == QP_PRIOR) {
        if ((rc = lb_launch_prior_grad(st, M, D, P, h->kp.sf2 + h->kp.noise, out, w.dMu.get(), w.dS2.get()))) return rc;
        h->launches++;
        return LB_OK;
    }
    auto at = [&](int64_t m0) { // the outputs from candidate m0 on
        LbGradOut o = out;
        o.mean = out.mean ? out.mean + m0 : nullptr;
        o.mean_grad = out.mean_grad ? out.mean_grad + m0 * D : nullptr;
        o.dmu = out.dmu ? out.dmu + m0 * D : nullptr;
        o.ds2 = out.ds2 ? out.ds2 + m0 * D : nullptr;
        o.acq = out.acq ? out.acq + m0 : nullptr;
        o.grad = out.grad ? out.grad + m0 * D : nullptr;
        return o;
    };
    const int64_t Mc = panel_chunk(h, M);
    return for_each_chunk(h, dQraw, M, Mc, LB_TILE, lb_query_panel_scratch_doubles(h, Mc), [&](int64_t m0, int64_t mc, int64_t mcp) {
        return lb_launch_query_grad(h, st, mc, w.dQs.get(), mcp, w.dV.get(), w.dMu.get() + m0 * P, w.dS2.get() + m0, at(m0), &h->launches);
    });
}

// lb_query_grad / lb_acq_grad and their _dev variants: mu, sigma^2 and their candidate gradients, and with acq_id >= 0 the
// acquisition's value and gradient (query_grad.cu), always on the panel path so that mu, sigma^2 and the values are bit-identical to
// lb_query / lb_acq_argmax on that path.  dev: every array is a device pointer (the coordinates are then not checked on the host).
static int grad_common(const lb_gp* hc, int64_t M, const double* Xq, bool dev, double* mu_out, double* s2_out, double* dmu_out,
    double* ds2_out, int acq_id, const double* acq_params, const double* mean_at_q, double mean_const, const double* mean_grad,
    double* acq_out, double* grad_out)
{
    if (!hc || M <= 0 || !Xq) return LB_ERR_ARG;
    if (acq_id >= 0 && ((acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) || !acq_params)) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    if (h->D <= 0 || !h->kernel_set) return LB_ERR_STATE;
    if (h->precision != LB_PREC_FP64) return LB_ERR_UNSUPPORTED;
    const int D = h->D, P = n_outputs(h);
    if (!coordinates_finite(Xq, M, D, dev)) return LB_ERR_ARG;
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    QueryWs& w = h->ex.ws;
    cudaStream_t st = h->stream;
    const bool prior = query_path(h, M) == QP_PRIOR;
    if (prior && h->N != 0) return LB_ERR_STATE;
    int rc;
    const double* dQraw = Xq;
    if (!prior && (rc = candidates_on_device(h, Xq, M, dev, &dQraw))) return rc;
    Staging io(h->device, st, dev); // the means (acquisitions only) and the gradient outputs
    LbGradOut out{};
    out.acq_id = acq_id;
    out.p0 = acq_id >= 0 ? acq_params[0] : 0.0;
    out.p1 = acq_id == LB_ACQ_EI ? acq_params[1] : 0.0;
    out.mean_const = mean_const;
    if ((rc = io.in(mean_at_q, M, &out.mean)) || (rc = io.in(mean_grad, (size_t)M * D, &out.mean_grad))
        || (rc = io.out(dmu_out, (size_t)M * D, &out.dmu)) || (rc = io.out(ds2_out, (size_t)M * D, &out.ds2))
        || (rc = io.out(acq_out, M, &out.acq)) || (rc = io.out(grad_out, (size_t)M * D, &out.grad)))
        return rc;
    if ((rc = grad_fill(h, M, dQraw, out))) return rc;
    const cudaMemcpyKind d2o = dev ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (mu_out) LB_CUDA(cudaMemcpyAsync(mu_out, w.dMu.get(), sizeof(double) * M * P, d2o, st));
    if (s2_out) LB_CUDA(cudaMemcpyAsync(s2_out, w.dS2.get(), sizeof(double) * M, d2o, st));
    if ((rc = io.finish())) return rc;
    if (dev) LB_CUDA(cudaStreamSynchronize(st)); // the device outputs are complete on return too
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

int lb_query_grad(const lb_gp* h, int64_t M, const double* Xq, double* mu, double* s2, double* dmu, double* ds2)
{
    return grad_common(h, M, Xq, false, mu, s2, dmu, ds2, -1, nullptr, nullptr, 0.0, nullptr, nullptr, nullptr);
}
int lb_query_grad_dev(const lb_gp* h, int64_t M, const double* dXq, double* dMu, double* dS2, double* dDmu, double* dDs2)
{
    return grad_common(h, M, dXq, true, dMu, dS2, dDmu, dDs2, -1, nullptr, nullptr, 0.0, nullptr, nullptr, nullptr);
}
int lb_acq_grad(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* Xq, const double* mean_at_q,
    double mean_const, const double* mean_grad_at_q, double* acq_out, double* grad_out)
{
    if (acq_id < 0) return LB_ERR_ARG;
    return grad_common(h, M, Xq, false, nullptr, nullptr, nullptr, nullptr, acq_id, acq_params, mean_at_q, mean_const, mean_grad_at_q,
        acq_out, grad_out);
}
int lb_acq_grad_dev(const lb_gp* h, int acq_id, const double* acq_params, int64_t M, const double* dXq, const double* dMean_at_q,
    double mean_const, const double* dMean_grad_at_q, double* dAcq_out, double* dGrad_out)
{
    if (acq_id < 0) return LB_ERR_ARG;
    return grad_common(h, M, dXq, true, nullptr, nullptr, nullptr, nullptr, acq_id, acq_params, dMean_at_q, mean_const, dMean_grad_at_q,
        dAcq_out, dGrad_out);
}

static int ensure_pair_events(lb_gp_full* h)
{
    for (cudaEvent_t& e : h->ex.ev_pair)
        if (!e) LB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    return LB_OK;
}

// f() under o's query lock, and under c's too when c is not NULL
extern "C++" {
template <typename F>
static int with_query_locks(lb_gp_full* o, lb_gp_full* c, F&& f)
{
    if (!c) {
        std::lock_guard<std::mutex> lock(o->ex.qmutex);
        return f();
    }
    std::scoped_lock lock(o->ex.qmutex, c->ex.qmutex); // deadlock-free whatever order other callers pass the pair in
    return f();
}

// the handles a call over several models forks to besides the first: one or two, the second only with the first; NULL slots unused
using Others = std::array<lb_gp_full*, 2>;

// What a call over several handles shares (ECI, EHVI; values and gradients): every handle's qmutex is held.  The candidates are
// uploaded once; pass(h, dXq) runs o's pass on o's stream and then, when that succeeded, each other handle's on its own stream, so
// that they may overlap.  o's stream then waits for each of the others, and epilogue() enqueues the work over every pass on o's
// stream.  The others' streams wait for the epilogue before the locks are released: a later call on them must not overwrite what
// it reads.  dev: Xq is a device pointer.
template <typename Pass, typename Epilogue>
static int pair_locked(lb_gp_full* o, Others cs, int64_t M, const double* Xq, bool dev, Pass&& pass, Epilogue&& epilogue)
{
    cudaStream_t st = o->stream;
    int rc;
    if ((rc = ensure_pair_events(o))) return rc;
    for (lb_gp_full* c : cs)
        if (c && (rc = ensure_pair_events(c))) return rc;
    const double* dXq = nullptr; // one upload, read by every pass
    if ((rc = candidates_on_device(o, Xq, M, dev, &dXq))) return rc;
    if (cs[0]) {
        LB_CUDA(cudaEventRecord(o->ex.ev_pair[0], st));
        for (lb_gp_full* c : cs)
            if (c) LB_CUDA(cudaStreamWaitEvent(c->stream, o->ex.ev_pair[0], 0));
    }
    rc = pass(o, dXq);
    int rc_c = LB_OK;
    for (lb_gp_full* c : cs)
        if (c && rc == LB_OK && rc_c == LB_OK) rc_c = pass(c, dXq);
    for (lb_gp_full* c : cs)
        if (c) { // o's stream waits for c's pass (and for c's last read of o's candidate buffer)
            LB_CUDA(cudaEventRecord(c->ex.ev_pair[0], c->stream));
            LB_CUDA(cudaStreamWaitEvent(st, c->ex.ev_pair[0], 0));
        }
    if (rc) return rc;
    if (rc_c) return rc_c;
    rc = epilogue();
    if (cs[0]) {
        LB_CUDA(cudaEventRecord(o->ex.ev_pair[1], st));
        for (lb_gp_full* c : cs)
            if (c) LB_CUDA(cudaStreamWaitEvent(c->stream, o->ex.ev_pair[1], 0));
    }
    if (rc) return rc;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// pair_locked for an argmax: each pass is query_fill, and score(dMeans, dAcq, dBestVal, dBestIdx) launches the fused scoring on o's
// stream, dMeans[i] being the i-th handle's (o, cs[0], cs[1]) mean at the candidates on the device (NULL: none).  dev: every
// pointer is a device pointer and the call does not synchronise.  acq_ws: give score a value buffer even when the caller asked
// for none.  After a timed-out reduced-precision pass, pair_locked still records the release of the others' streams: it only
// orders their later work after what o's stream already holds, as on every other path.
template <typename Score>
static int pair_argmax_locked(lb_gp_full* o, Others cs, int64_t M, const double* Xq, bool dev, std::array<const double*, 3> mean_at_q,
    double* acq_out, double* best_val, int64_t* best_idx, bool acq_ws, Score&& score)
{
    cudaStream_t st = o->stream;
    ArgmaxWs& am = o->ex.ws.am;
    auto pass = [&](lb_gp_full* h, const double* dXq) { return query_fill(h, M, dXq, true); };
    return pair_locked(o, cs, M, Xq, dev, pass, [&] {
        int rc;
        if (!dev && (rc = query_timed_out(o))) return rc;
        for (lb_gp_full* c : cs)
            if (!dev && c && (rc = query_timed_out(c))) return rc;
        if ((rc = am.reserve(o->device, st, M))) return rc;
        std::array<const double*, 3> dMeans = {nullptr, nullptr, nullptr};
        lb_gp_full* hs[3] = {o, cs[0], cs[1]};
        for (int i = 0; i < 3; ++i)
            if (hs[i] && (rc = mean_on_device(hs[i], st, mean_at_q[i], M, dev, &dMeans[i]))) return rc;
        double* dAcq = acq_out;
        if ((acq_out && !dev) || (!acq_out && acq_ws)) {
            if ((rc = ensure(o, am.vals, sizeof(double) * M))) return rc;
            dAcq = am.vals.get();
        }
        double* dBV = dev ? best_val : am.best_val.get();
        long long* dBI = dev ? (long long*)best_idx : am.best_idx.get();
        if ((rc = score(dMeans, dAcq, dBV, dBI))) return rc;
        return dev ? LB_OK : am.read_best(st, best_val, best_idx, acq_out, M);
    });
}

// pair_locked for a gradient: each pass is the handle's gradient pass (grad_fill, no acquisition) in its own chunk widths, into its
// own workspace (mu, sigma^2 and dGrad), and epilogue(mo, mc) gets mo / mc with those outputs filled in.
template <typename Epilogue>
static int pair_grad_locked(lb_gp_full* o, lb_gp_full* c, int64_t M, const double* Xq, bool dev, LbPairModel mo, LbPairModel mc,
    Epilogue&& epilogue)
{
    for (lb_gp_full* h : {o, c})
        if (h && query_path(h, M) == QP_PRIOR && h->N != 0) return LB_ERR_STATE;
    auto pass = [&](lb_gp_full* h, const double* dXq) {
        LbPairModel& pm = h == o ? mo : mc;
        const size_t nd = (size_t)M * h->D;
        int rc = ensure(h, h->ex.ws.dGrad, sizeof(double) * 2 * nd);
        if (rc) return rc;
        LbGradOut out{};
        out.acq_id = -1; // mu, sigma^2 and their gradients only
        pm.dmu = out.dmu = h->ex.ws.dGrad.get();
        pm.ds2 = out.ds2 = h->ex.ws.dGrad.get() + nd;
        if ((rc = grad_fill(h, M, dXq, out))) return rc;
        pm.mu = h->ex.ws.dMu.get(); // sized by grad_fill
        pm.p = n_outputs(h);
        pm.s2 = h->ex.ws.dS2.get();
        return LB_OK;
    };
    return pair_locked(o, {c, nullptr}, M, Xq, dev, pass, [&] { return epilogue(mo, mc); });
}
} // extern "C++"

// experimental/acqui/eci.hpp:76-130 over the objective handle o and the constraint handle c (NULL: no constraint model), the
// fused epilogue being query.cu's eci_kernel.
static int eci_locked(lb_gp_full* o, lb_gp_full* c, double f_max, double jitter, int64_t M, const double* Xq, bool dev,
    const double* obj_mean_at_q, double obj_mean_const, const double* con_mean_at_q, double con_mean_const, double* acq_out,
    double* best_val, int64_t* best_idx)
{
    cudaStream_t st = o->stream;
    if (o->N == 0) { // eci.hpp:86: no objective samples, every value is 0 and the first candidate wins
        int rc;
        if ((rc = zero_fill(acq_out, M, dev, st)) || (rc = zero_fill(best_val, 1, dev, st))) return rc;
        return zero_fill(best_idx, 1, dev, st);
    }
    if (o->D <= 0 || !o->kernel_set) return LB_ERR_STATE;
    const bool use_con = c && c->N > 0; // eci.hpp:124: Pf = 1 without constraint samples
    if (use_con && c->D != o->D) return LB_ERR_ARG;
    if (use_con && !c->kernel_set) return LB_ERR_STATE;
    lb_gp_full* cu = use_con ? c : nullptr;
    return pair_argmax_locked(o, {cu, nullptr}, M, Xq, dev, {obj_mean_at_q, con_mean_at_q, nullptr}, acq_out, best_val, best_idx, false,
        [&](std::array<const double*, 3> dMeans, double* dAcq, double* dBV, long long* dBI) {
            const double* dMeanObj = dMeans[0];
            const double* dMeanCon = dMeans[1];
            const int Po = n_outputs(o), Pc = use_con ? n_outputs(c) : 1;
            return lb_launch_eci_full(st, f_max, jitter, M, o->ex.ws.dMu.get(), Po, dMeanObj, obj_mean_const, o->ex.ws.dS2.get(),
                use_con ? c->ex.ws.dMu.get() : nullptr, Pc, dMeanCon, con_mean_const, use_con ? c->ex.ws.dS2.get() : nullptr, dAcq,
                o->ex.ws.am.blk_val.get(), o->ex.ws.am.blk_idx.get(), dBV, dBI, &o->launches);
        });
}

static int eci_common(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* Xq, bool dev,
    const double* obj_mean_at_q, double obj_mean_const, const double* con_mean_at_q, double con_mean_const, double* acq_out,
    double* best_val, int64_t* best_idx)
{
    if (!obj || obj == con || !eci_params || M <= 0 || !Xq || !best_val || !best_idx) return LB_ERR_ARG;
    if (con && con->device != obj->device) return LB_ERR_ARG;
    lb_gp_full* o = full(obj);
    lb_gp_full* c = con ? full(con) : nullptr;
    LB_DEVICE(o);
    return with_query_locks(o, c, [&] {
        return eci_locked(o, c, eci_params[0], eci_params[1], M, Xq, dev, obj_mean_at_q, obj_mean_const, con_mean_at_q, con_mean_const,
            acq_out, best_val, best_idx);
    });
}

int lb_eci_argmax(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* Xq_rowmajor,
    const double* obj_mean_at_q, double obj_mean_const, const double* con_mean_at_q, double con_mean_const, double* acq_out,
    double* best_val, int64_t* best_idx)
{
    return eci_common(obj, con, eci_params, M, Xq_rowmajor, false, obj_mean_at_q, obj_mean_const, con_mean_at_q, con_mean_const,
        acq_out, best_val, best_idx);
}
int lb_eci_argmax_dev(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* dXq_rowmajor,
    const double* dObj_mean_at_q, double obj_mean_const, const double* dCon_mean_at_q, double con_mean_const, double* dAcq_out,
    double* dBest_val, int64_t* dBest_idx)
{
    return eci_common(obj, con, eci_params, M, dXq_rowmajor, true, dObj_mean_at_q, obj_mean_const, dCon_mean_at_q, con_mean_const,
        dAcq_out, dBest_val, dBest_idx);
}

// The argument checks of lb_ehvi_argmax / lb_ehvi_grad (m2 NULL, k x 2 front) and lb_ehvi3d_argmax (k x 3) that need no lock, and
// what the device reads of the front.  Two objectives: the front sorted by f[0], stably by input index (ehvi2d's std::sort gives
// the same sum for a mutually non-dominated front).  Three: ehvi.cu's Front3, each axis sorted stably by input index.
static int ehvi_front(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k, const double* front,
    int64_t M, const double* Xq, std::vector<double>* sorted)
{
    const int K = m2 ? 3 : 2;
    if (!m0 || !m1 || m0 == m1 || !ref_point || k < 0 || (k > 0 && !front) || M <= 0 || !Xq) return LB_ERR_ARG;
    if (m2 && (m2 == m0 || m2 == m1 || m2->device != m0->device)) return LB_ERR_ARG;
    if (m0->device != m1->device) return LB_ERR_ARG;
    for (int d = 0; d < K; ++d)
        if (!std::isfinite(ref_point[d])) return LB_ERR_ARG;
    if (k > (m2 ? LB_EHVI3D_MAX_K : LB_EHVI_MAX_K)) return LB_ERR_UNSUPPORTED; // before the front is read
    for (int64_t i = 0; i < K * k; ++i)
        if (!std::isfinite(front[i])) return LB_ERR_ARG;
    std::vector<int64_t> ord[3];
    for (int d = 0; d < (m2 ? 3 : 1); ++d) {
        ord[d].resize((size_t)k);
        for (int64_t i = 0; i < k; ++i) ord[d][(size_t)i] = i;
        std::stable_sort(ord[d].begin(), ord[d].end(), [&](int64_t a, int64_t b) { return front[K * a + d] < front[K * b + d]; });
    }
    if (!m2) {
        sorted->resize((size_t)(2 * k));
        for (int64_t i = 0; i < k; ++i) {
            (*sorted)[(size_t)(2 * i)] = front[2 * ord[0][(size_t)i]];
            (*sorted)[(size_t)(2 * i + 1)] = front[2 * ord[0][(size_t)i] + 1];
        }
        return LB_OK;
    }
    std::vector<int64_t> rank[3]; // rank[d][p]: point p's position in axis d's order
    for (int d = 0; d < 3; ++d) {
        rank[d].resize((size_t)k);
        for (int64_t i = 0; i < k; ++i) rank[d][(size_t)ord[d][(size_t)i]] = i;
    }
    sorted->resize((size_t)(9 * k));
    double* o = sorted->data();
    for (int64_t i = 0; i < k; ++i) {
        for (int d = 0; d < 3; ++d) o[d * k + i] = front[3 * ord[d][(size_t)i] + d];
        const size_t pz = (size_t)ord[2][(size_t)i], px = (size_t)ord[0][(size_t)i], py = (size_t)ord[1][(size_t)i];
        o[3 * k + i] = (double)rank[0][pz];
        o[4 * k + i] = (double)rank[1][pz];
        o[5 * k + i] = (double)rank[1][px];
        o[6 * k + i] = (double)rank[2][px];
        o[7 * k + i] = (double)rank[0][py];
        o[8 * k + i] = (double)rank[2][py];
    }
    return LB_OK;
}

// ehvi_front's sorted front into a's dFront, on a's stream
static int upload_front(lb_gp_full* a, const std::vector<double>& sorted)
{
    if (sorted.empty()) return LB_OK;
    const size_t bytes = sizeof(double) * sorted.size();
    int rc = ensure(a, a->ex.ws.dFront, bytes);
    if (rc) return rc;
    LB_CUDA(cudaMemcpyAsync(a->ex.ws.dFront.get(), sorted.data(), bytes, cudaMemcpyHostToDevice, a->stream));
    return LB_OK;
}

// The scoring of lb_ehvi_argmax after the models' passes, on a's stream: ehvi_kernel over a's uploaded front and the argmax
static int ehvi_score(lb_gp_full* a, lb_gp_full* b, const double* ref_point, int64_t k, int64_t M, std::array<const double*, 3> dMeans,
    double mean0_const, double mean1_const, double* dAcq, double* dBV, long long* dBI)
{
    QueryWs& w = a->ex.ws;
    int rc;
    if ((rc = lb_launch_ehvi(a->stream, ref_point[0], ref_point[1], k, w.dFront.get(), M, w.dMu.get(), n_outputs(a), dMeans[0], mean0_const,
             w.dS2.get(), b->ex.ws.dMu.get(), n_outputs(b), dMeans[1], mean1_const, b->ex.ws.dS2.get(), dAcq, &a->launches)))
        return rc;
    return lb_launch_values_argmax(a->stream, M, dAcq, w.am.blk_val.get(), w.am.blk_idx.get(), dBV, dBI, &a->launches);
}

// experimental/acqui/ehvi.hpp:70-79 over the models m0 and m1 (ehvi.cu: ehvi_kernel), the front and the reference point on the
// host.  The front is sorted by f[0] once (ehvi_front).
static int ehvi_common(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front, int64_t M,
    const double* Xq, bool dev, const double* mean0_at_q, double mean0_const, const double* mean1_at_q, double mean1_const,
    double* acq_out, double* best_val, int64_t* best_idx)
{
    if (!best_val || !best_idx) return LB_ERR_ARG;
    std::vector<double> sorted;
    int rc = ehvi_front(m0, m1, nullptr, ref_point, k, front, M, Xq, &sorted);
    if (rc) return rc;
    lb_gp_full* a = full(m0);
    lb_gp_full* b = full(m1);
    LB_DEVICE(a);
    std::scoped_lock lock(a->ex.qmutex, b->ex.qmutex); // deadlock-free whatever order other callers pass the pair in
    if (a->D <= 0 || !a->kernel_set || b->D <= 0 || !b->kernel_set) return LB_ERR_STATE;
    if (a->D != b->D) return LB_ERR_ARG;
    return pair_argmax_locked(a, {b, nullptr}, M, Xq, dev, {mean0_at_q, mean1_at_q, nullptr}, acq_out, best_val, best_idx, true,
        [&](std::array<const double*, 3> dMeans, double* dAcq, double* dBV, long long* dBI) {
            int rc = upload_front(a, sorted);
            return rc ? rc : ehvi_score(a, b, ref_point, k, M, dMeans, mean0_const, mean1_const, dAcq, dBV, dBI);
        });
}

int lb_ehvi_argmax(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* Xq_rowmajor, const double* mean0_at_q, double mean0_const, const double* mean1_at_q, double mean1_const,
    double* acq_out, double* best_val, int64_t* best_idx)
{
    return ehvi_common(m0, m1, ref_point, k, front_rowmajor, M, Xq_rowmajor, false, mean0_at_q, mean0_const, mean1_at_q, mean1_const,
        acq_out, best_val, best_idx);
}
int lb_ehvi_argmax_dev(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* dXq_rowmajor, const double* dMean0_at_q, double mean0_const, const double* dMean1_at_q, double mean1_const,
    double* dAcq_out, double* dBest_val, int64_t* dBest_idx)
{
    return ehvi_common(m0, m1, ref_point, k, front_rowmajor, M, dXq_rowmajor, true, dMean0_at_q, mean0_const, dMean1_at_q, mean1_const,
        dAcq_out, dBest_val, dBest_idx);
}

// The front pass of lb_ehvi3d_argmax on a's stream: the sorted front into a's dFront and its per-cell planes into a's dEhvi3, sized
// for M candidates.  The cell passes of any number of M-candidate batches may follow.
static int ehvi3d_front_pass(lb_gp_full* a, const std::vector<double>& sorted, const double* ref_point, int64_t k, int64_t M)
{
    QueryWs& w = a->ex.ws;
    int rc;
    if ((rc = upload_front(a, sorted)) || (rc = ensure(a, w.dEhvi3, sizeof(double) * lb_ehvi3d_ws_doubles(k, M)))) return rc;
    return lb_launch_ehvi3d_front(a->stream, ref_point, k, w.dFront.get(), w.dEhvi3.get(), &a->launches);
}

// The scoring of lb_ehvi3d_argmax after the models' passes and the front pass, on a's stream: the cell pass and the argmax
static int ehvi3d_score(lb_gp_full* a, lb_gp_full* b, lb_gp_full* c, const double* ref_point, int64_t k, int64_t M,
    std::array<const double*, 3> dMeans, std::array<double, 3> mean_const, double* dAcq, double* dBV, long long* dBI)
{
    QueryWs& w = a->ex.ws;
    const LbEhvi3Model g0 = {w.dMu.get(), n_outputs(a), dMeans[0], mean_const[0], w.dS2.get()};
    const LbEhvi3Model g1 = {b->ex.ws.dMu.get(), n_outputs(b), dMeans[1], mean_const[1], b->ex.ws.dS2.get()};
    const LbEhvi3Model g2 = {c->ex.ws.dMu.get(), n_outputs(c), dMeans[2], mean_const[2], c->ex.ws.dS2.get()};
    int rc = lb_launch_ehvi3d_cells(a->stream, ref_point, k, w.dFront.get(), M, g0, g1, g2, w.dEhvi3.get(), dAcq, &a->launches);
    if (rc) return rc;
    return lb_launch_values_argmax(a->stream, M, dAcq, w.am.blk_val.get(), w.am.blk_idx.get(), dBV, dBI, &a->launches);
}

// ehvi3d_sliceupdate (src/ehvi/ehvi_sliceupdate.cc) over the models m0, m1 and m2 (ehvi.cu: the front pass and
// ehvi3d_cells_kernel), the front and the reference point on the host.  m0's stream forks to the other two and joins both before
// the scoring; the front's planes live in m0's query workspace.
static int ehvi3d_common(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k, const double* front,
    int64_t M, const double* Xq, bool dev, const double* mean0_at_q, double mean0_const, const double* mean1_at_q, double mean1_const,
    const double* mean2_at_q, double mean2_const, double* acq_out, double* best_val, int64_t* best_idx)
{
    if (!m2 || !best_val || !best_idx) return LB_ERR_ARG;
    std::vector<double> sorted;
    int rc = ehvi_front(m0, m1, m2, ref_point, k, front, M, Xq, &sorted);
    if (rc) return rc;
    lb_gp_full* a = full(m0);
    lb_gp_full* b = full(m1);
    lb_gp_full* c = full(m2);
    LB_DEVICE(a);
    std::scoped_lock lock(a->ex.qmutex, b->ex.qmutex, c->ex.qmutex); // deadlock-free whatever order other callers pass them in
    for (lb_gp_full* h : {a, b, c})
        if (h->D <= 0 || !h->kernel_set) return LB_ERR_STATE;
    if (a->D != b->D || a->D != c->D) return LB_ERR_ARG;
    return pair_argmax_locked(a, {b, c}, M, Xq, dev, {mean0_at_q, mean1_at_q, mean2_at_q}, acq_out, best_val, best_idx, true,
        [&](std::array<const double*, 3> dMeans, double* dAcq, double* dBV, long long* dBI) {
            int rc = ehvi3d_front_pass(a, sorted, ref_point, k, M);
            return rc ? rc : ehvi3d_score(a, b, c, ref_point, k, M, dMeans, {mean0_const, mean1_const, mean2_const}, dAcq, dBV, dBI);
        });
}

int lb_ehvi3d_argmax(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k, const double* front_rowmajor,
    int64_t M, const double* Xq_rowmajor, const double* mean0_at_q, double mean0_const, const double* mean1_at_q, double mean1_const,
    const double* mean2_at_q, double mean2_const, double* acq_out, double* best_val, int64_t* best_idx)
{
    return ehvi3d_common(m0, m1, m2, ref_point, k, front_rowmajor, M, Xq_rowmajor, false, mean0_at_q, mean0_const, mean1_at_q,
        mean1_const, mean2_at_q, mean2_const, acq_out, best_val, best_idx);
}
int lb_ehvi3d_argmax_dev(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k,
    const double* front_rowmajor, int64_t M, const double* dXq_rowmajor, const double* dMean0_at_q, double mean0_const,
    const double* dMean1_at_q, double mean1_const, const double* dMean2_at_q, double mean2_const, double* dAcq_out, double* dBest_val,
    int64_t* dBest_idx)
{
    return ehvi3d_common(m0, m1, m2, ref_point, k, front_rowmajor, M, dXq_rowmajor, true, dMean0_at_q, mean0_const, dMean1_at_q,
        mean1_const, dMean2_at_q, mean2_const, dAcq_out, dBest_val, dBest_idx);
}

// ---- batched CMA-ES (lb_acq_cmaes, lb_eci_cmaes, lb_ehvi_cmaes; lb_spgp_acq_cmaes in spgp.cu; cmaes.cu) -----------------------------

// Testing hook: with capture on, each search on the calling thread keeps the instances' states after every generation (R x
// lb_cmaes_state_doubles(D) doubles each), then the last generation's R lambda x D candidates and R lambda values.
static thread_local bool g_cmaes_capture = false;
static thread_local std::vector<double> g_cmaes_trace;
extern "C" int lb_debug_cmaes_capture(int on)
{
    g_cmaes_capture = on != 0;
    g_cmaes_trace.clear();
    return LB_OK;
}
// copies min(n, size) doubles of the last capture to dst (may be NULL) and returns its size
extern "C" long long lb_debug_cmaes_trace(double* dst, long long n)
{
    const long long size = (long long)g_cmaes_trace.size();
    if (dst) std::memcpy(dst, g_cmaes_trace.data(), sizeof(double) * (size_t)std::max(0LL, std::min(n, size)));
    return size;
}

extern "C++" {
// The search loop of every device CMA-ES (common.cuh).  prepare(M) runs once before the first generation; per generation the ask
// kernel writes the R lambda candidates to the device, score(dCand, M, dVals, dBestVal, dBestIdx) enqueues the scorer of the _dev
// entry points on them, and the tell kernel updates every live instance.  Each reduced-precision handle clears and sets its
// timeout word in every fill, so after each generation the words in on.timeouts are ORed into one word of the search: a timeout
// in any generation makes the search return LB_ERR_TIMEOUT.  After every 8th generation the host reads that word and the number
// of live instances, and stops when none is left.  The best point over the instances (ties to the lower instance) and the
// candidates scored come back on the host.
int lb_cmaes_search(const LbCmaesHost& on, const lb_cmaes_opts* opts, int64_t R, const double* starts, const LbCmaesPrepare& prepare,
    const LbCmaesScore& score, double* best_x, double* best_val, int64_t* n_evals, const int* cols, int q)
{
    const int D = on.D;
    LbCmaes s{};
    std::vector<double> w;
    int rc = lb_cmaes_setup(*opts, D, (int)R, &s, &w);
    if (rc) return rc;
    const int64_t S = lb_cmaes_state_doubles(D), M = R * s.lam;
    std::vector<double> hs((size_t)(R * S));
    for (int64_t r = 0; r < R; ++r) lb_cmaes_init_state(s, opts->sigma0, starts + r * D, hs.data() + r * S);
    cudaStream_t st = on.stream;
    StreamTemps tmp(on.device, st);
    double *dW = nullptr, *dVals = nullptr, *dBV = nullptr;
    long long* dBI = nullptr;
    int* dLive = nullptr; // [0] live instances, [1] a reduced-precision timeout in some generation
    const size_t nd = sizeof(double) * (size_t)(M * D);
    if ((rc = tmp.alloc(sizeof(double) * w.size(), &dW)) || (rc = tmp.alloc(sizeof(double) * hs.size(), &s.state)) || (rc = tmp.alloc(nd, &s.z))
        || (rc = tmp.alloc(nd, &s.y)) || (rc = tmp.alloc(nd, &s.cand)) || (rc = tmp.alloc(sizeof(double) * M, &dVals))
        || (rc = tmp.alloc(sizeof(double), &dBV)) || (rc = tmp.alloc(sizeof(long long), &dBI)) || (rc = tmp.alloc(2 * sizeof(int), &dLive)))
        return rc;
    LB_CUDA(cudaMemsetAsync(dLive, 0, 2 * sizeof(int), st));
    s.w = dW;
    LB_CUDA(cudaMemcpyAsync(dW, w.data(), sizeof(double) * w.size(), cudaMemcpyHostToDevice, st));
    LB_CUDA(cudaMemcpyAsync(s.state, hs.data(), sizeof(double) * hs.size(), cudaMemcpyHostToDevice, st));
    const bool capture = g_cmaes_capture;
    if (capture) g_cmaes_trace.clear();
    if ((rc = prepare(M))) return rc;
    int g = 0;
    while (g < opts->generations) {
        if ((rc = lb_launch_cmaes_ask(st, s, g, on.launches)) || (rc = score(s.cand, M, dVals, dBV, dBI))) return rc;
        for (const DevBuf<int>* e : on.timeouts) // the scoring of every handle is ordered before this point of the stream
            if (e && *e && (rc = lb_launch_cmaes_flag(st, e->get(), dLive + 1, on.launches))) return rc;
        const bool count = (g + 1) % 8 == 0 && g + 1 < opts->generations;
        if (count) LB_CUDA(cudaMemsetAsync(dLive, 0, sizeof(int), st));
        if ((rc = lb_launch_cmaes_tell(st, s, g, dVals, count ? dLive : nullptr, on.launches))) return rc;
        ++g;
        if (capture) {
            LB_CUDA(cudaMemcpyAsync(hs.data(), s.state, sizeof(double) * hs.size(), cudaMemcpyDeviceToHost, st));
            LB_CUDA(cudaStreamSynchronize(st));
            g_cmaes_trace.insert(g_cmaes_trace.end(), hs.begin(), hs.end());
        }
        if (count) {
            int word[2] = {0, 0};
            LB_CUDA(cudaMemcpyAsync(word, dLive, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
            LB_CUDA(cudaStreamSynchronize(st));
            if (word[1]) return LB_ERR_TIMEOUT;
            if (word[0] == 0) break;
        }
    }
    LB_CUDA(cudaMemcpyAsync(hs.data(), s.state, sizeof(double) * hs.size(), cudaMemcpyDeviceToHost, st));
    if (capture) {
        const size_t n0 = g_cmaes_trace.size();
        g_cmaes_trace.resize(n0 + (size_t)(M * D + M));
        LB_CUDA(cudaMemcpyAsync(g_cmaes_trace.data() + n0, s.cand, nd, cudaMemcpyDeviceToHost, st));
        LB_CUDA(cudaMemcpyAsync(g_cmaes_trace.data() + n0 + M * D, dVals, sizeof(double) * M, cudaMemcpyDeviceToHost, st));
    }
    int timeout = 0;
    LB_CUDA(cudaMemcpyAsync(&timeout, dLive + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    LB_CUDA(cudaStreamSynchronize(st));
    if (timeout) return LB_ERR_TIMEOUT;
    // per instance: best_x at 3 D, best_val at 4 D + 2 D^2 + 1 (cmaes.cu's layout); per column, the first instance bound to it
    // unless a later one is strictly better
    std::vector<int64_t> best((size_t)q, -1);
    for (int64_t r = 0; r < R; ++r) {
        int64_t& b = best[(size_t)(cols ? cols[r] : 0)];
        if (b < 0 || hs[(size_t)(r * S + S - 2)] > hs[(size_t)(b * S + S - 2)]) b = r;
    }
    for (int c = 0; c < q; ++c) {
        std::memcpy(best_x + (int64_t)c * D, hs.data() + best[(size_t)c] * S + 3 * D, sizeof(double) * D);
        best_val[c] = hs[(size_t)(best[(size_t)c] * S + S - 2)];
    }
    *n_evals = (int64_t)g * M;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// the checks every device CMA-ES entry point makes before any lock: pointers, R and finite starts (D columns)
int lb_cmaes_args(const lb_cmaes_opts* opts, int64_t R, const double* starts, int D, const double* best_x, const double* best_val,
    const int64_t* n_evals)
{
    if (!opts || !starts || !best_x || !best_val || !n_evals || R <= 0 || R > (int64_t)INT32_MAX) return LB_ERR_ARG;
    if (D > 0)
        for (int64_t i = 0; i < R * D; ++i)
            if (!std::isfinite(starts[i])) return LB_ERR_ARG;
    return LB_OK;
}

// the search runs on h's stream, pool and launch count and reads the timeout words of the reduced-precision handles it scores
static LbCmaesHost cmaes_host(lb_gp_full* h, std::array<lb_gp_full*, 3> scored)
{
    LbCmaesHost on{h->device, h->stream, h->D, &h->launches, {nullptr, nullptr, nullptr}};
    for (int i = 0; i < 3; ++i) {
        lb_gp_full* q = scored[(size_t)i];
        if (q && q->precision != LB_PREC_FP64 && q->N > 0) on.timeouts[(size_t)i] = &q->ex.ws.dErr; // N == 0: the prior, no word
    }
    return on;
}

static int cmaes_no_prepare(int64_t) { return LB_OK; }
} // extern "C++"

int lb_acq_cmaes(const lb_gp* hc, int acq_id, const double* acq_params, double mean_const, const lb_cmaes_opts* opts, int64_t R,
    const double* starts, double* best_x, double* best_val, int64_t* n_evals)
{
    if (!hc || !acq_params) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    int rc = lb_cmaes_args(opts, R, starts, h->D, best_x, best_val, n_evals);
    if (rc) return rc;
    if (h->D <= 0 || !h->kernel_set) return LB_ERR_STATE;
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex); // the model stays the same for the whole search
    return lb_cmaes_search(
        cmaes_host(h, {h, nullptr, nullptr}), opts, R, starts, cmaes_no_prepare,
        [&](const double* dCand, int64_t M, double* dVals, double* dBV, long long* dBI) {
            return query_common(h, M, dCand, true, nullptr, nullptr, true, acq_id, acq_params, nullptr, mean_const, dVals, dBV,
                (int64_t*)dBI, true, true);
        },
        best_x, best_val, n_evals);
}

int lb_acq_cmaes_cols(const lb_gp* hc, int acq_id, int64_t q, const double* acq_params, const double* mean_const, const lb_cmaes_opts* opts,
    int64_t R, const double* starts, const int* cols, double* best_x, double* best_val, int64_t* n_evals)
{
    if (!hc || !acq_params || !mean_const || !cols) return LB_ERR_ARG;
    if (acq_id != LB_ACQ_UCB && acq_id != LB_ACQ_EI) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    int rc = lb_cmaes_args(opts, R, starts, h->D, best_x, best_val, n_evals);
    if (rc) return rc;
    if (h->precision != LB_PREC_FP64) return LB_ERR_UNSUPPORTED;
    if (q != n_outputs(h)) return LB_ERR_ARG;
    std::vector<char> covered((size_t)q, 0);
    for (int64_t r = 0; r < R; ++r) {
        if (cols[r] < 0 || cols[r] >= q) return LB_ERR_ARG;
        covered[(size_t)cols[r]] = 1;
    }
    if (std::find(covered.begin(), covered.end(), 0) != covered.end()) return LB_ERR_ARG; // every column needs an instance
    if (h->D <= 0 || !h->kernel_set) return LB_ERR_STATE;
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex); // the model stays the same for the whole search
    StreamTemps tmp(h->device, h->stream);
    double* dParams = nullptr;
    int* dInstCol = nullptr;
    auto prepare = [&](int64_t) {
        int rc = tmp.alloc(sizeof(double) * 3 * q, &dParams);
        if (rc || (rc = tmp.alloc(sizeof(int) * R, &dInstCol))) return rc;
        LB_CUDA(cudaMemcpyAsync(dParams, acq_params, sizeof(double) * 2 * q, cudaMemcpyHostToDevice, h->stream));
        LB_CUDA(cudaMemcpyAsync(dParams + 2 * q, mean_const, sizeof(double) * q, cudaMemcpyHostToDevice, h->stream));
        LB_CUDA(cudaMemcpyAsync(dInstCol, cols, sizeof(int) * R, cudaMemcpyHostToDevice, h->stream));
        return LB_OK;
    };
    return lb_cmaes_search(
        cmaes_host(h, {h, nullptr, nullptr}), opts, R, starts, prepare,
        [&](const double* dCand, int64_t M, double* dVals, double* dBV, long long* dBI) {
            const AcqCols c{nullptr, dParams, dInstCol, (int)(M / R)};
            return query_common(h, M, dCand, true, nullptr, nullptr, true, acq_id, acq_params, nullptr, 0.0, dVals, dBV, (int64_t*)dBI, true,
                true, &c);
        },
        best_x, best_val, n_evals, cols, (int)q);
}

int lb_eci_cmaes(const lb_gp* obj, const lb_gp* con, const double* eci_params, double obj_mean_const, double con_mean_const,
    const lb_cmaes_opts* opts, int64_t R, const double* starts, double* best_x, double* best_val, int64_t* n_evals)
{
    if (!obj || obj == con || !eci_params) return LB_ERR_ARG;
    if (con && con->device != obj->device) return LB_ERR_ARG;
    int rc = lb_cmaes_args(opts, R, starts, obj->D, best_x, best_val, n_evals);
    if (rc) return rc;
    lb_gp_full* o = full(obj);
    lb_gp_full* c = con ? full(con) : nullptr;
    LB_DEVICE(o);
    return with_query_locks(o, c, [&] { // both models stay the same for the whole search
        if (o->D <= 0) return LB_ERR_STATE;
        if (o->N == 0) { // eci.hpp:86: every value is 0, so the first start wins and nothing is scored
            std::memcpy(best_x, starts, sizeof(double) * o->D);
            *best_val = 0.0;
            *n_evals = 0;
            return LB_OK;
        }
        if (!o->kernel_set) return LB_ERR_STATE;
        const bool use_con = c && c->N > 0; // eci_locked's rules: Pf = 1 without constraint samples
        if (use_con && c->D != o->D) return LB_ERR_ARG;
        if (use_con && !c->kernel_set) return LB_ERR_STATE;
        return lb_cmaes_search(
            cmaes_host(o, {o, use_con ? c : nullptr, nullptr}), opts, R, starts, cmaes_no_prepare,
            [&](const double* dCand, int64_t M, double* dVals, double* dBV, long long* dBI) {
                return eci_locked(o, c, eci_params[0], eci_params[1], M, dCand, true, nullptr, obj_mean_const, nullptr, con_mean_const,
                    dVals, dBV, (int64_t*)dBI);
            },
            best_x, best_val, n_evals);
    });
}

int lb_ehvi_cmaes(const lb_gp* m0, const lb_gp* m1, const lb_gp* m2, const double* ref_point, int64_t k, const double* front,
    double mean0_const, double mean1_const, double mean2_const, const lb_cmaes_opts* opts, int64_t R, const double* starts,
    double* best_x, double* best_val, int64_t* n_evals)
{
    if (!m0) return LB_ERR_ARG;
    int rc = lb_cmaes_args(opts, R, starts, m0->D, best_x, best_val, n_evals);
    if (rc) return rc;
    std::vector<double> sorted;
    if ((rc = ehvi_front(m0, m1, m2, ref_point, k, front, 1, starts, &sorted))) return rc;
    lb_gp_full* a = full(m0);
    lb_gp_full* b = full(m1);
    lb_gp_full* c = m2 ? full(m2) : nullptr;
    LB_DEVICE(a);
    auto locked = [&] {
        for (lb_gp_full* h : {a, b, c})
            if (h && (h->D <= 0 || !h->kernel_set)) return LB_ERR_STATE;
        if (a->D != b->D || (c && a->D != c->D)) return LB_ERR_ARG;
        auto prepare = [&](int64_t M) { return c ? ehvi3d_front_pass(a, sorted, ref_point, k, M) : upload_front(a, sorted); };
        auto score = [&](const double* dCand, int64_t M, double* dVals, double* dBV, long long* dBI) {
            return pair_argmax_locked(a, {b, c}, M, dCand, true, {nullptr, nullptr, nullptr}, dVals, dBV, (int64_t*)dBI, true,
                [&](std::array<const double*, 3> dMeans, double* dAcq, double* dB, long long* dI) {
                    return c ? ehvi3d_score(a, b, c, ref_point, k, M, dMeans, {mean0_const, mean1_const, mean2_const}, dAcq, dB, dI)
                             : ehvi_score(a, b, ref_point, k, M, dMeans, mean0_const, mean1_const, dAcq, dB, dI);
                });
        };
        return lb_cmaes_search(cmaes_host(a, {a, b, c}), opts, R, starts, prepare, score, best_x, best_val, n_evals);
    };
    if (c) {
        std::scoped_lock lock(a->ex.qmutex, b->ex.qmutex, c->ex.qmutex); // deadlock-free whatever order other callers pass them in
        return locked();
    }
    std::scoped_lock lock(a->ex.qmutex, b->ex.qmutex);
    return locked();
}

// ---- gradients of the two-model acquisitions (lb_eci_grad, lb_ehvi_grad) -------------------------------------------------------

// lb_eci_grad(_dev) under the locks: eci_locked's cases (no objective samples: 0 everywhere; a constraint without samples: Pf = 1),
// with query.cu's eci_grad_kernel as the epilogue
static int eci_grad_locked(lb_gp_full* o, lb_gp_full* c, double f_max, double jitter, int64_t M, const double* Xq, bool dev,
    const double* obj_mean, double obj_mean_const, const double* obj_mean_grad, const double* con_mean, double con_mean_const,
    const double* con_mean_grad, double* acq_out, double* grad_out)
{
    if (o->D <= 0) return LB_ERR_STATE; // the gradient has D columns: unlike eci_locked, the input dimension must be known
    const int D = o->D;
    if (c && c->D > 0 && c->D != D) return LB_ERR_ARG;
    if (!coordinates_finite(Xq, M, D, dev)) return LB_ERR_ARG;
    cudaStream_t st = o->stream;
    int rc;
    if (o->N == 0) { // eci.hpp:86: no objective samples, every value and gradient is 0 (before the kernel is consulted, as eci_locked)
        if ((rc = zero_fill(acq_out, M, dev, st))) return rc;
        return zero_fill(grad_out, M * D, dev, st);
    }
    if (!o->kernel_set) return LB_ERR_STATE;
    const bool use_con = c && c->N > 0; // eci.hpp:124: Pf = 1 without constraint samples
    if (use_con && !c->kernel_set) return LB_ERR_STATE;
    Staging io(o->device, st, dev);
    LbPairModel mo{}, mc{};
    double *dAcq = nullptr, *dGrad = nullptr;
    mo.mean_const = obj_mean_const;
    mc.mean_const = con_mean_const;
    if ((rc = io.in(obj_mean, M, &mo.mean)) || (rc = io.in(obj_mean_grad, (size_t)M * D, &mo.mean_grad))) return rc;
    if (use_con && ((rc = io.in(con_mean, M, &mc.mean)) || (rc = io.in(con_mean_grad, (size_t)M * D, &mc.mean_grad)))) return rc;
    if ((rc = io.out(acq_out, M, &dAcq)) || (rc = io.out(grad_out, (size_t)M * D, &dGrad))) return rc;
    rc = pair_grad_locked(o, use_con ? c : nullptr, M, Xq, dev, mo, mc, [&](const LbPairModel& a, const LbPairModel& b) {
        return lb_launch_eci_grad(st, f_max, jitter, M, D, a, b, dAcq, dGrad, &o->launches);
    });
    return rc ? rc : io.finish();
}

static int eci_grad_common(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* Xq, bool dev,
    const double* obj_mean, double obj_mean_const, const double* obj_mean_grad, const double* con_mean, double con_mean_const,
    const double* con_mean_grad, double* acq_out, double* grad_out)
{
    if (!obj || obj == con || !eci_params || M <= 0 || !Xq) return LB_ERR_ARG;
    if (con && con->device != obj->device) return LB_ERR_ARG;
    if (obj->precision != LB_PREC_FP64 || (con && con->precision != LB_PREC_FP64)) return LB_ERR_UNSUPPORTED;
    lb_gp_full* o = full(obj);
    lb_gp_full* c = con ? full(con) : nullptr;
    LB_DEVICE(o);
    return with_query_locks(o, c, [&] {
        return eci_grad_locked(o, c, eci_params[0], eci_params[1], M, Xq, dev, obj_mean, obj_mean_const, obj_mean_grad, con_mean,
            con_mean_const, con_mean_grad, acq_out, grad_out);
    });
}

int lb_eci_grad(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* Xq_rowmajor,
    const double* obj_mean_at_q, double obj_mean_const, const double* obj_mean_grad_at_q, const double* con_mean_at_q,
    double con_mean_const, const double* con_mean_grad_at_q, double* acq_out, double* grad_out)
{
    return eci_grad_common(obj, con, eci_params, M, Xq_rowmajor, false, obj_mean_at_q, obj_mean_const, obj_mean_grad_at_q,
        con_mean_at_q, con_mean_const, con_mean_grad_at_q, acq_out, grad_out);
}
int lb_eci_grad_dev(const lb_gp* obj, const lb_gp* con, const double* eci_params, int64_t M, const double* dXq_rowmajor,
    const double* dObj_mean_at_q, double obj_mean_const, const double* dObj_mean_grad_at_q, const double* dCon_mean_at_q,
    double con_mean_const, const double* dCon_mean_grad_at_q, double* dAcq_out, double* dGrad_out)
{
    return eci_grad_common(obj, con, eci_params, M, dXq_rowmajor, true, dObj_mean_at_q, obj_mean_const, dObj_mean_grad_at_q,
        dCon_mean_at_q, con_mean_const, dCon_mean_grad_at_q, dAcq_out, dGrad_out);
}

// lb_ehvi_grad(_dev): ehvi_common's checks and sorted front, ehvi.cu's ehvi_grad_kernel as the epilogue
static int ehvi_grad_common(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front, int64_t M,
    const double* Xq, bool dev, const double* mean0, double mean0_const, const double* mean0_grad, const double* mean1,
    double mean1_const, const double* mean1_grad, double* acq_out, double* grad_out)
{
    std::vector<double> sorted;
    int rc = ehvi_front(m0, m1, nullptr, ref_point, k, front, M, Xq, &sorted);
    if (rc) return rc;
    if (m0->precision != LB_PREC_FP64 || m1->precision != LB_PREC_FP64) return LB_ERR_UNSUPPORTED;
    lb_gp_full* a = full(m0);
    lb_gp_full* b = full(m1);
    LB_DEVICE(a);
    std::scoped_lock lock(a->ex.qmutex, b->ex.qmutex);
    if (a->D <= 0 || !a->kernel_set || b->D <= 0 || !b->kernel_set) return LB_ERR_STATE;
    if (a->D != b->D) return LB_ERR_ARG;
    const int D = a->D;
    if (!coordinates_finite(Xq, M, D, dev)) return LB_ERR_ARG;
    cudaStream_t st = a->stream;
    Staging io(a->device, st, dev);
    LbPairModel g0{}, g1{};
    double *dAcq = nullptr, *dGrad = nullptr;
    g0.mean_const = mean0_const;
    g1.mean_const = mean1_const;
    if ((rc = io.in(mean0, M, &g0.mean)) || (rc = io.in(mean0_grad, (size_t)M * D, &g0.mean_grad)) || (rc = io.in(mean1, M, &g1.mean))
        || (rc = io.in(mean1_grad, (size_t)M * D, &g1.mean_grad)))
        return rc;
    if ((rc = io.out(acq_out, M, &dAcq)) || (rc = io.out(grad_out, (size_t)M * D, &dGrad))) return rc;
    rc = pair_grad_locked(a, b, M, Xq, dev, g0, g1, [&](const LbPairModel& p0, const LbPairModel& p1) {
        const int r = upload_front(a, sorted);
        if (r) return r;
        return lb_launch_ehvi_grad(st, ref_point[0], ref_point[1], k, a->ex.ws.dFront.get(), M, D, p0, p1, dAcq, dGrad, &a->launches);
    });
    return rc ? rc : io.finish();
}

int lb_ehvi_grad(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* Xq_rowmajor, const double* mean0_at_q, double mean0_const, const double* mean0_grad_at_q, const double* mean1_at_q,
    double mean1_const, const double* mean1_grad_at_q, double* acq_out, double* grad_out)
{
    return ehvi_grad_common(m0, m1, ref_point, k, front_rowmajor, M, Xq_rowmajor, false, mean0_at_q, mean0_const, mean0_grad_at_q,
        mean1_at_q, mean1_const, mean1_grad_at_q, acq_out, grad_out);
}
int lb_ehvi_grad_dev(const lb_gp* m0, const lb_gp* m1, const double* ref_point, int64_t k, const double* front_rowmajor, int64_t M,
    const double* dXq_rowmajor, const double* dMean0_at_q, double mean0_const, const double* dMean0_grad_at_q,
    const double* dMean1_at_q, double mean1_const, const double* dMean1_grad_at_q, double* dAcq_out, double* dGrad_out)
{
    return ehvi_grad_common(m0, m1, ref_point, k, front_rowmajor, M, dXq_rowmajor, true, dMean0_at_q, mean0_const, dMean0_grad_at_q,
        dMean1_at_q, mean1_const, dMean1_grad_at_q, dAcq_out, dGrad_out);
}

// pareto::impl::pareto_set_std<K> (experimental/tools/pareto.hpp:138-162) on h's device and stream, under h's query lock: the
// domination test on the device (ehvi.cu: pareto_kernel), then the kept indices in compare_objs_lex order on the host
// (lexicographically descending; exact ties by ascending index, where the reference's unstable sort leaves them unordered).
static int pareto_common(const lb_gp* hc, int64_t n, int K, const double* objs, int64_t* idx, int64_t* n_front, bool dev)
{
    if (!hc || n < 0 || K < 1 || !n_front || (n > 0 && (!objs || !idx))) return LB_ERR_ARG;
    if (K > LB_PARETO_MAX_K || n >= INT32_MAX) return LB_ERR_UNSUPPORTED;
    lb_gp_full* h = full(hc);
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    *n_front = 0;
    if (n == 0) return LB_OK;
    cudaStream_t st = h->stream;
    std::vector<double> hobj;
    std::vector<int> keep((size_t)n);
    int herr = 0;
    int rc;
    {
        Staging io(h->device, st, dev);
        int* dKeep = nullptr;
        const double* dO = nullptr;
        if ((rc = io.tmp.alloc(sizeof(int) * (n + 1), &dKeep)) || (rc = io.in(objs, (size_t)(n * K), &dO))) return rc;
        LB_CUDA(cudaMemsetAsync(dKeep + n, 0, sizeof(int), st));
        if ((rc = lb_launch_pareto(st, n, K, dO, dKeep, dKeep + n, &h->launches))) return rc;
        LB_CUDA(cudaMemcpyAsync(keep.data(), dKeep, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
        LB_CUDA(cudaMemcpyAsync(&herr, dKeep + n, sizeof(int), cudaMemcpyDeviceToHost, st));
        if (dev) {
            hobj.resize((size_t)(n * K));
            LB_CUDA(cudaMemcpyAsync(hobj.data(), objs, sizeof(double) * n * K, cudaMemcpyDeviceToHost, st));
        }
        LB_CUDA(cudaStreamSynchronize(st));
    }
    if (herr) return LB_ERR_ARG;
    const double* O = dev ? hobj.data() : objs;
    std::vector<int64_t> front;
    for (int64_t i = 0; i < n; ++i)
        if (keep[(size_t)i]) front.push_back(i);
    std::sort(front.begin(), front.end(), [&](int64_t a, int64_t b) { // pareto.hpp:98-111, then the index
        for (int d = 0; d < K; ++d) {
            if (O[a * K + d] > O[b * K + d]) return true;
            if (O[a * K + d] < O[b * K + d]) return false;
        }
        return a < b;
    });
    *n_front = (int64_t)front.size();
    if (dev) {
        LB_CUDA(cudaMemcpyAsync(idx, front.data(), sizeof(int64_t) * front.size(), cudaMemcpyHostToDevice, st));
        LB_CUDA(cudaStreamSynchronize(st));
    }
    else std::memcpy(idx, front.data(), sizeof(int64_t) * front.size());
    return LB_OK;
}

int lb_pareto_set(const lb_gp* h, int64_t n, int K, const double* objs_rowmajor, int64_t* idx, int64_t* n_front)
{
    return pareto_common(h, n, K, objs_rowmajor, idx, n_front, false);
}
int lb_pareto_set_dev(const lb_gp* h, int64_t n, int K, const double* dObjs_rowmajor, int64_t* dIdx, int64_t* n_front)
{
    return pareto_common(h, n, K, dObjs_rowmajor, dIdx, n_front, true);
}

// model::SparsifiedGP::_sparsify (sparsified_gp.hpp:121-183) on h's device and stream, under h's query lock (the call uses h's
// stream but not its model state).  N <= max_points keeps every point and launches nothing.
static int sparsify_common(const lb_gp* hc, int64_t N, int D, const double* X, int64_t max_points, int64_t* kept, int64_t* n_kept,
    int64_t* removed, double* removed_score, bool dev)
{
    if (!hc || N < 0 || D < 1 || max_points < 0 || !n_kept || (N > 0 && (!X || !kept))) return LB_ERR_ARG;
    if (D > LB_MAX_D || N >= INT32_MAX) return LB_ERR_UNSUPPORTED;
    if (max_points < D) return LB_ERR_ARG; // the reference's partial_sort would run past end()
    lb_gp_full* h = full(hc);
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    cudaStream_t st = h->stream;
    if (N <= max_points) {
        std::vector<int64_t> all((size_t)N);
        for (int64_t i = 0; i < N; ++i) all[(size_t)i] = i;
        if (dev && N > 0) {
            LB_CUDA(cudaMemcpyAsync(kept, all.data(), sizeof(int64_t) * N, cudaMemcpyHostToDevice, st));
            LB_CUDA(cudaStreamSynchronize(st));
        }
        else if (N > 0) std::memcpy(kept, all.data(), sizeof(int64_t) * N);
        *n_kept = N;
        return LB_OK;
    }
    if (dev) return lb_run_sparsify(h, st, N, D, X, max_points, (long long*)kept, n_kept, (long long*)removed, removed_score, &h->launches);
    Staging io(h->device, st, false); // the outputs' lengths are known after the run: their copies back stay here
    const double* dX = nullptr;
    long long *dKept = nullptr, *dRm = nullptr;
    double* dRs = nullptr;
    int rc;
    if ((rc = io.in(X, (size_t)(N * D), &dX)) || (rc = io.tmp.alloc(sizeof(long long) * N, &dKept))
        || (removed && (rc = io.tmp.alloc(sizeof(long long) * N, &dRm)))
        || (removed_score && (rc = io.tmp.alloc(sizeof(double) * N, &dRs))))
        return rc;
    if ((rc = lb_run_sparsify(h, st, N, D, dX, max_points, dKept, n_kept, dRm, dRs, &h->launches))) return rc;
    const int64_t nr = N - *n_kept;
    LB_CUDA(cudaMemcpyAsync(kept, dKept, sizeof(int64_t) * *n_kept, cudaMemcpyDeviceToHost, st));
    if (removed && nr > 0) LB_CUDA(cudaMemcpyAsync(removed, dRm, sizeof(int64_t) * nr, cudaMemcpyDeviceToHost, st));
    if (removed_score && nr > 0) LB_CUDA(cudaMemcpyAsync(removed_score, dRs, sizeof(double) * nr, cudaMemcpyDeviceToHost, st));
    LB_CUDA(cudaStreamSynchronize(st));
    return LB_OK;
}

int lb_sparsify(const lb_gp* h, int64_t N, int D, const double* X_rowmajor, int64_t max_points, int64_t* kept, int64_t* n_kept,
    int64_t* removed, double* removed_score)
{
    return sparsify_common(h, N, D, X_rowmajor, max_points, kept, n_kept, removed, removed_score, false);
}
int lb_sparsify_dev(const lb_gp* h, int64_t N, int D, const double* dX_rowmajor, int64_t max_points, int64_t* dKept, int64_t* n_kept,
    int64_t* dRemoved, double* dRemovedScore)
{
    return sparsify_common(h, N, D, dX_rowmajor, max_points, dKept, n_kept, dRemoved, dRemovedScore, true);
}

int lb_log_lik(lb_gp* hh, double* out)
{
    if (!hh || !out) return LB_ERR_ARG;
    if (!hh->fitted) return LB_ERR_STATE;
    LB_DEVICE(hh);
    lb_gp_full* h = full(hh);
    int rc = lb_launch_loglik(h, h->ex.dMisc.get());
    if (rc) return rc;
    double v[3];
    LB_CUDA(cudaMemcpyAsync(v, h->ex.dMisc.get(), sizeof(v), cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    *out = v[2];
    return LB_OK;
}

int lb_compute_inv_kernel(lb_gp* h)
{
    if (!h) return LB_ERR_ARG;
    if (!h->fitted) return LB_ERR_STATE;
    if (h->kinv_valid) return LB_OK;
    LB_DEVICE(h);
    return lb_launch_kinv(h);
}

int lb_kernel_grad_log_lik(lb_gp* hh, int optimize_noise, double* grad)
{
    if (!hh || !grad) return LB_ERR_ARG;
    if (!hh->fitted) return LB_ERR_STATE;
    LB_DEVICE(hh);
    lb_gp_full* h = full(hh);
    int rc;
    if (!h->kinv_valid && (rc = lb_launch_kinv(h))) return rc;
    const int nh = h->n_hparams + (optimize_noise ? 1 : 0);
    if (nh > LB_MAX_HPARAMS) return LB_ERR_ARG;
    if ((rc = lb_launch_grad(h, optimize_noise, h->ex.dMisc.get() + 8))) return rc;
    LB_CUDA(cudaMemcpyAsync(grad, h->ex.dMisc.get() + 8, sizeof(double) * nh, cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    return LB_OK;
}

// GP::compute_log_lik and compute_kernel_grad_log_lik at R kernel states of this handle's data (lml_batch.cu), under the query
// lock.  The per-vector kernel state is derived on the host by lb_set_kernel's kernel_state, so a vector sees the K the single
// path builds.
static int lml_grad_batch_common(lb_gp* hh, int kernel_id, int64_t R, int n_hparams, const double* log_hparams, const double* noise,
    int optimize_noise, double* lik, double* grad, int* info, bool dev)
{
    if (!hh) return LB_ERR_ARG;
    if (hh->D <= 0 || hh->N == 0 || !hh->dX) return LB_ERR_STATE;
    if (R <= 0 || R > INT32_MAX || !log_hparams || !noise || !lik) return LB_ERR_ARG;
    if (kernel_id < 0 || kernel_id > 3) return LB_ERR_ARG;
    const int Draw = hh->D;
    const int klam = hparam_klam(kernel_id, Draw, n_hparams);
    if (klam < 0) return klam;
    if (hh->N > LB_LML_BATCH_MAX_N) return LB_ERR_UNSUPPORTED;
    lb_gp_full* h = full(hh);
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    cudaStream_t st = h->stream;
    std::vector<double> hp_dev, no_dev;
    const double* hp = log_hparams;
    const double* no = noise;
    if (dev) { // the kernel state is derived on the host: fetch the vectors
        hp_dev.resize((size_t)(R * n_hparams));
        no_dev.resize((size_t)R);
        LB_CUDA(cudaMemcpyAsync(hp_dev.data(), log_hparams, sizeof(double) * hp_dev.size(), cudaMemcpyDeviceToHost, st));
        LB_CUDA(cudaMemcpyAsync(no_dev.data(), noise, sizeof(double) * R, cudaMemcpyDeviceToHost, st));
        LB_CUDA(cudaStreamSynchronize(st));
        hp = hp_dev.data();
        no = no_dev.data();
    }
    for (int64_t i = 0; i < R * n_hparams; ++i)
        if (!std::isfinite(hp[i])) return LB_ERR_ARG;
    for (int64_t r = 0; r < R; ++r)
        if (!std::isfinite(no[r])) return LB_ERR_ARG;
    std::vector<KernParams> kps((size_t)R);
    for (int64_t r = 0; r < R; ++r) kernel_state(kps[(size_t)r], kernel_id, Draw, klam, hp + r * n_hparams, n_hparams, no[r]);
    const int nh = n_hparams + (optimize_noise ? 1 : 0);
    Staging io(h->device, st, dev);
    double *dLik = nullptr, *dGrad = nullptr;
    int* dInfo = nullptr;
    int rc;
    if ((rc = io.out(lik, (size_t)R, &dLik)) || (rc = io.out(grad, (size_t)(R * nh), &dGrad)) || (rc = io.out(info, (size_t)R, &dInfo)))
        return rc;
    if ((rc = lb_launch_lml_batch(st, io.tmp, kps.data(), hp, n_hparams, (int)R, h->dX, h->Np, h->dY, (int)h->N, h->P, nh,
             optimize_noise ? 1 : 0, dLik, dGrad, dInfo, &h->launches)))
        return rc;
    if ((rc = io.finish())) return rc;
    if (dev) LB_CUDA(cudaStreamSynchronize(st)); // the device outputs are complete on return too
    return LB_OK;
}

int lb_lml_grad_batch(lb_gp* h, int kernel_id, int64_t R, int n_hparams, const double* log_hparams, const double* noise,
    int optimize_noise, double* lik, double* grad, int* info)
{
    return lml_grad_batch_common(h, kernel_id, R, n_hparams, log_hparams, noise, optimize_noise, lik, grad, info, false);
}
int lb_lml_grad_batch_dev(lb_gp* h, int kernel_id, int64_t R, int n_hparams, const double* dLog_hparams, const double* dNoise,
    int optimize_noise, double* dLik, double* dGrad, int* dInfo)
{
    return lml_grad_batch_common(h, kernel_id, R, n_hparams, dLog_hparams, dNoise, optimize_noise, dLik, dGrad, dInfo, true);
}

int lb_log_loo_cv(lb_gp* hh, double* out)
{
    if (!hh || !out) return LB_ERR_ARG;
    if (!hh->fitted) return LB_ERR_STATE;
    LB_DEVICE(hh);
    lb_gp_full* h = full(hh);
    int rc = lb_launch_loo_value(h, h->ex.dMisc.get() + 4);
    if (rc) return rc;
    LB_CUDA(cudaMemcpyAsync(out, h->ex.dMisc.get() + 4, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    return LB_OK;
}

int lb_kernel_grad_log_loo_cv(lb_gp* hh, int optimize_noise, double* grad)
{
    if (!hh || !grad) return LB_ERR_ARG;
    if (!hh->fitted) return LB_ERR_STATE;
    LB_DEVICE(hh);
    lb_gp_full* h = full(hh);
    const int nh = h->n_hparams + (optimize_noise ? 1 : 0);
    if (nh > LB_MAX_HPARAMS) return LB_ERR_ARG;
    int rc = lb_launch_loo_grad(h, optimize_noise, h->ex.dMisc.get() + 8);
    if (rc) return rc;
    LB_CUDA(cudaMemcpyAsync(grad, h->ex.dMisc.get() + 8, sizeof(double) * nh, cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    return LB_OK;
}

int lb_kinv_obs_mean(lb_gp* h, double* out)
{
    if (!h || !out) return LB_ERR_ARG;
    if (!h->fitted) return LB_ERR_STATE;
    LB_DEVICE(h);
    StreamTemps tmp(h->device, h->stream);
    double* dOut = nullptr;
    int rc;
    if ((rc = tmp.alloc(sizeof(double) * h->N * h->P, &dOut)) || (rc = lb_launch_kinv_obs(h, dOut))) return rc;
    LB_CUDA(cudaMemcpyAsync(out, dOut, sizeof(double) * h->N * h->P, cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    return LB_OK;
}

int lb_get(lb_gp* h, int what, double* dst)
{
    if (!h || !dst) return LB_ERR_ARG;
    if (h->N == 0) return LB_ERR_STATE;
    LB_DEVICE(h);
    const int64_t N = h->N, Np = h->Np;
    int rc;
    if (what == LB_GET_ALPHA) {
        if (!h->fitted) return LB_ERR_STATE;
        LB_CUDA(cudaMemcpy2DAsync(dst, N * 8, h->dAlpha, Np * 8, N * 8, h->P, cudaMemcpyDeviceToHost, h->stream));
        LB_CUDA(cudaStreamSynchronize(h->stream));
        return LB_OK;
    }
    if ((rc = lb_ensure_scratch(h, sizeof(double) * (size_t)(Np * Np + N * N)))) return rc;
    double* dTmp = h->dScratch.get();
    double* dOut = h->dScratch.get() + Np * Np;
    const double* src = nullptr;
    int lower = 0;
    if (what == LB_GET_K) {
        if (!h->kernel_set) return LB_ERR_STATE;
        if ((rc = make_unique(h, &h->dXs, shared_bytes(h).Xs, false))) return rc;
        if ((rc = lb_launch_scale_x(h))) return rc;
        if ((rc = lb_launch_kbuild(h, dTmp))) return rc;
        src = dTmp;
    }
    else if (what == LB_GET_L) {
        if (!h->fitted) return LB_ERR_STATE;
        src = h->dL;
        lower = 1;
    }
    else if (what == LB_GET_KINV) {
        if (!h->fitted) return LB_ERR_STATE;
        if (!h->kinv_valid && (rc = lb_launch_kinv(h))) return rc;
        if (!h->kinv_sym) {
            if ((rc = lb_launch_symmetrize(h, h->dKinv.get()))) return rc;
            h->kinv_sym = true;
        }
        src = h->dKinv.get();
    }
    else
        return LB_ERR_ARG;
    extract_kernel<<<1024, 256, 0, h->stream>>>(src, Np, N, dOut, lower);
    h->launches++;
    LB_CUDA(cudaMemcpyAsync(dst, dOut, sizeof(double) * N * N, cudaMemcpyDeviceToHost, h->stream));
    LB_CUDA(cudaStreamSynchronize(h->stream));
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// The copy constructor KernelLFOptimization relies on (model/gp/kernel_lf_opt.hpp:79).  Nothing is copied: the clone
// references the source's buffers, and whichever of the two writes first (lb_fit, lb_append, lb_set_data, ...) takes a
// private buffer from the pool at that point (make_unique).  K^-1 / L^-1 are not carried over (the reference's copy
// keeps _inv_kernel, but every consumer recomputes it after recompute(), and lb_compute_inv_kernel rebuilds it on demand).
int lb_clone(const lb_gp* src, lb_gp** out)
{
    if (!src || !out) return LB_ERR_ARG;
    LB_DEVICE(src);
    lb_gp* h = nullptr;
    int rc = lb_create(&h, src->device, src->precision);
    if (rc) return rc;
    // pending writes of the source (e.g. lb_fit_async) must be complete before another stream reads the shared buffers
    if (cudaStreamSynchronize(src->stream) != cudaSuccess) { lb_destroy(h); return LB_ERR_CUDA; }
    h->kp = src->kp; h->kernel_set = src->kernel_set; h->n_hparams = src->n_hparams;
    h->N = src->N; h->D = src->D; h->P = src->P;
    h->kp.lambda = nullptr;
    std::memcpy(full(h)->ex.lambda_host, full(src)->ex.lambda_host, sizeof(full(h)->ex.lambda_host));
    if (src->kp.klam > 0) { // own copy of the Lambda matrix (rewritten by every lb_set_kernel)
        if (h->dLambda.resize(h, sizeof(double) * LB_MAX_D * LB_MAX_LAMBDA)
            || cudaMemcpyAsync(h->dLambda.get(), src->dLambda.get(), sizeof(double) * LB_MAX_D * LB_MAX_LAMBDA, cudaMemcpyDeviceToDevice, h->stream) != cudaSuccess) {
            lb_destroy(h);
            return LB_ERR_CUDA;
        }
        h->kp.lambda = h->dLambda.get();
    }
    if (src->Np > 0) {
        h->Np = src->Np;
        auto share = [](double* p) { lb_pool_retain(p); return p; };
        h->dX = share(src->dX);
        h->dY = share(src->dY);
        h->dXs = share(src->dXs);
        if (src->fitted) {
            h->dAlpha = share(src->dAlpha);
            h->dL = share(src->dL);
            h->dInvD = share(src->dInvD);
            h->fitted = true;
        }
        if (src->dFlags && h->dFlags.resize(h, sizeof(int) * (src->Np / LB_TILE + 8))) { lb_destroy(h); return LB_ERR_ALLOC; }
    }
    *out = h;
    return LB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Distributed fit (limbo_b200/dist_fit.py): the factor of ONE GP is computed by all ranks together with the block-cyclic
// panel factorisation of config 5 (potrf.cu lb_dchol_*), and every rank assembles the complete factor in its own handle
// from the panels that travel anyway, so that prediction / acquisition can then shard over the ranks without any further
// exchange.  The panel message of pair p is  [ head: the pair's 256 x 256 diagonal block, column-major ld 256 |
// inv(L_kk), inv(L_k+1,k+1) : 2 x 128 x 128 | rows below the pair, ld = Nd - (kpair + 2) * 128 ]  (LB_DCHOL_HEAD doubles
// before the rows).  The update order per tile is lb_fit's, so the assembled factor is bit-identical to lb_fit's.
// ---------------------------------------------------------------------------------------------------------------------
#define LB_DCHOL_HEAD (2 * LB_TILE * 2 * LB_TILE + 2 * LB_TILE * LB_TILE)

namespace {
// head of the message from the owner's pair columns (dCols: Nd x 256, ld = Nd) and its two diagonal-block inverses
__global__ void __launch_bounds__(256)
dchol_pack_head_kernel(const double* __restrict__ cols, int64_t ld, int64_t row0, const double* __restrict__ invD, double* __restrict__ head)
{
    const int idx = blockIdx.x * 256 + threadIdx.x;
    constexpr int DIAG = 2 * LB_TILE * 2 * LB_TILE;
    if (idx < DIAG) {
        const int r = idx & 255, c = idx >> 8;
        head[idx] = cols[row0 + r + (int64_t)c * ld];
    }
    else if (idx < LB_DCHOL_HEAD)
        head[idx] = invD[idx - DIAG];
}
// message -> this rank's factor storage: L[row0 + r, row0 + c] (r < 256: head; r >= 256: rows below), invD[kpair], invD[kpair + 1]
__global__ void __launch_bounds__(256)
dchol_unpack_kernel(const double* __restrict__ msg, int64_t ldp, double* __restrict__ L, int64_t ld, int64_t row0, double* __restrict__ invD_pair)
{
    const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x; // row inside the column block, 0 .. 256 + ldp
    const int c = blockIdx.y;
    constexpr int DIAG = 2 * LB_TILE * 2 * LB_TILE;
    if (r < 2 * LB_TILE) L[row0 + r + (row0 + c) * ld] = msg[r + c * 2 * LB_TILE];
    else if (r < 2 * LB_TILE + ldp) L[row0 + r + (row0 + c) * ld] = msg[LB_DCHOL_HEAD + (r - 2 * LB_TILE) + (int64_t)c * ldp];
    if (blockIdx.x == 0) { // the two inverse blocks: 32768 doubles over 256 columns x 256 threads
        const int idx = c * 256 + threadIdx.x;
        if (idx < 2 * LB_TILE * LB_TILE) invD_pair[idx] = msg[DIAG + idx];
    }
}
} // namespace

// the owner of pair `kpair`: writes the head of the message (after lb_dchol_panel has factored the pair; same stream)
int lb_dchol_pack_head(lb_gp* h, const double* dCols, int64_t Nd, int kpair, const double* dInvD, double* dMsg)
{
    if (!h || !dCols || !dInvD || !dMsg) return LB_ERR_ARG;
    LB_DEVICE(h);
    dchol_pack_head_kernel<<<(LB_DCHOL_HEAD + 255) / 256, 256, 0, h->stream>>>(dCols, Nd, (int64_t)kpair * LB_TILE, dInvD, dMsg);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}

// Target handle (data and kernel already set, lb_set_data + lb_set_kernel): private factor buffers, staged samples.  The padded
// order of the handle must equal the distributed order Nd (N a multiple of 256, or 128 < N mod 256).
int lb_dchol_adopt_begin(lb_gp* h, int64_t Nd)
{
    if (!h) return LB_ERR_ARG;
    if (!h->kernel_set || h->N == 0 || h->Np == 0 || !h->dX) return LB_ERR_STATE;
    if (h->Np != Nd) return LB_ERR_UNSUPPORTED;
    LB_DEVICE(h);
    int rc = stage_fit(h);
    if (rc) return rc;
    LB_CUDA(cudaMemsetAsync(h->dInfo.get(), 0, 2 * sizeof(int), h->stream));
    h->fitted = false;
    lb_factor_changed(h);
    return LB_OK;
}
// one received (or own) panel message into the handle's L / invD, on `stream` (cudaStream_t as void*; NULL = the handle's)
int lb_dchol_unpack(lb_gp* h, const double* dMsg, int64_t Nd, int kpair, void* stream)
{
    if (!h || !dMsg || !h->dL || !h->dInvD || h->Np != Nd) return LB_ERR_ARG;
    LB_DEVICE(h);
    const int64_t row0 = (int64_t)kpair * LB_TILE, ldp = Nd - row0 - 2 * LB_TILE;
    cudaStream_t st = stream ? (cudaStream_t)stream : h->stream;
    dim3 grid((unsigned)((2 * LB_TILE + ldp + 255) / 256), 2 * LB_TILE);
    dchol_unpack_kernel<<<grid, 256, 0, st>>>(dMsg, ldp, h->dL, Nd, row0, h->dInvD + (int64_t)kpair * LB_TILE * LB_TILE);
    h->launches++;
    LB_CUDA(cudaGetLastError());
    return LB_OK;
}
// all panels are in: the handle is fitted (info = the distributed factorisation's), alpha is solved locally (gp.hpp:605-611)
int lb_dchol_adopt_end(lb_gp* h, int info)
{
    if (!h) return LB_ERR_ARG;
    LB_DEVICE(h);
    if (info > 0) return info;
    h->fitted = true;
    lb_factor_changed(h);
    int rc = lb_launch_solve_alpha(h);
    if (rc) return rc;
    return check_info(h);
}

// ---- inversion of the factor spread over G GPUs, for the reduced-precision candidate path (limbo_b200_dist.h) --------------------

static int dinv_check(const lb_gp* h, int rank, int G)
{
    if (!h || G < 1 || rank < 0 || rank >= G) return LB_ERR_ARG;
    if (!h->fitted || h->N == 0) return LB_ERR_STATE;
    if (h->precision != LB_PREC_TF32 && h->precision != LB_PREC_FP16 && h->precision != LB_PREC_FP16X3) return LB_ERR_UNSUPPORTED;
    return LB_OK;
}

long long lb_dinv_chunk_bytes(const lb_gp* h, int G)
{
    int rc = dinv_check(h, 0, G);
    return rc ? (long long)rc : (long long)lb_dinv_chunk_bytes_impl(h, G);
}

int lb_dinv_columns(lb_gp* hc, int rank, int G, double* absmax_host)
{
    int rc = dinv_check(hc, rank, G);
    if (rc) return rc;
    if (!absmax_host) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    QueryWs& w = h->ex.ws;
    if ((rc = ensure(h, w.dV, sizeof(double) * lb_linv_columns_scratch_doubles(h, G)))) return rc;
    if ((rc = lb_launch_linv_columns(h, h->stream, rank, G, w.dV.get(), &h->launches))) return rc;
    return lb_dinv_absmax(h, w.dV.get(), G, absmax_host);
}

int lb_dinv_pack(lb_gp* hc, int rank, int G, double absmax_all, void* dChunk)
{
    int rc = dinv_check(hc, rank, G);
    if (rc) return rc;
    if (!dChunk) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    QueryWs& w = h->ex.ws;
    if (!w.dV || w.dV.bytes() < sizeof(double) * lb_linv_columns_scratch_doubles(h, G)) return LB_ERR_STATE; // lb_dinv_columns first
    return lb_dinv_pack_impl(h, w.dV.get(), rank, G, absmax_all, dChunk);
}

int lb_dinv_adopt(lb_gp* hc, int G, const void* dAll, double absmax_all)
{
    int rc = dinv_check(hc, 0, G);
    if (rc) return rc;
    if (!dAll) return LB_ERR_ARG;
    lb_gp_full* h = full(hc);
    LB_DEVICE(h);
    std::lock_guard<std::mutex> lock(h->ex.qmutex);
    return lb_dinv_adopt_impl(h, G, dAll, absmax_all);
}

// per-kernel-class event timing for bench.py's roofline (not part of the reference-facing header)
int lb_profile_enable(lb_gp* h, int on)
{
    if (!h) return LB_ERR_ARG;
    LB_DEVICE(h);
    if (on && !h->prof) h->prof = new Profiler();
    if (!on && h->prof) {
        cudaStreamSynchronize(h->stream);
        Profiler* p = (Profiler*)h->prof;
        for (auto& r : p->recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
        for (auto e : p->pool) cudaEventDestroy(e);
        delete p;
        h->prof = nullptr;
    }
    return LB_OK;
}
// accumulates finished records; ms_out / count_out have LB_PC_COUNT entries; reset != 0 clears the totals
int lb_profile_read(lb_gp* h, double* ms_out, long long* count_out, int reset)
{
    if (!h || !h->prof) return LB_ERR_STATE;
    LB_DEVICE(h);
    Profiler* p = (Profiler*)h->prof;
    LB_CUDA(cudaStreamSynchronize(h->stream));
    std::lock_guard<std::mutex> lk(p->mu);
    const bool dump = getenv("LB_PROF_TIMELINE") != nullptr; // debug: per-launch (class, start, end) in ms from the first record
    for (auto& r : p->recs) {
        float ms = 0.f;
        if (dump && !p->recs.empty()) {
            float t0 = 0.f, t1 = 0.f;
            if (cudaEventElapsedTime(&t0, p->recs[0].a, r.a) == cudaSuccess && cudaEventElapsedTime(&t1, p->recs[0].a, r.b) == cudaSuccess)
                fprintf(stderr, "LBTL %d %.3f %.3f\n", r.cls, t0, t1);
        }
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { p->ms[r.cls] += ms; p->n[r.cls]++; }
        p->pool.push_back(r.a); p->pool.push_back(r.b);
    }
    p->recs.clear();
    for (int c = 0; c < LB_PC_COUNT; ++c) {
        if (ms_out) ms_out[c] = p->ms[c];
        if (count_out) count_out[c] = p->n[c];
        if (reset) { p->ms[c] = 0; p->n[c] = 0; }
    }
    return LB_OK;
}

const char* lb_strerror(int code)
{
    if (code > 0) return "kernel matrix is not positive definite (value = 1-based index of the failing pivot)";
    switch (code) {
    case LB_OK: return "ok";
    case LB_ERR_ARG: return "invalid argument";
    case LB_ERR_CUDA: return "CUDA runtime error (see lb_last_cuda_error)";
    case LB_ERR_STATE: return "call sequence error (data / kernel / fit missing)";
    case LB_ERR_ALLOC: return "device memory allocation failed";
    case LB_ERR_UNSUPPORTED: return "unsupported kernel / acquisition / precision";
    case LB_ERR_TIMEOUT: return "device-side wait timed out";
    default: return "unknown error";
    }
}

const char* lb_last_cuda_error(void) { return g_last_cuda_error.c_str(); }

} // extern "C"
