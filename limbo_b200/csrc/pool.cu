// limbo_b200/csrc/pool.cu — per-device buffer pool with reference counts.
//
// model::gp::KernelLFOpt copies the whole GP for every likelihood evaluation (model/gp/kernel_lf_opt.hpp:79:
// `GP gp(this->_original_gp)`), and opt::ParallelRepeater does that from several threads
// (opt/parallel_repeater.hpp:86-103).  On the CPU that copy is a memcpy next to an O(N^3) refit; on the GPU a
// cudaMalloc / cudaFree pair per N x N buffer (2.1 GB at N = 16384) synchronises the device and costs more than the
// kernels it feeds.  So:
//   * every device buffer of a handle comes from this pool and goes back to it (exact-size free lists, bounded by
//     LB_POOL_BYTES, default 48 GiB per device) - after the first evaluation a clone allocates nothing;
//   * buffers carry a reference count: lb_clone shares X, Y, the factor, ... with its source, and a handle takes a
//     private buffer only when it is about to WRITE one that is still shared (copy-on-write; the copy itself is
//     skipped when the writer overwrites the whole buffer, which is what recompute() does).
// Callers guarantee that a buffer has no pending device work when its last reference is dropped (handles synchronise
// their stream before releasing).
#include "common.cuh"
#include <cstdlib>
#include <map>
#include <mutex>
#include <unordered_map>
#include <vector>

namespace {

struct Entry { size_t bytes; int device; int ref; };

struct Pool {
    std::mutex mu;
    std::unordered_map<void*, Entry> live;                  // leased buffers
    std::map<std::pair<int, size_t>, std::vector<void*>> free_; // (device, rounded bytes) -> idle buffers
    size_t free_bytes[64] = {};
    long long n_malloc = 0, n_hit = 0;
    size_t cap = 0;
};

Pool& pool()
{
    static Pool* p = [] {
        Pool* q = new Pool(); // leaked on purpose: handles may be destroyed from static destructors
        const char* e = getenv("LB_POOL_BYTES");
        q->cap = e ? (size_t)strtoull(e, nullptr, 10) : ((size_t)48 << 30);
        return q;
    }();
    return *p;
}

size_t round_size(size_t b)
{
    if (b < 256) return 256;
    if (b <= ((size_t)1 << 20)) { // powers of two below 1 MiB
        size_t r = 256;
        while (r < b) r <<= 1;
        return r;
    }
    const size_t g = (size_t)1 << 20;
    return (b + g - 1) / g * g;
}

// drop idle buffers of `device` until at most `keep` bytes stay (largest first); pool mutex held
void trim_locked(Pool& P, int device, size_t keep)
{
    while (P.free_bytes[device] > keep) {
        auto best = P.free_.end();
        for (auto it = P.free_.begin(); it != P.free_.end(); ++it)
            if (it->first.first == device && !it->second.empty() && (best == P.free_.end() || it->first.second > best->first.second)) best = it;
        if (best == P.free_.end()) break;
        void* p = best->second.back();
        best->second.pop_back();
        P.free_bytes[device] -= best->first.second;
        cudaFree(p);
    }
}

} // namespace

void* lb_pool_alloc(int device, size_t bytes)
{
    if (device < 0 || device >= 64) return nullptr;
    Pool& P = pool();
    const size_t rb = round_size(bytes);
    {
        std::lock_guard<std::mutex> lk(P.mu);
        auto it = P.free_.find({device, rb});
        if (it != P.free_.end() && !it->second.empty()) {
            void* p = it->second.back();
            it->second.pop_back();
            P.free_bytes[device] -= rb;
            P.live[p] = Entry{rb, device, 1};
            P.n_hit++;
            return p;
        }
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, rb);
    if (e != cudaSuccess) { // give the idle buffers back and retry once
        cudaGetLastError();
        {
            std::lock_guard<std::mutex> lk(P.mu);
            trim_locked(P, device, 0);
        }
        e = cudaMalloc(&p, rb);
        if (e != cudaSuccess) {
            lb_set_last_cuda_error(e, __FILE__, __LINE__);
            return nullptr;
        }
    }
    std::lock_guard<std::mutex> lk(P.mu);
    P.live[p] = Entry{rb, device, 1};
    P.n_malloc++;
    return p;
}

void lb_pool_retain(void* p)
{
    if (!p) return;
    Pool& P = pool();
    std::lock_guard<std::mutex> lk(P.mu);
    auto it = P.live.find(p);
    if (it != P.live.end()) it->second.ref++;
}

bool lb_pool_shared(void* p)
{
    if (!p) return false;
    Pool& P = pool();
    std::lock_guard<std::mutex> lk(P.mu);
    auto it = P.live.find(p);
    return it != P.live.end() && it->second.ref > 1;
}

void lb_pool_free(void* p)
{
    if (!p) return;
    Pool& P = pool();
    std::lock_guard<std::mutex> lk(P.mu);
    auto it = P.live.find(p);
    if (it == P.live.end()) { // not ours (should not happen): plain free
        cudaFree(p);
        return;
    }
    if (--it->second.ref > 0) return;
    const Entry e = it->second;
    P.live.erase(it);
    P.free_[{e.device, e.bytes}].push_back(p);
    P.free_bytes[e.device] += e.bytes;
    if (P.free_bytes[e.device] > P.cap) trim_locked(P, e.device, P.cap);
}

extern "C" {
// cudaMalloc calls / pool hits so far (tests: a likelihood evaluation on a warm pool allocates nothing)
long long lb_debug_pool_mallocs(void) { Pool& P = pool(); std::lock_guard<std::mutex> lk(P.mu); return P.n_malloc; }
long long lb_debug_pool_hits(void) { Pool& P = pool(); std::lock_guard<std::mutex> lk(P.mu); return P.n_hit; }
// buffers currently leased (tests: a balanced round of calls returns every lease it took)
long long lb_debug_pool_live(void) { Pool& P = pool(); std::lock_guard<std::mutex> lk(P.mu); return (long long)P.live.size(); }
// release every idle buffer of every device back to the driver
int lb_pool_trim(void)
{
    Pool& P = pool();
    int prev = -1;
    cudaGetDevice(&prev);
    std::lock_guard<std::mutex> lk(P.mu);
    for (int d = 0; d < 64; ++d)
        if (P.free_bytes[d]) {
            cudaSetDevice(d);
            trim_locked(P, d, 0);
        }
    if (prev >= 0) cudaSetDevice(prev);
    return LB_OK;
}
}
