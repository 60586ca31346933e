// gem_b200/csrc/core.cu -- context, errors, pinned memory, NCCL bootstrap, graph upload.
#include "common.cuh"
#include "nccl_api.h"
#include <dlfcn.h>
#include <stdarg.h>
#include <string.h>
#include <atomic>
#include <map>
#include <mutex>
#include <unordered_map>
#include <stdlib.h>

namespace gemb {

static thread_local char g_err[1024] = "";
static std::atomic<long long> g_launches{0};
void count_launch(int k) { g_launches.fetch_add(k, std::memory_order_relaxed); }
long long launches_total() { return g_launches.load(std::memory_order_relaxed); }

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

int launch_status(const void *kernel) {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) {
        count_launch();
        return GEMB_OK;
    }
    const char *name = nullptr;
    if (cudaFuncGetName(&name, kernel) != cudaSuccess || !name) name = "a kernel";
    set_error("launch of %s failed: %s", name, cudaGetErrorString(e));
    (void)cudaGetLastError();   // clear a non-sticky error for later calls
    return GEMB_ERR_CUDA;
}

int copy_sync(gemb_ctx *ctx, void *dst, const void *src, size_t bytes, cudaMemcpyKind kind) {
    GEMB_CUDA(cudaMemcpyAsync(dst, src, bytes, kind, ctx->stream));
    GEMB_CUDA(cudaStreamSynchronize(ctx->stream));
    return GEMB_OK;
}

int Timer::begin(cudaStream_t s) {
    if (used + 2 > ev.size()) {
        size_t old = ev.size();
        ev.resize(old + 64);
        for (size_t i = old; i < ev.size(); i++) GEMB_CUDA(cudaEventCreate(&ev[i]));
    }
    GEMB_CUDA(cudaEventRecord(ev[used], s));
    return GEMB_OK;
}
int Timer::end(cudaStream_t s) {
    GEMB_CUDA(cudaEventRecord(ev[used + 1], s));
    used += 2;
    return GEMB_OK;
}
double Timer::total_ms() {
    double t = 0;
    for (size_t i = 0; i + 1 < used; i += 2) {
        float ms = 0;
        if (cudaEventSynchronize(ev[i + 1]) != cudaSuccess) return -1;
        if (cudaEventElapsedTime(&ms, ev[i], ev[i + 1]) != cudaSuccess) return -1;
        t += ms;
    }
    return t;
}
void Timer::destroy() {
    for (auto e : ev) cudaEventDestroy(e);
    ev.clear();
    used = 0;
}

static NcclApi g_nccl;
static int g_nccl_state = 0;  // 0 untried, 1 ok, -1 failed

NcclApi *nccl_api() {
    if (g_nccl_state == 1) return &g_nccl;
    if (g_nccl_state == -1) return nullptr;
    void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
        set_error("cannot dlopen libnccl.so.2: %s", dlerror());
        g_nccl_state = -1;
        return nullptr;
    }
#define LOAD(name)                                                      \
    g_nccl.name = (decltype(g_nccl.name))dlsym(h, "nccl" #name);        \
    if (!g_nccl.name) {                                                 \
        set_error("libnccl lacks symbol nccl" #name);                   \
        g_nccl_state = -1;                                              \
        return nullptr;                                                 \
    }
    LOAD(GetUniqueId) LOAD(CommInitRank) LOAD(CommDestroy) LOAD(AllReduce) LOAD(AllGather) LOAD(Broadcast)
    LOAD(GetErrorString) LOAD(GetVersion)
#undef LOAD
    g_nccl_state = 1;
    return &g_nccl;
}

// ---- device block cache (see common.cuh).  One free list per device, keyed by rounded size.
namespace {
struct BlockCache {
    std::mutex mu;
    std::multimap<size_t, void *> free_[64];
    std::unordered_map<void *, std::pair<size_t, int>> live;   // cached-class blocks handed out: ptr -> (size, device)
    size_t cached_bytes = 0;
    long long limit = -1;
    size_t cap() {
        if (limit < 0) { const char *e = getenv("GEMB_CACHE_MB"); limit = (e ? atoll(e) : 65536LL) << 20; }
        return (size_t)limit;
    }
    void trim_locked(int dev) {   // dev < 0: all devices
        int cur = 0; cudaGetDevice(&cur);
        for (int d = 0; d < 64; d++) {
            if ((dev >= 0 && d != dev) || free_[d].empty()) continue;
            cudaSetDevice(d);
            for (auto &kv : free_[d]) { cudaFree(kv.second); cached_bytes -= kv.first; }
            free_[d].clear();
        }
        cudaSetDevice(cur);
    }
};
BlockCache g_cache;
const size_t kCacheMin = (size_t)1 << 20, kCacheRound = (size_t)2 << 20;
}  // namespace

cudaError_t dmalloc_bytes(void **p, size_t bytes) {
    if (g_cache.cap() == 0) return cudaMalloc(p, bytes ? bytes : 4);
    const size_t rnd = bytes < kCacheMin ? 512 : kCacheRound;   // small blocks are cached too: fewer driver calls per call
    const size_t sz = (bytes + rnd - 1) / rnd * rnd + (bytes == 0 ? rnd : 0);
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lk(g_cache.mu);
    if (dev < 64) {
        auto it = g_cache.free_[dev].find(sz);
        if (it != g_cache.free_[dev].end()) {
            *p = it->second;
            g_cache.free_[dev].erase(it);
            g_cache.cached_bytes -= sz;
            g_cache.live[*p] = {sz, dev};
            return cudaSuccess;
        }
    }
    e = cudaMalloc(p, sz);
    if (e == cudaErrorMemoryAllocation) {   // give the cached blocks back to the driver and retry once
        (void)cudaGetLastError();
        g_cache.trim_locked(dev);
        e = cudaMalloc(p, sz);
    }
    if (e == cudaSuccess && dev < 64) g_cache.live[*p] = {sz, dev};
    return e;
}

cudaError_t dfree(void *p) {
    if (!p) return cudaSuccess;
    {
        std::lock_guard<std::mutex> lk(g_cache.mu);
        auto it = g_cache.live.find(p);
        if (it != g_cache.live.end()) {
            const size_t sz = it->second.first;
            const int dev = it->second.second;
            g_cache.live.erase(it);
            if (g_cache.cached_bytes + sz <= g_cache.cap()) {
                int cur = 0; cudaGetDevice(&cur);
                if (cur != dev) cudaSetDevice(dev);
                cudaError_t e = cudaDeviceSynchronize();   // what cudaFree would have done: no kernel still uses the block
                if (cur != dev) cudaSetDevice(cur);
                if (e == cudaSuccess) {
                    g_cache.free_[dev].emplace(sz, p);
                    g_cache.cached_bytes += sz;
                    return cudaSuccess;
                }
            }
        }
    }
    return cudaFree(p);
}

}  // namespace gemb

using namespace gemb;

extern "C" {

int gemb_mem_trim(void) {
    std::lock_guard<std::mutex> lk(g_cache.mu);
    g_cache.trim_locked(-1);
    return GEMB_OK;
}

size_t gemb_mem_cached_bytes(void) {
    std::lock_guard<std::mutex> lk(g_cache.mu);
    return g_cache.cached_bytes;
}

size_t gemb_mem_live_blocks(void) {
    std::lock_guard<std::mutex> lk(g_cache.mu);
    return g_cache.live.size();
}

int gemb_version(void) { return GEMB_VERSION; }
int64_t gemb_launch_count(void) { return (int64_t)gemb::launches_total(); }
const char *gemb_last_error(void) { return g_err; }

int gemb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int gemb_ctx_create(int device, gemb_ctx **out) {
    GEMB_ARG(out != nullptr, "out");
    int n = gemb_device_count();
    if (n <= 0) {
        set_error("no CUDA device visible: libgemb200 has no CPU fallback");
        return GEMB_ERR_CUDA;
    }
    GEMB_ARG(device >= 0 && device < n, "device index");
    GEMB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    GEMB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("device %d is sm_%d%d; libgemb200 is built for sm_90a (H100) only", device, prop.major,
                  prop.minor);
        return GEMB_ERR_CUDA;
    }
    gemb_ctx *c = new gemb_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    GEMB_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    GEMB_CUDA(cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking));
    *out = c;
    return GEMB_OK;
}

int gemb_ctx_destroy(gemb_ctx *c) {
    if (!c) return GEMB_OK;
    cudaSetDevice(c->device);
    gemb::halo_pool_release(c);
    if (c->comm) {
        NcclApi *api = nccl_api();
        if (api) api->CommDestroy((ncclComm_t)c->comm);
    }
    c->t_spmm.destroy();
    c->t_dense.destroy();
    c->t_comm.destroy();
    c->t_misc.destroy();
    dfree(c->spmm_scratch);
    dfree(c->red_scratch);
    if (c->stream) cudaStreamDestroy(c->stream);
    if (c->side) cudaStreamDestroy(c->side);
    delete c;
    return GEMB_OK;
}

int gemb_host_alloc(size_t bytes, void **out) {
    GEMB_ARG(out != nullptr, "out");
    GEMB_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
    return GEMB_OK;
}
int gemb_host_free(void *p) {
    if (p) GEMB_CUDA(cudaFreeHost(p));
    return GEMB_OK;
}

int gemb_comm_unique_id(void *id_out) {
    GEMB_ARG(id_out != nullptr, "id_out");
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    ncclUniqueId id;
    ncclResult_t r = api->GetUniqueId(&id);
    if (r != ncclSuccess) {
        set_error("ncclGetUniqueId: %s", api->GetErrorString(r));
        return GEMB_ERR_NCCL;
    }
    static_assert(sizeof(id) == GEMB_UNIQUE_ID_BYTES, "ncclUniqueId size");
    memcpy(id_out, &id, sizeof id);
    return GEMB_OK;
}

int gemb_comm_init(gemb_ctx *c, int rank, int nranks, const void *idp) {
    GEMB_ARG(c && idp, "ctx/id");
    GEMB_ARG(nranks >= 1 && rank >= 0 && rank < nranks, "rank/nranks");
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    GEMB_CUDA(cudaSetDevice(c->device));
    ncclUniqueId id;
    memcpy(&id, idp, sizeof id);
    ncclComm_t comm;
    ncclResult_t r = api->CommInitRank(&comm, nranks, id, rank);
    if (r != ncclSuccess) {
        set_error("ncclCommInitRank: %s", api->GetErrorString(r));
        return GEMB_ERR_NCCL;
    }
    c->comm = comm;
    c->rank = rank;
    c->nranks = nranks;
    return GEMB_OK;
}

// flags[0] |= 1: offsets not monotone; |= 2: a column id outside [0, n)   (ADVICE r1: a malformed CSR must fail
// loudly at upload, not read out of bounds in the sweeps)
__global__ void csr_validate_kernel(int64_t n_local, int64_t nnz, int64_t n, const int32_t *__restrict__ indptr,
                                    const int32_t *__restrict__ indices, int *__restrict__ flags) {
    int bad = 0;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_local; r += stride)
        if (indptr[r + 1] < indptr[r]) bad |= 1;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += stride) {
        const int32_t cidx = indices[i];
        if (cidx < 0 || (int64_t)cidx >= n) bad |= 2;
    }
    if (bad) atomicOr(flags, bad);
}

static int upload_csr(gemb_ctx *c, int64_t n, int64_t n_local, const int32_t *indptr, const int32_t *indices,
                      const float *data, gemb_csr_dev *d) {
    int64_t nnz = indptr[n_local] - indptr[0];
    GEMB_ARG(indptr[0] == 0, "indptr[0] must be 0 (shard-local offsets)");
    GEMB_ARG(nnz >= 0 && nnz < (int64_t)2147483647, "nnz per shard must be < 2^31");
    d->nnz = nnz;
    GEMB_CUDA(dmalloc(&d->indptr, sizeof(int32_t) * (n_local + 1)));
    GEMB_CUDA(dmalloc(&d->indices, sizeof(int32_t) * ((nnz > 0 ? nnz : 1) + 4)));
    GEMB_CUDA(cudaMemcpyAsync(d->indptr, indptr, sizeof(int32_t) * (n_local + 1),
                              cudaMemcpyHostToDevice, c->stream));
    if (nnz)
        GEMB_CUDA(cudaMemcpyAsync(d->indices, indices, sizeof(int32_t) * nnz, cudaMemcpyHostToDevice,
                                  c->stream));
    if (data && nnz) {
        GEMB_CUDA(dmalloc(&d->data, sizeof(float) * (nnz + 4)));
        GEMB_CUDA(cudaMemcpyAsync(d->data, data, sizeof(float) * nnz, cudaMemcpyHostToDevice,
                                  c->stream));
    }
    {
        DeviceBuffer<int> flags;
        int h = 0;
        GEMB_CUDA(flags.alloc(1));
        GEMB_CUDA(cudaMemsetAsync(flags.get(), 0, sizeof(int), c->stream));
        GEMB_TRY(launch(c, csr_validate_kernel, c->sm_count * 4, 256, 0, n_local, nnz, n, d->indptr, d->indices, flags.get()));
        GEMB_TRY(copy_sync(c, &h, flags.get(), sizeof(int), cudaMemcpyDeviceToHost));
        if (h) {
            set_error("malformed CSR:%s%s", (h & 1) ? " row offsets are not monotone;" : "",
                      (h & 2) ? " a column id lies outside [0, n)" : "");
            return GEMB_ERR_ARG;
        }
    }
    // heavy rows -> chunk work items (see common.cuh); one pass over the host offsets
    std::vector<int32_t> hrow, hfirst, irow, ibeg;
    for (int64_t r = 0; r < n_local; r++) {
        const int32_t s = indptr[r], e = indptr[r + 1];
        if (e - s <= SPMM_HEAVY_DEG) continue;
        hrow.push_back((int32_t)r);
        hfirst.push_back((int32_t)irow.size());
        for (int32_t b0 = s; b0 < e; b0 += SPMM_HEAVY_CHUNK) { irow.push_back((int32_t)r); ibeg.push_back(b0); }
    }
    d->n_heavy = (int32_t)hrow.size();
    d->n_items = (int32_t)irow.size();
    if (d->n_heavy) {
        hfirst.push_back(d->n_items);
        GEMB_CUDA(dmalloc(&d->heavy_row, sizeof(int32_t) * hrow.size()));
        GEMB_CUDA(dmalloc(&d->heavy_first, sizeof(int32_t) * hfirst.size()));
        GEMB_CUDA(dmalloc(&d->item_row, sizeof(int32_t) * irow.size()));
        GEMB_CUDA(dmalloc(&d->item_beg, sizeof(int32_t) * ibeg.size()));
        // synchronous copies: the staging vectors die with this scope
        GEMB_CUDA(cudaMemcpy(d->heavy_row, hrow.data(), sizeof(int32_t) * hrow.size(), cudaMemcpyHostToDevice));
        GEMB_CUDA(cudaMemcpy(d->heavy_first, hfirst.data(), sizeof(int32_t) * hfirst.size(), cudaMemcpyHostToDevice));
        GEMB_CUDA(cudaMemcpy(d->item_row, irow.data(), sizeof(int32_t) * irow.size(), cudaMemcpyHostToDevice));
        GEMB_CUDA(cudaMemcpy(d->item_beg, ibeg.data(), sizeof(int32_t) * ibeg.size(), cudaMemcpyHostToDevice));
    }
    return GEMB_OK;
}

int gemb_graph_upload(gemb_ctx *c, int64_t n, int64_t row0, int64_t n_local, const int32_t *indptr,
                      const int32_t *indices, const float *data, const int32_t *indptr_t,
                      const int32_t *indices_t, const float *data_t, gemb_graph **out) {
    GEMB_ARG(c && out && indptr, "ctx/out/indptr");
    GEMB_ARG(n > 0 && n < (int64_t)2147483647, "n");
    GEMB_ARG(row0 >= 0 && n_local >= 0 && row0 + n_local <= n, "row range");
    GEMB_ARG(indices != nullptr || indptr[n_local] == 0, "indices");
    GEMB_CUDA(cudaSetDevice(c->device));
    gemb_graph *g = new gemb_graph();
    g->ctx = c;
    g->n = n;
    g->row0 = row0;
    g->n_local = n_local;
    g->n_shard = (n + c->nranks - 1) / c->nranks;
    g->n_pad = g->n_shard * c->nranks;
    if (c->nranks > 1) {
        // either this rank's row shard (HOPE) or the whole graph replicated on every rank (node2vec)
        g->replicated = (row0 == 0 && n_local == n);
        if (!g->replicated && (row0 != g->n_shard * c->rank || n_local > g->n_shard)) {
            set_error("multi-GPU upload must be rows [rank*ceil(n/P), ...) or the whole graph: got row0=%lld n_local=%lld",
                      (long long)row0, (long long)n_local);
            delete g;
            return GEMB_ERR_ARG;
        }
    } else {
        if (row0 != 0 || n_local != n) {
            set_error("single-GPU upload needs row0=0, n_local=n");
            delete g;
            return GEMB_ERR_ARG;
        }
    }
    int s = upload_csr(c, n, n_local, indptr, indices, data, &g->A);
    if (s != GEMB_OK) { gemb_graph_free(g); return s; }
    if (indptr_t) {
        s = upload_csr(c, n, n_local, indptr_t, indices_t, data_t, &g->AT);
        if (s != GEMB_OK) { gemb_graph_free(g); return s; }
        g->symmetric = false;
    } else {
        g->AT = g->A;
        g->symmetric = true;
    }
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) {
        set_error("graph upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        gemb_graph_free(g);
        return GEMB_ERR_CUDA;
    }
    *out = g;
    return GEMB_OK;
}

int gemb_graph_free(gemb_graph *g) {
    if (!g) return GEMB_OK;
    cudaSetDevice(g->ctx->device);
    gemb::halo_free(g);   // collective when a halo exchange was set up (every rank frees its shard)
    if (!g->symmetric) {
        dfree(g->AT.indptr);
        dfree(g->AT.indices);
        dfree(g->AT.data);
        dfree(g->AT.heavy_row); dfree(g->AT.heavy_first); dfree(g->AT.item_row); dfree(g->AT.item_beg);
    }
    dfree(g->A.indptr);
    dfree(g->A.indices);
    dfree(g->A.data);
    dfree(g->A.heavy_row); dfree(g->A.heavy_first); dfree(g->A.item_row); dfree(g->A.item_beg);
    delete g;
    return GEMB_OK;
}

}  // extern "C"
