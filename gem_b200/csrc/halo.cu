// gem_b200/csrc/halo.cu -- multi-GPU HOPE without a per-sweep collective (replaces the ncclAllGather of the whole
// n x b block in front of every SpMM that round 1 used; the reference itself is single-process, SURVEY 2.2).
//
// Row-sharded symmetric A, one process per GPU.  At set-up every rank works out
//   * H_p: the sorted distinct REMOTE columns its CSR shard references (the "halo"; an SBM shard at P = 8 needs
//     ~2.75 M of the 7 M remote rows, an all-gather delivers all 7 M), and a second copy of the column ids in which a
//     local column c becomes c - row0 and a remote one n_shard + (its position in H_p);
//   * from the all-gathered H_q: for each of its own rows the list of (peer q, slot in H_q) that reference it.
// Work blocks are laid out [n_shard local rows | halo rows] and every rank maps every peer's blocks and barrier flags
// with CUDA IPC.  The kernel that produces a block writes each local row into the peers' halo slots with plain 16-byte
// stores over NVLink (posted writes: fire-and-forget, they overlap the producer's own gathers and FMAs tile by tile),
// a flag barrier closes the sweep, and the next SpMM gathers from local HBM only.
#include "common.cuh"
#include "nccl_api.h"
#include <cub/cub.cuh>
#include <algorithm>
#include <vector>

namespace gemb {

#define NCCL_TRY(call, what)                                                                   \
    do {                                                                                       \
        ncclResult_t _r = (call);                                                              \
        if (_r != ncclSuccess) { set_error("%s: %s", what, api->GetErrorString(_r)); return GEMB_ERR_NCCL; } \
    } while (0)

struct IsRemote {
    int32_t lo, hi;   // local columns are [lo, hi)
    __host__ __device__ bool operator()(const int32_t &c) const { return c < lo || c >= hi; }
};

__device__ __forceinline__ int64_t lower_bound_i32(const int32_t *a, int64_t n, int32_t x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t m = (lo + hi) >> 1;
        if (a[m] < x) lo = m + 1; else hi = m;
    }
    return lo;
}

__global__ void halo_remap_kernel(int64_t nnz, const int32_t *__restrict__ idx, int32_t lo, int32_t hi,
                                  const int32_t *__restrict__ H, int64_t nH, int32_t n_shard,
                                  int32_t *__restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nnz; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t c = idx[i];
        out[i] = (c >= lo && c < hi) ? c - lo : n_shard + (int32_t)lower_bound_i32(H, nH, c);
    }
}

// seg[2q], seg[2q+1]: the slots of H_q that hold rows of [lo, hi)
__global__ void halo_segments_kernel(int nranks, const int32_t *__restrict__ Hall, int64_t maxH,
                                     const long long *__restrict__ counts, int32_t lo, int32_t hi,
                                     long long *__restrict__ seg) {
    const int q = threadIdx.x;
    if (q >= nranks) return;
    const int32_t *H = Hall + (int64_t)q * maxH;
    seg[2 * q] = lower_bound_i32(H, counts[q], lo);
    seg[2 * q + 1] = lower_bound_i32(H, counts[q], hi);
}

// pass 0: cnt[row]++ ; pass 1: push_dst[push_ptr[row] + cursor[row]++] = (q << 29) | slot
template <int PASS>
__global__ void halo_pushlist_kernel(int q, const int32_t *__restrict__ H, long long s0, long long s1, int32_t row0,
                                     int32_t *__restrict__ cnt, const int32_t *__restrict__ push_ptr,
                                     uint32_t *__restrict__ push_dst) {
    for (long long t = s0 + (long long)blockIdx.x * blockDim.x + threadIdx.x; t < s1; t += (long long)gridDim.x * blockDim.x) {
        const int32_t row = H[t] - row0;
        const int pos = atomicAdd(cnt + row, 1);
        if (PASS == 1) push_dst[push_ptr[row] + pos] = ((uint32_t)q << 29) | (uint32_t)t;
    }
}

static int ipc_exchange(gemb_ctx *c, void *const *mine, int count, void **peers /* [count][GEMB_MAX_RANKS] */) {
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    const int P = c->nranks;
    std::vector<cudaIpcMemHandle_t> h(count), all((size_t)count * P);
    for (int i = 0; i < count; i++) GEMB_CUDA(cudaIpcGetMemHandle(&h[i], mine[i]));
    DeviceBuffer<char> dsend, drecv;
    const size_t bytes = sizeof(cudaIpcMemHandle_t) * count;
    GEMB_CUDA(dsend.upload((const char *)h.data(), bytes, c->stream));
    GEMB_CUDA(drecv.alloc(bytes * P));
    NCCL_TRY(api->AllGather(dsend.get(), drecv.get(), bytes, ncclChar, (ncclComm_t)c->comm, c->stream), "ncclAllGather(ipc handles)");
    GEMB_TRY(copy_sync(c, all.data(), drecv.get(), bytes * P, cudaMemcpyDeviceToHost));
    dsend.reset(); drecv.reset();
    for (int i = 0; i < count; i++)
        for (int q = 0; q < P; q++) {
            void **slot = peers + (size_t)i * GEMB_MAX_RANKS + q;
            if (q == c->rank) { *slot = mine[i]; continue; }
            cudaError_t e = cudaIpcOpenMemHandle(slot, all[(size_t)q * count + i], cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                (void)cudaGetLastError();
                set_error("cudaIpcOpenMemHandle (rank %d -> rank %d): %s", c->rank, q, cudaGetErrorString(e));
                return GEMB_ERR_CUDA;
            }
        }
    return GEMB_OK;
}

static int nccl_barrier(gemb_ctx *c) {
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    DeviceBuffer<int> d;
    GEMB_CUDA(d.alloc(1));
    GEMB_CUDA(cudaMemsetAsync(d.get(), 0, sizeof(int), c->stream));
    NCCL_TRY(api->AllReduce(d.get(), d.get(), 1, ncclInt, ncclSum, (ncclComm_t)c->comm, c->stream), "ncclAllReduce(barrier)");
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

// the exchange plan of halo_build (indices_ext, push_ptr, push_dst, halo_rows, push_total); its scratch is released
// when it returns
static int halo_plan(gemb_graph *g, NcclApi *api) {
    gemb_halo &H = g->halo;
    gemb_ctx *c = g->ctx;
    const int P = c->nranks;
    const int64_t nnz = g->A.nnz;
    const int32_t lo = (int32_t)g->row0, hi = (int32_t)std::min<int64_t>(g->row0 + g->n_shard, g->n);
    cudaStream_t st = c->stream;

    // ---- distinct remote columns, sorted
    DeviceBuffer<int32_t> rem, rem_sorted, Hd;
    DeviceBuffer<long long> d_num;
    GEMB_CUDA(rem.alloc(std::max<int64_t>(nnz, 1)));
    GEMB_CUDA(rem_sorted.alloc(std::max<int64_t>(nnz, 1)));
    GEMB_CUDA(Hd.alloc(std::max<int64_t>(nnz, 1)));
    GEMB_CUDA(d_num.alloc(2 * GEMB_MAX_RANKS + 2));
    size_t tb = 0, need = 0;
    DeviceBuffer<char> tmp;
    IsRemote pred{lo, hi};
    cub::DeviceSelect::If(nullptr, need, g->A.indices, rem.get(), d_num.get(), nnz, pred, st); tb = need;
    cub::DeviceRadixSort::SortKeys(nullptr, need, rem.get(), rem_sorted.get(), nnz, 0, 32, st); tb = std::max(tb, need);
    cub::DeviceSelect::Unique(nullptr, need, rem_sorted.get(), Hd.get(), d_num.get(), nnz, st); tb = std::max(tb, need);
    GEMB_CUDA(tmp.alloc(tb));
    long long n_rem = 0, n_H = 0;
    if (nnz > 0) {
        GEMB_CUDA(cub::DeviceSelect::If(tmp.get(), tb, g->A.indices, rem.get(), d_num.get(), nnz, pred, st));
        GEMB_TRY(copy_sync(c, &n_rem, d_num.get(), sizeof n_rem, cudaMemcpyDeviceToHost));
        if (n_rem > 0) {
            GEMB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.get(), tb, rem.get(), rem_sorted.get(), n_rem, 0, 32, st));
            GEMB_CUDA(cub::DeviceSelect::Unique(tmp.get(), tb, rem_sorted.get(), Hd.get(), d_num.get(), n_rem, st));
            GEMB_TRY(copy_sync(c, &n_H, d_num.get(), sizeof n_H, cudaMemcpyDeviceToHost));
        }
    }
    count_launch(3);
    H.halo_rows = n_H;
    GEMB_ARG(n_H < ((int64_t)1 << 29), "halo too large for 29-bit slots");

    // ---- remapped column ids
    GEMB_CUDA(dmalloc(&H.indices_ext, sizeof(int32_t) * (std::max<int64_t>(nnz, 1) + 4)));   // + the x4 padding the bulk copies of spmm.cu read
    if (nnz > 0)
        GEMB_TRY(launch(c, halo_remap_kernel, c->sm_count * 8, 256, 0, nnz, g->A.indices, lo, hi, Hd.get(), n_H, (int32_t)g->n_shard,
                        H.indices_ext));

    // ---- everyone's halo lists -> who needs my rows
    long long *d_cnt_all = d_num.get() + 2;                 // [P]
    long long h_cnt_all[GEMB_MAX_RANKS];
    GEMB_CUDA(cudaMemcpyAsync(d_num.get(), &n_H, sizeof n_H, cudaMemcpyHostToDevice, st));
    NCCL_TRY(api->AllGather(d_num.get(), d_cnt_all, 1, ncclInt64, (ncclComm_t)c->comm, st), "ncclAllGather(halo counts)");
    GEMB_TRY(copy_sync(c, h_cnt_all, d_cnt_all, sizeof(long long) * P, cudaMemcpyDeviceToHost));
    long long maxH = 1;
    for (int q = 0; q < P; q++) maxH = std::max(maxH, h_cnt_all[q]);
    DeviceBuffer<int32_t> Hpad, Hall;
    GEMB_CUDA(Hpad.alloc(maxH));
    GEMB_CUDA(Hall.alloc(maxH * P));
    GEMB_CUDA(cudaMemsetAsync(Hpad.get(), 0x7f, sizeof(int32_t) * maxH, st));
    if (n_H) GEMB_CUDA(cudaMemcpyAsync(Hpad.get(), Hd.get(), sizeof(int32_t) * n_H, cudaMemcpyDeviceToDevice, st));
    NCCL_TRY(api->AllGather(Hpad.get(), Hall.get(), (size_t)maxH, ncclInt32, (ncclComm_t)c->comm, st), "ncclAllGather(halo lists)");
    DeviceBuffer<long long> seg_dev;
    GEMB_CUDA(seg_dev.alloc(2 * GEMB_MAX_RANKS));
    GEMB_TRY(launch(c, halo_segments_kernel, 1, 32, 0, P, Hall.get(), maxH, d_cnt_all, lo, hi, seg_dev.get()));
    long long seg[2 * GEMB_MAX_RANKS];
    GEMB_TRY(copy_sync(c, seg, seg_dev.get(), sizeof(long long) * 2 * P, cudaMemcpyDeviceToHost));

    DeviceBuffer<int32_t> cnt;
    const int64_t nl = g->n_local;
    GEMB_CUDA(cnt.alloc(nl + 1));
    GEMB_CUDA(dmalloc(&H.push_ptr, sizeof(int32_t) * (nl + 1)));
    GEMB_CUDA(cudaMemsetAsync(cnt.get(), 0, sizeof(int32_t) * (nl + 1), st));
    long long total = 0;
    for (int q = 0; q < P; q++) {
        if (q == c->rank) continue;
        const long long m = seg[2 * q + 1] - seg[2 * q];
        total += m;
        if (m <= 0) continue;
        GEMB_TRY(launch(c, halo_pushlist_kernel<0>, grid_stride(c, m, 256, 8), 256, 0, q, Hall.get() + (int64_t)q * maxH, seg[2 * q],
                        seg[2 * q + 1], lo, cnt.get(), nullptr, nullptr));
    }
    GEMB_ARG(total < ((long long)1 << 31), "push list too long");
    H.push_total = total;
    size_t sb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, sb, cnt.get(), H.push_ptr, (int)(nl + 1), st);
    DeviceBuffer<char> stmp;
    GEMB_CUDA(stmp.alloc(sb));
    GEMB_CUDA(cub::DeviceScan::ExclusiveSum(stmp.get(), sb, cnt.get(), H.push_ptr, (int)(nl + 1), st));
    GEMB_CUDA(cudaMemsetAsync(cnt.get(), 0, sizeof(int32_t) * (nl + 1), st));
    GEMB_CUDA(dmalloc(&H.push_dst, sizeof(uint32_t) * std::max<long long>(total, 1)));
    for (int q = 0; q < P; q++) {
        if (q == c->rank) continue;
        const long long m = seg[2 * q + 1] - seg[2 * q];
        if (m <= 0) continue;
        GEMB_TRY(launch(c, halo_pushlist_kernel<1>, grid_stride(c, m, 256, 8), 256, 0, q, Hall.get() + (int64_t)q * maxH, seg[2 * q],
                        seg[2 * q + 1], lo, cnt.get(), H.push_ptr, H.push_dst));
    }
    GEMB_CUDA(cudaStreamSynchronize(st));
    return GEMB_OK;
}

int halo_build(gemb_graph *g) {
    gemb_halo &H = g->halo;
    if (H.ready) return GEMB_OK;
    gemb_ctx *c = g->ctx;
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    GEMB_ARG(c->nranks > 1 && c->nranks <= GEMB_MAX_RANKS, "halo exchange supports 2..8 ranks");
    GEMB_ARG(g->symmetric && !g->replicated, "halo exchange needs a symmetric row shard");
    GEMB_ARG(g->n_shard + 1 < (int64_t)1 << 29, "shard too large for 29-bit halo slots");
    const int P = c->nranks;
    GEMB_TRY(halo_plan(g, api));

    // ---- barrier flags: owned by the context (plain cudaMalloc: exported through CUDA IPC, never recycled by the block
    //      cache), set up once and shared by every graph of this context
    gemb_halo_pool &PL = c->halo_pool;
    if (!PL.flags) {
        GEMB_CUDA(cudaMalloc(&PL.flags, sizeof(unsigned long long) * GEMB_MAX_RANKS));
        GEMB_CUDA(cudaMemset(PL.flags, 0, sizeof(unsigned long long) * GEMB_MAX_RANKS));
        GEMB_CUDA(cudaMalloc(&PL.timeout_flag, sizeof(int)));
        GEMB_CUDA(cudaMemset(PL.timeout_flag, 0, sizeof(int)));
        void *mine[1] = {PL.flags};
        void *peers[GEMB_MAX_RANKS] = {};
        GEMB_TRY(ipc_exchange(c, mine, 1, peers));
        for (int q = 0; q < P; q++) PL.peer_flags[q] = (unsigned long long *)peers[q];
        PL.epoch = 0;
    }
    H.flags = PL.flags;
    H.timeout_flag = PL.timeout_flag;
    for (int q = 0; q < P; q++) H.peer_flags[q] = PL.peer_flags[q];
    H.ready = true;
    return GEMB_OK;
}

// collective: every rank drops its mappings of the peers' blocks, then frees its own
static int halo_pool_drop_blocks(gemb_ctx *c) {
    gemb_halo_pool &PL = c->halo_pool;
    if (PL.nbuf == 0) return GEMB_OK;
    cudaStreamSynchronize(c->stream);
    for (int i = 0; i < PL.nbuf; i++)
        for (int q = 0; q < c->nranks; q++)
            if (q != c->rank && PL.peer_buf[i][q]) { cudaIpcCloseMemHandle(PL.peer_buf[i][q]); PL.peer_buf[i][q] = nullptr; }
    GEMB_TRY(nccl_barrier(c));     // nobody still maps what is freed next
    for (int i = 0; i < PL.nbuf; i++) { cudaFree(PL.buf[i]); PL.buf[i] = nullptr; }
    PL.nbuf = 0; PL.cap_floats = 0;
    return GEMB_OK;
}

int halo_buffers(gemb_graph *g, int nbuf, int width) {
    gemb_halo &H = g->halo;
    gemb_ctx *c = g->ctx;
    gemb_halo_pool &PL = c->halo_pool;
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    GEMB_ARG(H.ready && nbuf >= 1 && nbuf <= GEMB_HALO_BUFS, "halo_buffers");
    const size_t rows = (size_t)(g->n_shard + H.halo_rows);
    // the pool is (re)built only when some rank needs more than it holds: the decision comes from an all-reduce (max)
    // of the need, so every rank takes the same branch
    long long need = (long long)(rows * (size_t)width);
    DeviceBuffer<long long> d_need;
    GEMB_CUDA(d_need.upload(&need, 1, c->stream));
    NCCL_TRY(api->AllReduce(d_need.get(), d_need.get(), 1, ncclInt64, ncclMax, (ncclComm_t)c->comm, c->stream), "ncclAllReduce(halo block size)");
    GEMB_TRY(copy_sync(c, &need, d_need.get(), sizeof need, cudaMemcpyDeviceToHost));
    d_need.reset();
    if (PL.nbuf < nbuf || PL.cap_floats < (size_t)need) {
        GEMB_TRY(halo_pool_drop_blocks(c));
        const size_t cap = (size_t)std::max<long long>(need, 1);
        void *mine[GEMB_HALO_BUFS];
        for (int i = 0; i < nbuf; i++) {
            cudaError_t e = cudaMalloc(&PL.buf[i], sizeof(float) * cap);
            if (e != cudaSuccess) {
                (void)cudaGetLastError();
                gemb_mem_trim();
                e = cudaMalloc(&PL.buf[i], sizeof(float) * cap);
            }
            GEMB_CUDA(e);
            mine[i] = PL.buf[i];
        }
        void *peers[GEMB_HALO_BUFS * GEMB_MAX_RANKS] = {};
        PL.nbuf = nbuf; PL.cap_floats = cap;
        GEMB_TRY(ipc_exchange(c, mine, nbuf, peers));
        for (int i = 0; i < nbuf; i++)
            for (int q = 0; q < c->nranks; q++) PL.peer_buf[i][q] = (float *)peers[(size_t)i * GEMB_MAX_RANKS + q];
    } else {
        // blocks of the previous call are being reused: no rank may still be pushing into them
        GEMB_TRY(nccl_barrier(c));
    }
    for (int i = 0; i < nbuf; i++) {
        GEMB_CUDA(cudaMemsetAsync(PL.buf[i], 0, sizeof(float) * rows * width, c->stream));
        H.buf[i] = PL.buf[i];
        for (int q = 0; q < c->nranks; q++) H.peer_buf[i][q] = PL.peer_buf[i][q];
    }
    H.nbuf = nbuf; H.width = width;
    // the zero fill must be complete everywhere before any peer's first push can land
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    GEMB_TRY(nccl_barrier(c));
    return GEMB_OK;
}

void halo_push_args(const gemb_graph *g, int bi, HaloPushArgs *out) {
    const gemb_halo &H = g->halo;
    out->push_ptr = H.push_ptr;
    out->push_dst = H.push_dst;
    for (int q = 0; q < GEMB_MAX_RANKS; q++) out->peer[q] = (float4 *)H.peer_buf[bi][q];
    out->halo_row0 = g->n_shard;
}

// group of G threads per local row: copy the row into every peer slot that references it
__global__ void __launch_bounds__(256)
halo_push_kernel(int64_t n_rows, int G, int rows_per_cta, const float4 *__restrict__ Y, HaloPushArgs P) {
    const int lr = threadIdx.x / G, c = threadIdx.x - lr * G;
    if (lr >= rows_per_cta) return;
    const int64_t row = (int64_t)blockIdx.x * rows_per_cta + lr;
    if (row >= n_rows) return;
    if (P.push_ptr[row] == P.push_ptr[row + 1]) return;
    halo_push_row(P, row, G, c, Y[row * G + c]);
}

int halo_push_launch(gemb_graph *g, int bi, int width) {
    gemb_ctx *c = g->ctx;
    if (g->n_local == 0 || g->halo.push_total == 0) return GEMB_OK;
    const int G = width / 4;
    GEMB_ARG(G >= 1 && G <= 256, "width");
    const int rpc = 256 / G;
    HaloPushArgs P;
    halo_push_args(g, bi, &P);
    return launch(c, halo_push_kernel, (unsigned)((g->n_local + rpc - 1) / rpc), 256, 0, g->n_local, G, rpc,
                  (const float4 *)g->halo.buf[bi], P);
}

struct BarrierArgs {
    unsigned long long *peer[GEMB_MAX_RANKS];
};

// One warp: lane q posts this rank's epoch into peer q's flag word, then waits for peer q's.  Stream order puts this
// kernel after the producer kernel, whose (peer) stores are performed before the kernel completes; the fences keep the
// flag behind them.  The wait is bounded (~2 s): a lost rank must surface as an error, never as a hung GPU.
__global__ void halo_barrier_kernel(BarrierArgs A, volatile unsigned long long *mine, unsigned long long epoch, int rank,
                                    int nranks, int *timeout_flag) {
    const int q = threadIdx.x;
    if (q >= nranks || q == rank) return;
    __threadfence_system();
    *(volatile unsigned long long *)(A.peer[q] + rank) = epoch;
    __threadfence_system();
    const long long t0 = clock64();
    while (mine[q] < epoch) {
        if (clock64() - t0 > 4000000000LL) { atomicExch(timeout_flag, 1); break; }
        __nanosleep(100);
    }
    __threadfence_system();
}

int halo_barrier(gemb_graph *g) {
    gemb_halo &H = g->halo;
    gemb_ctx *c = g->ctx;
    BarrierArgs A;
    for (int q = 0; q < GEMB_MAX_RANKS; q++) A.peer[q] = H.peer_flags[q];
    c->halo_pool.epoch++;
    return launch(c, halo_barrier_kernel, 1, 32, 0, A, H.flags, c->halo_pool.epoch, c->rank, c->nranks, H.timeout_flag);
}

int halo_check_timeout(gemb_graph *g) {
    gemb_halo &H = g->halo;
    if (!H.ready) return GEMB_OK;
    int h = 0;
    GEMB_TRY(copy_sync(g->ctx, &h, H.timeout_flag, sizeof h, cudaMemcpyDeviceToHost));
    if (h) {
        set_error("multi-GPU HOPE: a peer did not reach the sweep barrier within 2 s (rank %d of %d)", g->ctx->rank, g->ctx->nranks);
        return GEMB_ERR_NCCL;
    }
    return GEMB_OK;
}

int halo_free(gemb_graph *g) {
    gemb_halo &H = g->halo;
    if (!H.ready) return GEMB_OK;
    cudaStreamSynchronize(g->ctx->stream);
    dfree(H.indices_ext); dfree(H.push_ptr); dfree(H.push_dst);     // the plan; blocks and flags belong to the context
    H = gemb_halo();
    return GEMB_OK;
}

// context destruction: not collective (the peers may already be gone); a peer that still maps these blocks keeps its
// mapping valid until it closes it or exits
void halo_pool_release(gemb_ctx *c) {
    gemb_halo_pool &PL = c->halo_pool;
    cudaStreamSynchronize(c->stream);
    for (int i = 0; i < PL.nbuf; i++)
        for (int q = 0; q < c->nranks; q++)
            if (q != c->rank && PL.peer_buf[i][q]) cudaIpcCloseMemHandle(PL.peer_buf[i][q]);
    for (int q = 0; q < c->nranks; q++)
        if (q != c->rank && PL.peer_flags[q]) cudaIpcCloseMemHandle(PL.peer_flags[q]);
    for (int i = 0; i < PL.nbuf; i++) cudaFree(PL.buf[i]);
    cudaFree(PL.flags); cudaFree(PL.timeout_flag);
    (void)cudaGetLastError();
    PL = gemb_halo_pool();
}

}  // namespace gemb
