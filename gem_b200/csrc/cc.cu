// gem_b200/csrc/cc.cu -- weakly connected components of a stored CSR and the extraction of the largest one
// (graph_util.py:29-34 get_lcc: max(weakly_connected_component_subgraphs(G), key=len), relabelled 0..k-1).
//
// Labelling (gemb_cc_create): union-find over integer atomics.  Every stored edge (u, v) joins u and v whatever its
// direction, so the out-CSR alone is enough.  parent[x] <= x holds at all times (a root is only ever hooked under a
// SMALLER root by atomicCAS), so every root ends as the smallest vertex id of its component and the labels do not
// depend on the order in which the atomics run: two runs give the same bits.  There is no host-driven convergence
// loop at all: one hooking pass, one flattening pass.  Reads of parent inside the loops are volatile, so a thread never
// spins on a stale value.
//
// Every find halves the path it walks (each node on it is pointed at its grandparent), in the hooking pass and in the
// flattening pass.  Without that, linking by index alone builds chains of depth Theta(n) on adversarial numberings
// (a path numbered h, h-1, h+1, h-2, h+2, ...), and walking them costs Theta(n^2) in total.  With halving, a sequential
// row-order emulation of both passes reads parent 6.8e6 + 3.1e6 times on that graph at n = 2^20, and the counts grow
// linearly in n.  That linear growth is a measurement of the sequential order; no bound is claimed for every
// concurrent schedule.  A halving store is a plain store of an ancestor (grandparent g < parent p < x keeps
// parent[x] <= x) into a node that is not a root, and atomicCAS only ever succeeds on a root, so the store never undoes
// a hook.  Two stores racing on one node both write ancestors of it, so either result is valid.
//
// Work is edge-balanced: a CTA takes a tile of CC_TILE consecutive stored edges and finds each edge's row by a binary
// search restricted to the rows the tile spans, so an R-MAT hub row of 10^5 edges is spread over many CTAs instead of
// one thread.
//
// Sizes are integer counters; the largest component (LCC) is the maximum of the 64-bit key (size << 32 | ~root): the
// largest size, the smallest root on a tie -- max(nx.weakly_connected_components(G), key=len) over row order, because
// networkx yields components in the order of their first node and max keeps the first maximal one.  Components are
// numbered 0..k-1 in the order of their smallest member (exclusive scan of the roots).
//
// Extraction (gemb_cc_lcc): new id = exclusive scan of LCC membership in row order.  The map is monotone, so every row
// keeps its column ids sorted; a weak component holds every edge of its rows, so no edge is filtered: the new indptr is
// the scan of the kept rows' degrees, and every output edge is gathered (edge-balanced again) with its column remapped
// and its fp64 weight copied.  No floating-point atomics anywhere.
#include "common.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <vector>

struct gemb_cc {
    gemb_ctx *ctx = nullptr;
    int64_t n = 0, nnz = 0;
    int64_t *indptr = nullptr;   // n + 1
    int32_t *indices = nullptr;  // nnz
    int32_t *labels = nullptr;   // n: component number, 0..n_comp-1 in the order of the smallest member
    int64_t n_comp = 0, lcc_root = -1, lcc_size = 0, lcc_nnz = 0;
    int32_t lcc_label = -1;
    double label_ms = 0.0, extract_ms = 0.0;
};

namespace gemb {

constexpr int CC_THREADS = 256, CC_PER_THREAD = 8, CC_TILE = CC_THREADS * CC_PER_THREAD;

// largest r in [lo, hi] with indptr[r] <= e  (the row of stored position e; indptr[lo] <= e is given)
__device__ __forceinline__ int64_t cc_row_of(const int64_t *__restrict__ indptr, int64_t lo, int64_t hi, int64_t e) {
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo + 1) / 2;
        if (indptr[mid] <= e) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// rows [*r0, *r1] hold the stored positions [t0, t1) of this CTA's tile (t0 < t1 <= indptr[n])
__device__ __forceinline__ void cc_tile_rows(const int64_t *__restrict__ indptr, int64_t n, int64_t t0, int64_t t1,
                                             int64_t *r0, int64_t *r1) {
    __shared__ int64_t rows[2];
    if (threadIdx.x == 0) rows[0] = cc_row_of(indptr, 0, n - 1, t0);
    if (threadIdx.x == 32) rows[1] = cc_row_of(indptr, 0, n - 1, t1 - 1);
    __syncthreads();
    *r0 = rows[0];
    *r1 = rows[1];
}

// root of x, halving the path on the way; every step moves to a strictly smaller id
__device__ __forceinline__ int cc_find(volatile int32_t *parent, int x) {
    int p = parent[x];
    while (p != x) {
        const int g = parent[p];
        if (g == p) return p;
        parent[x] = g;
        x = g;
        p = parent[x];
    }
    return x;
}

__global__ void cc_init_kernel(int64_t n, int32_t *__restrict__ parent) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        parent[i] = (int32_t)i;
}

// one CTA per tile of CC_TILE stored edges: hook the root of the larger id under the root of the smaller
__global__ void __launch_bounds__(CC_THREADS)
cc_hook_kernel(int64_t n, int64_t nnz, const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
               int32_t *parent) {
    const int64_t t0 = (int64_t)blockIdx.x * CC_TILE, t1 = min(t0 + CC_TILE, nnz);
    int64_t r0, r1;
    cc_tile_rows(indptr, n, t0, t1, &r0, &r1);
    volatile int32_t *vp = parent;
    for (int64_t e = t0 + threadIdx.x; e < t1; e += CC_THREADS) {
        const int u = (int)cc_row_of(indptr, r0, r1, e), v = indices[e];
        if (u == v) continue;
        int ru = cc_find(vp, u), rv = cc_find(vp, v);
        while (ru != rv) {
            // hook the larger root under the smaller; a failed CAS returns hi's new (smaller) parent: climb from there
            const int hi = max(ru, rv), lo = min(ru, rv);
            const int old = atomicCAS(&parent[hi], hi, lo);
            if (old == hi) break;
            ru = old;
            rv = lo;
        }
    }
}

// root[x] = root of x (no hooking runs concurrently, so the walk ends at the final root); is_root[x]; size[root]++.
// The roots go to their own array: the halving stores of other threads may still rewrite parent[x] with an ancestor.
__global__ void cc_flatten_kernel(int64_t n, int32_t *parent, int32_t *__restrict__ root, int32_t *__restrict__ is_root,
                                  uint32_t *__restrict__ size) {
    volatile int32_t *vp = parent;
    // whole warps step together (the stride is a multiple of 32), so the warp-wide match below sees every lane
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i - (threadIdx.x & 31) < n;
         i += (int64_t)gridDim.x * blockDim.x) {
        int r = -1;
        if (i < n) {
            r = cc_find(vp, (int)i);
            root[i] = r;
            is_root[i] = r == (int)i ? 1 : 0;
        }
        // one atomic per distinct root in the warp: the giant component would otherwise serialise on one counter
        const unsigned peers = __match_any_sync(0xffffffffu, r);
        if (r >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&size[r], (uint32_t)__popc(peers));
    }
}

// key = max over roots of (size << 32 | ~root): the largest component, the smallest root on a tie
__global__ void __launch_bounds__(CC_THREADS)
cc_lcc_key_kernel(int64_t n, const int32_t *__restrict__ is_root, const uint32_t *__restrict__ size,
                  unsigned long long *__restrict__ key) {
    unsigned long long best = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (is_root[i]) best = max(best, ((unsigned long long)size[i] << 32) | (unsigned long long)(~(uint32_t)i));
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    __shared__ unsigned long long part[CC_THREADS / 32];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < CC_THREADS / 32; w++) best = max(best, part[w]);
        atomicMax(key, best);
    }
}

__device__ __forceinline__ int32_t cc_key_root(unsigned long long key) { return (int32_t)~(uint32_t)key; }

// labels[x] = component number of x's root (in place over the roots); the LCC's stored edges counted into *lcc_nnz
__global__ void __launch_bounds__(CC_THREADS)
cc_relabel_kernel(int64_t n, const int64_t *__restrict__ indptr, const int32_t *__restrict__ comp_of_root,
                  const unsigned long long *__restrict__ key, int32_t *__restrict__ labels,
                  unsigned long long *__restrict__ lcc_nnz) {
    const int32_t root = cc_key_root(*key);
    unsigned long long edges = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = labels[i];
        if (r == root) edges += (unsigned long long)(indptr[i + 1] - indptr[i]);
        labels[i] = comp_of_root[r];
    }
    for (int o = 16; o > 0; o >>= 1) edges += __shfl_xor_sync(0xffffffffu, edges, o);
    if ((threadIdx.x & 31) == 0 && edges) atomicAdd(lcc_nnz, edges);
}

__global__ void cc_member_kernel(int64_t n, const int32_t *__restrict__ labels, int32_t lcc_label,
                                 int32_t *__restrict__ in_lcc) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
        in_lcc[i] = (i < n && labels[i] == lcc_label) ? 1 : 0;
}

// node_l[new] = old and the degree of every kept row at its new position
__global__ void cc_keep_rows_kernel(int64_t n, const int64_t *__restrict__ indptr, const int32_t *__restrict__ in_lcc,
                                    const int32_t *__restrict__ new_id, int64_t *__restrict__ node_l,
                                    int64_t *__restrict__ deg) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (in_lcc[i]) {
            node_l[new_id[i]] = i;
            deg[new_id[i]] = indptr[i + 1] - indptr[i];
        }
}

// one CTA per tile of CC_TILE output edges: row r of the LCC is row node_l[r] of the graph
__global__ void __launch_bounds__(CC_THREADS)
cc_gather_kernel(int64_t k, int64_t m, const int64_t *__restrict__ out_ptr, const int64_t *__restrict__ node_l,
                 const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                 const int32_t *__restrict__ new_id, const double *__restrict__ data, int32_t *__restrict__ out_idx,
                 double *__restrict__ out_data) {
    const int64_t t0 = (int64_t)blockIdx.x * CC_TILE, t1 = min(t0 + CC_TILE, m);
    int64_t r0, r1;
    cc_tile_rows(out_ptr, k, t0, t1, &r0, &r1);
    for (int64_t f = t0 + threadIdx.x; f < t1; f += CC_THREADS) {
        const int64_t r = cc_row_of(out_ptr, r0, r1, f);
        const int64_t e = indptr[node_l[r]] + (f - out_ptr[r]);
        out_idx[f] = new_id[indices[e]];
        if (data) out_data[f] = data[e];
    }
}

// out[0..count) = exclusive prefix sums of in[0..count)
template <class T>
static int cc_exclusive_sum(gemb_ctx *c, const T *in, T *out, int64_t count) {
    size_t tb = 0;
    GEMB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, count, c->stream));
    DeviceBuffer<unsigned char> tmp;
    GEMB_CUDA(tmp.alloc(tb));
    GEMB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb, in, out, count, c->stream));
    count_launch(2);   // CUB's tile-state initialisation and the scan
    return GEMB_OK;
}

}  // namespace gemb

using namespace gemb;

extern "C" {

int gemb_cc_create(gemb_ctx *c, int64_t n, const int64_t *indptr, const int32_t *indices, gemb_cc **out) {
    GEMB_ARG(c && out, "ctx/out");
    GEMB_ARG(n >= 0 && n < ((int64_t)1 << 31), "0 <= n < 2^31");
    GEMB_ARG(indptr, "indptr");
    GEMB_ARG(indptr[0] == 0, "indptr[0] == 0");
    for (int64_t i = 0; i < n; i++) GEMB_ARG(indptr[i + 1] >= indptr[i], "indptr non-decreasing");
    const int64_t nnz = indptr[n];
    GEMB_ARG(nnz == 0 || indices, "indices");
    bool bad = false;
    for (int64_t t = 0; t < nnz; t++) bad |= (uint32_t)indices[t] >= (uint64_t)n;
    GEMB_ARG(!bad, "column ids in [0, n)");
    GEMB_CUDA(cudaSetDevice(c->device));
    DeviceBuffer<int64_t> dptr;
    DeviceBuffer<int32_t> dix, parent, root, is_root, comp;
    DeviceBuffer<uint32_t> size;
    DeviceBuffer<unsigned long long> dred;   // [0] LCC key, [1] LCC stored edges
    CallEvents<2> ev;
    GEMB_CUDA(ev.create());
    cudaStream_t st = c->stream;
    GEMB_CUDA(dptr.upload(indptr, (size_t)n + 1, st));
    GEMB_CUDA(dix.upload(indices, (size_t)nnz, st));
    GEMB_CUDA(parent.alloc((size_t)std::max<int64_t>(n, 1)));
    GEMB_CUDA(root.alloc((size_t)std::max<int64_t>(n, 1)));
    GEMB_CUDA(is_root.alloc((size_t)n + 1));
    GEMB_CUDA(comp.alloc((size_t)n + 1));
    GEMB_CUDA(size.alloc((size_t)std::max<int64_t>(n, 1)));
    GEMB_CUDA(dred.alloc(2));
    unsigned long long red[2] = {0, 0};
    int32_t n_comp = 0;
    GEMB_CUDA(cudaEventRecord(ev[0], st));
    if (n) {
        GEMB_CUDA(cudaMemsetAsync(size.get(), 0, sizeof(uint32_t) * (size_t)n, st));
        GEMB_CUDA(cudaMemsetAsync(is_root.get() + n, 0, sizeof(int32_t), st));
        GEMB_CUDA(cudaMemsetAsync(dred.get(), 0, 2 * sizeof(unsigned long long), st));
        const int grid = grid_stride(c, n, CC_THREADS, 16);
        GEMB_TRY(launch(c, cc_init_kernel, grid, CC_THREADS, 0, n, parent.get()));
        if (nnz)
            GEMB_TRY(launch(c, cc_hook_kernel, (unsigned)((nnz + CC_TILE - 1) / CC_TILE), CC_THREADS, 0, n, nnz, dptr.get(),
                            dix.get(), parent.get()));
        GEMB_TRY(launch(c, cc_flatten_kernel, grid, CC_THREADS, 0, n, parent.get(), root.get(), is_root.get(), size.get()));
        GEMB_TRY(launch(c, cc_lcc_key_kernel, grid, CC_THREADS, 0, n, is_root.get(), size.get(), dred.get()));
        GEMB_TRY(cc_exclusive_sum(c, is_root.get(), comp.get(), n + 1));
        GEMB_TRY(launch(c, cc_relabel_kernel, grid, CC_THREADS, 0, n, dptr.get(), comp.get(), dred.get(), root.get(),
                        dred.get() + 1));
        GEMB_CUDA(cudaMemcpyAsync(red, dred.get(), sizeof(red), cudaMemcpyDeviceToHost, st));
        GEMB_CUDA(cudaMemcpyAsync(&n_comp, comp.get() + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    GEMB_CUDA(cudaEventRecord(ev[1], st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    const int64_t lcc_root = n ? (int64_t)(uint32_t)~(uint32_t)red[0] : -1;
    int32_t lcc_label = -1;   // the LCC's component number = the number of roots before its root
    if (n) GEMB_TRY(copy_sync(c, &lcc_label, comp.get() + lcc_root, sizeof(int32_t), cudaMemcpyDeviceToHost));
    gemb_cc *r = new gemb_cc();
    r->ctx = c; r->n = n; r->nnz = nnz;
    r->n_comp = n_comp;
    r->lcc_root = lcc_root;
    r->lcc_label = lcc_label;
    r->lcc_size = (int64_t)(red[0] >> 32);
    r->lcc_nnz = (int64_t)red[1];
    r->label_ms = ev.ms(0, 1);
    r->indptr = dptr.release();
    r->indices = dix.release();
    r->labels = root.release();
    *out = r;
    return GEMB_OK;
}

int gemb_cc_free(gemb_cc *r) {
    if (!r) return GEMB_OK;
    cudaSetDevice(r->ctx->device);
    dfree(r->indptr);
    dfree(r->indices);
    dfree(r->labels);
    delete r;
    return GEMB_OK;
}

int gemb_cc_info(gemb_cc *r, int64_t *n_comp, int64_t *lcc_root, int64_t *lcc_size, int64_t *lcc_nnz) {
    GEMB_ARG(r, "cc");
    if (n_comp) *n_comp = r->n_comp;
    if (lcc_root) *lcc_root = r->lcc_root;
    if (lcc_size) *lcc_size = r->lcc_size;
    if (lcc_nnz) *lcc_nnz = r->lcc_nnz;
    return GEMB_OK;
}

int gemb_cc_times(gemb_cc *r, double *label_ms, double *extract_ms) {
    GEMB_ARG(r, "cc");
    if (label_ms) *label_ms = r->label_ms;
    if (extract_ms) *extract_ms = r->extract_ms;
    return GEMB_OK;
}

int gemb_cc_labels(gemb_cc *r, int32_t *comp_out) {
    GEMB_ARG(r && (r->n == 0 || comp_out), "cc/comp_out");
    if (r->n == 0) return GEMB_OK;
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    return copy_sync(c, comp_out, r->labels, sizeof(int32_t) * (size_t)r->n, cudaMemcpyDeviceToHost);
}

int gemb_cc_lcc(gemb_cc *r, const double *data, int64_t *node_l_out, int64_t *indptr_out, int32_t *indices_out,
                double *data_out) {
    GEMB_ARG(r && indptr_out, "cc/indptr_out");
    const int64_t n = r->n, k = r->lcc_size, m = r->lcc_nnz;
    GEMB_ARG(k == 0 || node_l_out, "node_l_out");
    GEMB_ARG(m == 0 || indices_out, "indices_out");
    GEMB_ARG(!data || m == 0 || data_out, "data_out (weights given)");
    indptr_out[0] = 0;
    if (k == 0) return GEMB_OK;
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    cudaStream_t st = c->stream;
    DeviceBuffer<int32_t> in_lcc, new_id, oix;
    DeviceBuffer<int64_t> node_l, deg, optr;
    DeviceBuffer<double> ddata, odata;
    CallEvents<2> ev;
    GEMB_CUDA(ev.create());
    GEMB_CUDA(in_lcc.alloc((size_t)n + 1));
    GEMB_CUDA(new_id.alloc((size_t)n + 1));
    GEMB_CUDA(node_l.alloc((size_t)k));
    GEMB_CUDA(deg.alloc((size_t)k + 1));
    GEMB_CUDA(optr.alloc((size_t)k + 1));
    GEMB_CUDA(oix.alloc((size_t)std::max<int64_t>(m, 1)));
    const bool weighted = data && m;
    if (weighted) {
        GEMB_CUDA(ddata.upload(data, (size_t)r->nnz, st));
        GEMB_CUDA(odata.alloc((size_t)m));
    }
    GEMB_CUDA(cudaEventRecord(ev[0], st));
    GEMB_TRY(launch(c, cc_member_kernel, grid_stride(c, n + 1, CC_THREADS, 16), CC_THREADS, 0, n, r->labels, r->lcc_label,
                    in_lcc.get()));
    GEMB_TRY(cc_exclusive_sum(c, in_lcc.get(), new_id.get(), n + 1));
    GEMB_CUDA(cudaMemsetAsync(deg.get() + k, 0, sizeof(int64_t), st));
    GEMB_TRY(launch(c, cc_keep_rows_kernel, grid_stride(c, n, CC_THREADS, 16), CC_THREADS, 0, n, r->indptr, in_lcc.get(),
                    new_id.get(), node_l.get(), deg.get()));
    GEMB_TRY(cc_exclusive_sum(c, deg.get(), optr.get(), k + 1));
    if (m)
        GEMB_TRY(launch(c, cc_gather_kernel, (unsigned)((m + CC_TILE - 1) / CC_TILE), CC_THREADS, 0, k, m, optr.get(),
                        node_l.get(), r->indptr, r->indices, new_id.get(), weighted ? ddata.get() : nullptr, oix.get(),
                        odata.get()));
    GEMB_CUDA(cudaEventRecord(ev[1], st));
    GEMB_CUDA(cudaMemcpyAsync(node_l_out, node_l.get(), sizeof(int64_t) * (size_t)k, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(indptr_out, optr.get(), sizeof(int64_t) * (size_t)(k + 1), cudaMemcpyDeviceToHost, st));
    if (m) GEMB_CUDA(cudaMemcpyAsync(indices_out, oix.get(), sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, st));
    if (weighted)
        GEMB_CUDA(cudaMemcpyAsync(data_out, odata.get(), sizeof(double) * (size_t)m, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    r->extract_ms = ev.ms(0, 1);
    return GEMB_OK;
}

}  // extern "C"
