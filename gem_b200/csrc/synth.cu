// gem_b200/csrc/synth.cu -- Graph500 R-MAT generator on the device (bench infrastructure for BASELINE.json configs[3]
// and configs[4]: R-MAT scale 24 = 16.7M nodes / 268M directed edges).  The host generator (gem_b200/synth.py::rmat,
// NumPy) needs minutes and ~20 GB of host memory per rank at that scale; this one produces the same KIND of graph
// (edge_factor * 2^scale undirected pairs from the (a, b, c, d) recursion, vertices relabelled by a random permutation,
// symmetrised, self loops and duplicates removed, unit weights, sorted column ids) in well under a second, and hands
// back only the row shard the caller asks for.  Counter-based RNG (splitmix64 of seed, pair index, level): every rank
// of a multi-GPU run generates the identical graph without communicating.  No reference counterpart (GEM ships no
// generator; the reference tests load fixed fixtures).
#include "common.cuh"
#include <cub/cub.cuh>
#include <algorithm>

namespace gemb {

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

__global__ void rmat_perm_keys_kernel(int64_t n, uint64_t seed, uint64_t *__restrict__ key, int32_t *__restrict__ val) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        key[i] = splitmix64(seed ^ (0xA5A5A5A5ull << 32) ^ (uint64_t)i * 0xD1B54A32D192ED03ull);
        val[i] = (int32_t)i;
    }
}

// pair e -> (u, v) by `scale` levels of the quadrant recursion; both directions as 64-bit keys (row << 32 | col);
// a self loop becomes the all-ones sentinel (sorted to the end, removed by the caller)
__global__ void rmat_pairs_kernel(int64_t m, int scale, uint32_t ta, uint32_t tab, uint32_t tabc, uint64_t seed,
                                  const int32_t *__restrict__ perm, uint64_t *__restrict__ keys) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < m; e += (int64_t)gridDim.x * blockDim.x) {
        uint32_t u = 0, v = 0;
        uint64_t h = 0;
        for (int l = 0; l < scale; l++) {
            if ((l & 1) == 0) h = splitmix64(seed + (uint64_t)e * 0x9E3779B97F4A7C15ull + (uint64_t)(l >> 1) * 0xC2B2AE3D27D4EB4Full);
            const uint32_t r = (l & 1) ? (uint32_t)(h >> 32) : (uint32_t)h;
            const uint32_t ubit = r >= tab;                                  // quadrants c, d
            const uint32_t vbit = ((r >= ta) & (r < tab)) | (r >= tabc);     // quadrants b, d
            u = (u << 1) | ubit;
            v = (v << 1) | vbit;
        }
        if (perm) { u = (uint32_t)perm[u]; v = (uint32_t)perm[v]; }
        if (u == v) { keys[2 * e] = ~0ull; keys[2 * e + 1] = ~0ull; }
        else { keys[2 * e] = ((uint64_t)u << 32) | v; keys[2 * e + 1] = ((uint64_t)v << 32) | u; }
    }
}

__device__ __forceinline__ int64_t lower_bound_u64(const uint64_t *a, int64_t n, uint64_t x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// indptr[r] = (first key of row row0 + r) - (first key of row row0), r = 0 .. n_rows
__global__ void rmat_rowptr_kernel(int64_t n_rows, int64_t row0, const uint64_t *__restrict__ keys, int64_t nkeys,
                                   int64_t *__restrict__ indptr, int64_t *__restrict__ first) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n_rows; r += (int64_t)gridDim.x * blockDim.x) {
        const int64_t p = lower_bound_u64(keys, nkeys, (uint64_t)(row0 + r) << 32);
        indptr[r] = p;
        if (r == 0) *first = p;
    }
}
__global__ void rmat_rebase_kernel(int64_t n_rows, int64_t *__restrict__ indptr, const int64_t *__restrict__ first) {
    const int64_t f = *first;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n_rows; r += (int64_t)gridDim.x * blockDim.x) indptr[r] -= f;
}
__global__ void rmat_cols_kernel(int64_t cnt, const uint64_t *__restrict__ keys, int32_t *__restrict__ cols) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += (int64_t)gridDim.x * blockDim.x)
        cols[i] = (int32_t)(uint32_t)keys[i];
}

// gemb_synth_rmat without the argument checks and the final trim: its scratch is released when it returns
static int rmat_generate(gemb_ctx *ctx, int scale, int edge_factor, double a, double b, double c, uint64_t seed, int permute,
                         int64_t row0, int64_t n_rows, int64_t *nnz_out, int64_t *nnz_total_out, int64_t *indptr_out,
                         int32_t *indices_out, int64_t cap) {
    const int64_t n = (int64_t)1 << scale, m = n * edge_factor, nk = 2 * m;
    cudaStream_t st = ctx->stream;
    const int grid = ctx->sm_count * 8;
    DeviceBuffer<uint64_t> pk, pk2, keys, keys2;
    DeviceBuffer<int32_t> pv, perm, cols;
    DeviceBuffer<int64_t> d_ip, d_cnt;
    DeviceBuffer<char> tmp;
    size_t tb = 0, need = 0;
    if (permute) {
        GEMB_CUDA(pk.alloc(n)); GEMB_CUDA(pk2.alloc(n));
        GEMB_CUDA(pv.alloc(n)); GEMB_CUDA(perm.alloc(n));
        cub::DeviceRadixSort::SortPairs(nullptr, need, pk.get(), pk2.get(), pv.get(), perm.get(), n, 0, 64, st); tb = std::max(tb, need);
    }
    GEMB_CUDA(keys.alloc(nk)); GEMB_CUDA(keys2.alloc(nk));
    GEMB_CUDA(d_cnt.alloc(2));
    cub::DeviceRadixSort::SortKeys(nullptr, need, keys.get(), keys2.get(), nk, 0, 64, st); tb = std::max(tb, need);
    cub::DeviceSelect::Unique(nullptr, need, keys2.get(), keys.get(), d_cnt.get(), nk, st); tb = std::max(tb, need);
    GEMB_CUDA(tmp.alloc(tb));
    if (permute) {
        GEMB_TRY(launch(ctx, rmat_perm_keys_kernel, grid, 256, 0, n, seed, pk.get(), pv.get()));
        GEMB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tb, pk.get(), pk2.get(), pv.get(), perm.get(), n, 0, 64, st));
        count_launch();
    }
    const uint32_t ta = (uint32_t)std::min(4294967295.0, a * 4294967296.0);
    const uint32_t tab = (uint32_t)std::min(4294967295.0, (a + b) * 4294967296.0);
    const uint32_t tabc = (uint32_t)std::min(4294967295.0, (a + b + c) * 4294967296.0);
    GEMB_TRY(launch(ctx, rmat_pairs_kernel, grid, 256, 0, m, scale, ta, tab, tabc, seed, permute ? perm.get() : nullptr, keys.get()));
    GEMB_CUDA(cub::DeviceRadixSort::SortKeys(tmp.get(), tb, keys.get(), keys2.get(), nk, 0, 64, st));
    GEMB_CUDA(cub::DeviceSelect::Unique(tmp.get(), tb, keys2.get(), keys.get(), d_cnt.get(), nk, st));
    count_launch(2);
    int64_t nu = 0;
    GEMB_TRY(copy_sync(ctx, &nu, d_cnt.get(), 8, cudaMemcpyDeviceToHost));
    uint64_t last = 0;
    if (nu > 0) {
        GEMB_TRY(copy_sync(ctx, &last, keys.get() + (nu - 1), 8, cudaMemcpyDeviceToHost));
        if (last == ~0ull) nu--;                                   // the self-loop sentinel
    }
    if (nnz_total_out) *nnz_total_out = nu;
    GEMB_CUDA(d_ip.alloc(n_rows + 1));
    GEMB_TRY(launch(ctx, rmat_rowptr_kernel, grid, 256, 0, n_rows, row0, keys.get(), nu, d_ip.get(), d_cnt.get() + 1));
    int64_t ends[2] = {0, 0};
    GEMB_CUDA(cudaMemcpyAsync(&ends[0], d_ip.get(), 8, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(&ends[1], d_ip.get() + n_rows, 8, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    const int64_t cnt = ends[1] - ends[0];
    if (nnz_out) *nnz_out = cnt;
    if (!indices_out) return GEMB_OK;
    GEMB_ARG(indptr_out && cap >= cnt, "indptr_out / cap");
    GEMB_TRY(launch(ctx, rmat_rebase_kernel, grid, 256, 0, n_rows, d_ip.get(), d_cnt.get() + 1));
    GEMB_CUDA(cols.alloc(std::max<int64_t>(cnt, 1)));
    GEMB_TRY(launch(ctx, rmat_cols_kernel, grid, 256, 0, cnt, keys.get() + ends[0], cols.get()));
    GEMB_CUDA(cudaMemcpyAsync(indptr_out, d_ip.get(), 8 * (size_t)(n_rows + 1), cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(indices_out, cols.get(), 4 * (size_t)cnt, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    return GEMB_OK;
}

}  // namespace gemb

using namespace gemb;

// Rows [row0, row0 + n_rows) of the graph (n_rows < 0: all rows).  Call 1: indices_out = NULL -> *nnz_out = nonzeros of
// the shard, *nnz_total_out = nonzeros of the whole graph.  Call 2: indptr_out (n_rows + 1 int64, shard-local offsets)
// and indices_out (cap >= nnz int32, global column ids) are filled.  Both calls regenerate (0.2 s at scale 24).
extern "C" int gemb_synth_rmat(gemb_ctx *ctx, int scale, int edge_factor, double a, double b, double c, uint64_t seed,
                               int permute, int64_t row0, int64_t n_rows, int64_t *nnz_out, int64_t *nnz_total_out,
                               int64_t *indptr_out, int32_t *indices_out, int64_t cap) {
    GEMB_ARG(ctx, "ctx");
    GEMB_ARG(scale >= 1 && scale <= 30 && edge_factor >= 1, "scale / edge_factor");
    GEMB_ARG(a > 0 && b >= 0 && c >= 0 && a + b + c < 1.0, "quadrant probabilities");
    const int64_t n = (int64_t)1 << scale;
    if (n_rows < 0) { row0 = 0; n_rows = n; }
    GEMB_ARG(row0 >= 0 && row0 + n_rows <= n, "row range");
    GEMB_CUDA(cudaSetDevice(ctx->device));
    const int status = rmat_generate(ctx, scale, edge_factor, a, b, c, seed, permute, row0, n_rows, nnz_out, nnz_total_out,
                                     indptr_out, indices_out, cap);
    gemb_mem_trim();            // ~7 GB of generator scratch at scale 24: give it back before the solver allocates
    return status;
}
