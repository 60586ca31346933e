// gem_b200/csrc/recon.cu -- graph reconstruction from an embedding and the counting kernels of its evaluation
// (SURVEY 8(f) rank 1: the step right after learn_embedding in every reference test, tests/fit_model.py:10).
//
//   reference                                                         here
//   static_graph_embedding.py:48-65  A_hat[i][j] = get_edge_weight    gemb_recon_create: A_hat = L R^T on the device,
//     (n^2 Python calls of hope.py:43-44 / node2vec.py:56-57)           64-column panels through the wgmma 3xTF32
//                                                                       kernel of apply_tc.cu (CUDA-core tile kernel
//                                                                       when the shape does not fit), diagonal zeroed
//   evaluation_util.py:20-36   scan adj for entries > 0               never materialised on the host: the kernels
//   metrics.py:28-46  computeMAP: per node, sort its predicted          below COUNT instead of sorting --
//     edges by weight, precision at every true edge                     rank(e) = 1 + #{j' : a[i][j'] > a[i][j_e] or
//                                                                       (== and j' < j_e)}  (stable descending order)
//   metrics.py:6-25   computePrecisionCurve: global sort              threshold of the K-th best entry by bisection
//                                                                       on the float bit pattern (one counting pass
//                                                                       per bit), then one compaction pass
//   evaluate_graph_reconstruction.py:37-40  weighted error            gemb_recon_pairs gathers a[i][j] of the edges
//
// Layout: A_hat is n x n_pad fp32, n_pad = 64 * ceil(n / 64), PANEL-major: element (i, j) at
// ((j / 64) * n + i) * 64 + j % 64 -- each 64-column panel is the contiguous n x 64 output of one apply launch
// (ldo = 64: the rows of one panel are adjacent).  Padded columns hold 0.
// Roofline: HBM writes of 4 n^2 bytes for the product (k = 64: 32 flop per byte written, far below the tensor
// pipe), HBM reads of 4 n^2 bytes per counting pass.
//
// Gaussian kind (LaplacianEigenmaps / LocallyLinearEmbedding, lap.py:39-42, lle.py:37-40: exp(-|x_i - x_j|^2)):
// the panels hold an ORDER KEY instead of the score, key = bits 0x7f800000 - bits(delta) with delta = |x_i - x_j|^2
// (0 when delta > 745.1332f, the last fp32 delta whose fp64 exp(-delta) is > 0).  The key is a positive float that
// orders exactly as the score does, so the counting kernels below run on it unchanged; fp32 exp(-delta) would merge
// distinct distances.  delta is summed in the difference form (recon_sqdist_kernel): exact 0 for equal rows.
//
// Link prediction (evaluation_util.py:39-53 splits the graph; the held-out edges are ranked among the candidates that
// are not training edges): gemb_recon_exclude keeps the panel offsets of the training edges.  An entry that holds 0
// is not a candidate in any counting kernel (nor, for the Gaussian kind, key 0), so ranks and top run unchanged on
// the panels with those entries set to 0: recon_swap_kernel zeroes them and keeps their values for the length of
// the call, and puts them back before it returns (dense and pairs always see the unmasked values).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

struct gemb_recon {
    gemb_ctx *ctx = nullptr;
    int64_t n = 0, n_pad = 0;
    int k = 0;
    int kind = 0;             // GEMB_RECON_DOT, _SPLIT or _GAUSS
    float *adj = nullptr;     // n x n_pad, panel-major
    // gemb_recon_top cache (the bisection is 31 passes; the caller asks for the count first, then the entries)
    int top_valid = 0, top_und = 0;
    int64_t top_k = 0, top_count = 0;
    uint32_t top_bits = 0;
    // exclusion (gemb_recon_exclude): ex_nnz distinct panel offsets, and their values while a ranks / top call has
    // them masked (0 between calls); nullptr = none
    int64_t *ex_off = nullptr;
    float *ex_saved = nullptr;
    int64_t ex_nnz = 0;
};

namespace gemb {

constexpr int PW = 64;   // panel width

__host__ __device__ __forceinline__ size_t adj_index(int64_t i, int64_t j, int64_t n) {
    return ((size_t)(j >> 6) * (size_t)n + (size_t)i) * PW + (size_t)(j & 63);
}

// L[i][c] = X[i][c], c < k  (left factor, contiguous)
__global__ void recon_left_kernel(int64_t n, int d, int k, const float *__restrict__ X, float *__restrict__ L) {
    const int64_t total = n * k;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = idx / k;
        const int c = (int)(idx - i * k);
        L[idx] = X[i * d + c];
    }
}

// Rt[c][j] = X[j][off + c] for j < n, 0 for the padding  (right factor transposed: the M operand of the panels)
__global__ void recon_right_t_kernel(int64_t n, int64_t n_pad, int d, int k, int off, const float *__restrict__ X,
                                     float *__restrict__ Rt) {
    __shared__ float tile[32][33];
    const int64_t j0 = (int64_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int64_t j = j0 + r;
        const int c = c0 + threadIdx.x;
        tile[r][threadIdx.x] = (j < n && c < k) ? X[j * d + off + c] : 0.f;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += blockDim.y) {
        const int c = c0 + r;
        const int64_t j = j0 + threadIdx.x;
        if (c < k && j < n_pad) Rt[(size_t)c * n_pad + j] = tile[threadIdx.x][r];
    }
}

__global__ void recon_zero_diag_kernel(int64_t n, float *__restrict__ adj) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        adj[adj_index(i, i, n)] = 0.f;
}

// row-major copy of rows [r0, r0 + rows): out[(i - r0) * n + j]
__global__ void recon_rowmajor_kernel(int64_t n, int64_t r0, int64_t rows, const float *__restrict__ adj,
                                      float *__restrict__ out) {
    const int64_t total = rows * n;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t ii = idx / n, j = idx - ii * n;
        out[idx] = adj[adj_index(r0 + ii, j, n)];
    }
}

__global__ void recon_pairs_kernel(int64_t n, int64_t m, const int32_t *__restrict__ pi, const int32_t *__restrict__ pj,
                                   const float *__restrict__ adj, float *__restrict__ out) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = pi[t], j = pj[t];
        out[t] = (i == j) ? 0.f : adj[adj_index(i, j, n)];
    }
}

// One warp per row i.  Edge e = (i -> j_e) of the true graph is in the predicted list iff j_e != i, (undirected:
// j_e > i) and a[i][j_e] > 0; its 1-based position in the list sorted by weight (descending, stable in j) is
// 1 + #{valid j' : a[i][j'] > a_e  or  (a[i][j'] == a_e and j' < j_e)}.  rank_out[e] = that position or 0.
__global__ void __launch_bounds__(256)
recon_rank_kernel(int64_t n, const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                  int undirected, const float *__restrict__ adj, int32_t *__restrict__ rank_out,
                  int32_t *__restrict__ n_pred_row) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        const int64_t lo = undirected ? i + 1 : 0;
        const int e_begin = indptr[i], e_end = indptr[i + 1];
        const int nchunks = e_end > e_begin ? (e_end - e_begin + 31) / 32 : 1;   // chunk 0 also counts the row
        for (int ch = 0; ch < nchunks; ch++) {
            const int e = e_begin + ch * 32 + lane;
            long long je = -1;
            float se = -1.f;
            if (e < e_end) {
                je = indices[e];
                if (je != i && je >= lo) {
                    const float v = adj[adj_index(i, je, n)];
                    if (v > 0.f) se = v;
                }
            }
            const bool any_valid = __any_sync(0xffffffffu, se > 0.f);
            int mine = 0;
            if (any_valid || ch == 0) {
                int cnt[32];
#pragma unroll
                for (int t = 0; t < 32; t++) cnt[t] = 0;
                int npred = 0;
                for (int64_t j0 = lo & ~(int64_t)31; j0 < n; j0 += 32) {
                    const int64_t jj = j0 + lane;
                    float v = 0.f;
                    if (jj >= lo && jj < n && jj != i) v = adj[adj_index(i, jj, n)];
                    const bool pos = v > 0.f;
                    npred += pos ? 1 : 0;
                    if (any_valid) {
#pragma unroll
                        for (int t = 0; t < 32; t++) {
                            const float st = __shfl_sync(0xffffffffu, se, t);
                            const long long jt = __shfl_sync(0xffffffffu, je, t);
                            cnt[t] += (pos && (v > st || (v == st && (long long)jj < jt))) ? 1 : 0;
                        }
                    }
                }
                if (ch == 0) {
                    for (int o = 16; o > 0; o >>= 1) npred += __shfl_xor_sync(0xffffffffu, npred, o);
                    if (lane == 0) n_pred_row[i] = npred;
                }
                if (any_valid) {
#pragma unroll
                    for (int t = 0; t < 32; t++) {
                        int c = cnt[t];
                        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
                        if (lane == t) mine = c;
                    }
                }
            }
            if (e < e_end) rank_out[e] = se > 0.f ? mine + 1 : 0;
        }
    }
}

// count (and optionally collect) the valid entries whose bit pattern is >= bits (positive floats order like uints)
template <bool COLLECT>
__global__ void __launch_bounds__(256)
recon_select_kernel(int64_t n, int64_t n_panels, int undirected, uint32_t bits, const float *__restrict__ adj,
                    unsigned long long *__restrict__ counter, int64_t cap, int32_t *__restrict__ oi,
                    int32_t *__restrict__ oj, float *__restrict__ ow) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t segs = n_panels * n;       // segment = 64 consecutive floats: panel p, row i
    unsigned long long local = 0;
    for (int64_t s = warp; s < segs; s += nwarps) {
        const int64_t p = s / n, i = s - p * n;
        if (undirected && p * PW + PW - 1 <= i) continue;      // every column of the panel is <= i
        const float *seg = adj + (size_t)s * PW;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int64_t j = p * PW + h * 32 + lane;
            const float v = seg[h * 32 + lane];
            const bool valid = j < n && j != i && (!undirected || j > i) && v > 0.f && __float_as_uint(v) >= bits;
            if (COLLECT) {
                const unsigned mask = __ballot_sync(0xffffffffu, valid);
                if (mask) {
                    unsigned long long base = 0;
                    if (lane == 0) base = atomicAdd(counter, (unsigned long long)__popc(mask));
                    base = __shfl_sync(0xffffffffu, base, 0);
                    if (valid) {
                        const int64_t slot = (int64_t)base + __popc(mask & ((1u << lane) - 1u));
                        if (slot < cap) { oi[slot] = (int32_t)i; oj[slot] = (int32_t)j; ow[slot] = v; }
                    }
                }
            } else {
                local += valid ? 1ull : 0ull;
            }
        }
    }
    if (!COLLECT) {
        for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
        if (lane == 0 && local) atomicAdd(counter, local);
    }
}

// ---- Gaussian kind
constexpr uint32_t GAUSS_KEY_ONE = 0x7f800000u;      // key of delta = 0: +inf
constexpr uint32_t GAUSS_DELTA_MAX = 0x443a4886u;    // 745.1332f: fp64 exp(-delta) > 0 up to here, 0.0 above

__device__ __forceinline__ float gauss_key(float delta) {
    const uint32_t b = __float_as_uint(delta);       // delta >= 0 (or +inf), so its bits order like the value
    return b <= GAUSS_DELTA_MAX ? __uint_as_float(GAUSS_KEY_ONE - b) : 0.f;
}

constexpr int SQD_ROWS = 128, SQD_KC = 16, SQD_THREADS = 256;   // 16 x 16 threads, 8 rows x 4 columns each

// One launch over every (128-row x 64-column) tile, tile t = panel (t / row_tiles), row tile (t % row_tiles): the row
// tiles of one panel run next to each other and share its 64 column vectors in L2.  The rows and the panel's
// columns are staged k-major in shared memory, SQD_KC coordinates at a time; each thread keeps an 8 x 4 tile of
// sum_k (x_ik - x_jk)^2 (FADD + FFMA per term, fp32) and its 16 threads of a row write the whole 256-byte panel row.
// Diagonal and padded columns get key 0.
__global__ void __launch_bounds__(SQD_THREADS)
recon_sqdist_kernel(int64_t n, int d, int64_t row_tiles, const float *__restrict__ X, float *__restrict__ adj) {
    __shared__ __align__(16) float xr[SQD_KC][SQD_ROWS + 4];
    __shared__ __align__(16) float xc[SQD_KC][PW + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t p = (int64_t)blockIdx.x / row_tiles;
    const int64_t i0 = ((int64_t)blockIdx.x - p * row_tiles) * SQD_ROWS, j0 = p * PW;
    float acc[8][4];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) acc[r][c] = 0.f;
    for (int k0 = 0; k0 < d; k0 += SQD_KC) {
        const int kc = min(SQD_KC, d - k0);
        for (int idx = tid; idx < SQD_ROWS * SQD_KC; idx += SQD_THREADS) {
            const int kk = idx % SQD_KC, r = idx / SQD_KC;
            const int64_t i = i0 + r;
            xr[kk][r] = (i < n && kk < kc) ? X[i * d + k0 + kk] : 0.f;
        }
        for (int idx = tid; idx < PW * SQD_KC; idx += SQD_THREADS) {
            const int kk = idx % SQD_KC, c = idx / SQD_KC;
            const int64_t j = j0 + c;
            xc[kk][c] = (j < n && kk < kc) ? X[j * d + k0 + kk] : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int kk = 0; kk < kc; kk++) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&xr[kk][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&xr[kk][ty * 8 + 4]);
            const float4 b4 = *reinterpret_cast<const float4 *>(&xc[kk][tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const float t = a[r] - b[c];
                    acc[r][c] = fmaf(t, t, acc[r][c]);
                }
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const int64_t i = i0 + ty * 8 + r;
        if (i >= n) break;
        float v[4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const int64_t j = j0 + tx * 4 + c;
            v[c] = (j < n && j != i) ? gauss_key(acc[r][c]) : 0.f;
        }
        *reinterpret_cast<float4 *>(adj + ((size_t)p * (size_t)n + (size_t)i) * PW + tx * 4) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// key -> delta in place (key 0: the diagonal, padding or an underflowed score -> +inf, so exp(-delta) = 0 there too)
__global__ void recon_key_to_delta_kernel(int64_t m, float *__restrict__ w) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = __float_as_uint(w[t]);
        w[t] = b ? __uint_as_float(GAUSS_KEY_ONE - b) : __uint_as_float(GAUSS_KEY_ONE);
    }
}

// ---- exclusion (link prediction)
// adj[off[t]] <-> saved[t]: with saved all 0 the first launch masks the excluded entries, the second restores them.
// The offsets are distinct, so no two threads touch one entry.
__global__ void recon_swap_kernel(int64_t m, const int64_t *__restrict__ off, float *__restrict__ saved,
                                  float *__restrict__ adj) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const float v = adj[off[t]];
        adj[off[t]] = saved[t];
        saved[t] = v;
    }
}

static int count_ge(gemb_recon *r, int undirected, uint32_t bits, unsigned long long *dcounter, int64_t *out) {
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaMemsetAsync(dcounter, 0, sizeof(unsigned long long), c->stream));
    const int64_t n_panels = r->n_pad / PW;
    GEMB_TRY(launch(c, recon_select_kernel<false>, grid_stride(c, n_panels * r->n * 32, 256, 16), 256, 0, r->n, n_panels,
                    undirected, bits, r->adj, dcounter, 0, nullptr, nullptr, nullptr));
    unsigned long long h = 0;
    GEMB_TRY(copy_sync(c, &h, dcounter, sizeof h, cudaMemcpyDeviceToHost));
    *out = (int64_t)h;
    return GEMB_OK;
}

// Gaussian kind: turn the m keys at w (device) into delta before they are copied out; a no-op for the other kinds
static int decode_out(const gemb_recon *r, int64_t m, float *w) {
    if (r->kind != GEMB_RECON_GAUSS || m == 0) return GEMB_OK;
    return launch(r->ctx, recon_key_to_delta_kernel, grid_stride(r->ctx, m, 256, 16), 256, 0, m, w);
}

static int swap_excluded(gemb_recon *r) {
    const int64_t m = r->ex_nnz;
    if (m == 0) return GEMB_OK;
    return launch(r->ctx, recon_swap_kernel, grid_stride(r->ctx, m, 256, 16), 256, 0, m, r->ex_off, r->ex_saved, r->adj);
}

// run body() on the panels with the excluded entries set to 0, and restore them whatever body() returns; the first
// error wins.  Without an exclusion, body() alone.
template <class F> static int with_exclusion_masked(gemb_recon *r, F body) {
    GEMB_TRY(swap_excluded(r));
    const int st = body();
    const int st_restore = swap_excluded(r);
    return st != GEMB_OK ? st : st_restore;
}

}  // namespace gemb

using namespace gemb;

extern "C" {

static int recon_create_gauss(gemb_ctx *c, const float *X, int64_t n, int d, int64_t n_pad, float *adj) {
    DeviceBuffer<float> dX;
    GEMB_CUDA(dX.upload(X, (size_t)n * d, c->stream));
    const int64_t row_tiles = (n + SQD_ROWS - 1) / SQD_ROWS;
    GEMB_TRY(launch(c, recon_sqdist_kernel, (unsigned)(row_tiles * (n_pad / PW)), SQD_THREADS, 0, n, d, row_tiles, dX.get(), adj));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

int gemb_recon_create(gemb_ctx *c, const float *X, int64_t n, int d, int kind, gemb_recon **out) {
    GEMB_ARG(c && X && out, "ctx/X/out");
    GEMB_ARG(n > 0 && n < ((int64_t)1 << 31), "n");
    if (kind != GEMB_RECON_DOT && kind != GEMB_RECON_GAUSS) kind = GEMB_RECON_SPLIT;
    const bool split = kind == GEMB_RECON_SPLIT;
    GEMB_ARG(d > 0 && (!split || d % 2 == 0), "d (even when split)");
    if (kind == GEMB_RECON_GAUSS) {
        const size_t total = (size_t)n * (size_t)d;
        for (size_t t = 0; t < total; t++)
            GEMB_ARG(std::isfinite(X[t]), "X finite (a NaN or infinite distance has no place in the order)");
    }
    GEMB_CUDA(cudaSetDevice(c->device));
    const int k = split ? d / 2 : d;
    const int64_t n_pad = (n + PW - 1) / PW * PW;
    size_t free_b = 0, total_b = 0;
    GEMB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const double factors = kind == GEMB_RECON_GAUSS ? 0.0 : 8.0 * (double)n_pad * k;   // L and Rt
    const double need = 4.0 * (double)n * (double)n_pad + 4.0 * (double)n * d + factors;
    if (need > 0.9 * ((double)free_b + (double)gemb_mem_cached_bytes())) {
        set_error("gemb_recon_create: the %lld x %lld reconstruction needs %.1f GB of device memory, %.1f GB free "
                  "(evaluate a node sample instead, as evaluate_graph_reconstruction.py does at scale)",
                  (long long)n, (long long)n, need / 1e9, (double)free_b / 1e9);
        return GEMB_ERR_NOMEM;
    }
    if (kind == GEMB_RECON_GAUSS) {
        DeviceBuffer<float> adj;
        GEMB_CUDA(adj.alloc((size_t)n * n_pad));
        GEMB_TRY(recon_create_gauss(c, X, n, d, n_pad, adj.get()));
        gemb_recon *r = new gemb_recon();
        r->ctx = c; r->n = n; r->n_pad = n_pad; r->k = d; r->kind = kind;
        r->adj = adj.release();
        *out = r;
        return GEMB_OK;
    }
    DeviceBuffer<float> dX, L, Rt, adj;
    GEMB_CUDA(dX.upload(X, (size_t)n * d, c->stream));
    GEMB_CUDA(Rt.alloc((size_t)n_pad * k));
    GEMB_CUDA(adj.alloc((size_t)n * n_pad));
    const float *Lp = dX.get();
    if (split) {
        GEMB_CUDA(L.alloc((size_t)n * k));
        GEMB_TRY(launch(c, recon_left_kernel, grid_stride(c, n * k, 256, 16), 256, 0, n, d, k, dX.get(), L.get()));
        Lp = L.get();
    }
    GEMB_TRY(launch(c, recon_right_t_kernel, dim3((unsigned)((n_pad + 31) / 32), (unsigned)((k + 31) / 32)), dim3(32, 8), 0, n,
                    n_pad, d, k, split ? k : 0, dX.get(), Rt.get()));
    for (int64_t p = 0; p < n_pad / PW; p++)
        GEMB_TRY(apply_launch(c, n, Lp, k, Rt.get() + p * PW, (int)n_pad, PW, adj.get() + (size_t)p * n * PW, PW));
    GEMB_TRY(launch(c, recon_zero_diag_kernel, grid_stride(c, n, 256, 16), 256, 0, n, adj.get()));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    gemb_recon *r = new gemb_recon();
    r->ctx = c; r->n = n; r->n_pad = n_pad; r->k = k; r->kind = kind;
    r->adj = adj.release();
    *out = r;
    return GEMB_OK;
}

int gemb_recon_free(gemb_recon *r) {
    if (!r) return GEMB_OK;
    cudaSetDevice(r->ctx->device);
    dfree(r->adj);
    dfree(r->ex_off);
    dfree(r->ex_saved);
    delete r;
    return GEMB_OK;
}

int gemb_recon_dense(gemb_recon *r, float *adj_out) {
    GEMB_ARG(r && adj_out, "recon/out");
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    const int64_t n = r->n;
    int64_t rows = std::max<int64_t>(1, std::min<int64_t>(n, ((int64_t)256 << 20) / (4 * n)));   // <= 256 MB chunks
    DeviceBuffer<float> buf;
    GEMB_CUDA(buf.alloc((size_t)rows * n));
    for (int64_t r0 = 0; r0 < n; r0 += rows) {
        const int64_t nr = std::min(rows, n - r0);
        GEMB_TRY(launch(c, recon_rowmajor_kernel, grid_stride(c, nr * n, 256, 16), 256, 0, n, r0, nr, r->adj, buf.get()));
        GEMB_TRY(decode_out(r, nr * n, buf.get()));
        GEMB_TRY(copy_sync(c, adj_out + (size_t)r0 * n, buf.get(), sizeof(float) * (size_t)nr * n, cudaMemcpyDeviceToHost));
    }
    return GEMB_OK;
}

int gemb_recon_pairs(gemb_recon *r, const int32_t *pi, const int32_t *pj, int64_t m, float *out) {
    GEMB_ARG(r && (m == 0 || (pi && pj && out)), "recon/pairs/out");
    if (m == 0) return GEMB_OK;
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    for (int64_t t = 0; t < m; t++)
        GEMB_ARG(pi[t] >= 0 && pi[t] < r->n && pj[t] >= 0 && pj[t] < r->n, "pair index out of range");
    DeviceBuffer<int32_t> di, dj;
    DeviceBuffer<float> dout;
    GEMB_CUDA(di.upload(pi, (size_t)m, c->stream));
    GEMB_CUDA(dj.upload(pj, (size_t)m, c->stream));
    GEMB_CUDA(dout.alloc((size_t)m));
    GEMB_TRY(launch(c, recon_pairs_kernel, grid_stride(c, m, 256, 16), 256, 0, r->n, m, di.get(), dj.get(), r->adj, dout.get()));
    GEMB_TRY(decode_out(r, m, dout.get()));
    return copy_sync(c, out, dout.get(), sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost);
}

int gemb_recon_ranks(gemb_recon *r, const int32_t *indptr, const int32_t *indices, int is_undirected,
                     int32_t *rank_out, int32_t *n_pred_row) {
    GEMB_ARG(r && indptr && n_pred_row, "recon/indptr/n_pred_row");
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    const int64_t n = r->n;
    const int64_t nnz = indptr[n];
    GEMB_ARG(indptr[0] == 0 && nnz >= 0 && (nnz == 0 || (indices && rank_out)), "CSR");
    for (int64_t t = 0; t < nnz; t++) GEMB_ARG(indices[t] >= 0 && indices[t] < n, "column id out of range");
    return with_exclusion_masked(r, [&]() -> int {
        DeviceBuffer<int32_t> dp, dix, drank, dnp;
        GEMB_CUDA(dp.upload(indptr, (size_t)(n + 1), c->stream));
        GEMB_CUDA(dix.upload(indices, (size_t)nnz, c->stream));
        GEMB_CUDA(drank.alloc((size_t)std::max<int64_t>(nnz, 1)));
        GEMB_CUDA(dnp.alloc((size_t)n));
        GEMB_TRY(launch(c, recon_rank_kernel, grid_stride(c, n * 32, 256, 16), 256, 0, n, dp.get(), dix.get(), is_undirected ? 1 : 0,
                        r->adj, drank.get(), dnp.get()));
        if (nnz) GEMB_CUDA(cudaMemcpyAsync(rank_out, drank.get(), sizeof(int32_t) * (size_t)nnz, cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaMemcpyAsync(n_pred_row, dnp.get(), sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaStreamSynchronize(c->stream));
        return GEMB_OK;
    });
}

int gemb_recon_exclude(gemb_recon *r, const int32_t *ex_indptr, const int32_t *ex_indices) {
    GEMB_ARG(r, "recon");
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    const int64_t n = r->n;
    std::vector<int64_t> off;
    if (ex_indptr) {
        const int64_t nnz = ex_indptr[n];
        GEMB_ARG(ex_indptr[0] == 0 && nnz >= 0 && (nnz == 0 || ex_indices), "exclusion CSR");
        off.reserve((size_t)nnz);
        for (int64_t i = 0; i < n; i++) {
            GEMB_ARG(ex_indptr[i + 1] >= ex_indptr[i], "exclusion offsets non-decreasing");
            for (int64_t t = ex_indptr[i]; t < ex_indptr[i + 1]; t++) {
                GEMB_ARG(ex_indices[t] >= 0 && ex_indices[t] < n, "exclusion column id out of range");
                GEMB_ARG(t == ex_indptr[i] || ex_indices[t] > ex_indices[t - 1], "exclusion columns strictly ascending");
                off.push_back((int64_t)adj_index(i, ex_indices[t], n));
            }
        }
    }
    dfree(r->ex_off);
    dfree(r->ex_saved);
    r->ex_off = nullptr;
    r->ex_saved = nullptr;
    r->ex_nnz = 0;
    r->top_valid = 0;
    if (off.empty()) return GEMB_OK;
    DeviceBuffer<int64_t> doff;
    DeviceBuffer<float> dsaved;
    GEMB_CUDA(doff.upload(off.data(), off.size(), c->stream));
    GEMB_CUDA(dsaved.alloc(off.size()));
    GEMB_CUDA(cudaMemsetAsync(dsaved.get(), 0, sizeof(float) * off.size(), c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    r->ex_off = doff.release();
    r->ex_saved = dsaved.release();
    r->ex_nnz = (int64_t)off.size();
    return GEMB_OK;
}

int gemb_recon_top(gemb_recon *r, int is_undirected, int64_t max_k, int64_t cap, int32_t *i_out, int32_t *j_out,
                   float *w_out, int64_t *m_out) {
    GEMB_ARG(r && m_out, "recon/m_out");
    GEMB_ARG(cap == 0 || (i_out && j_out && w_out), "output arrays");
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    const int und = is_undirected ? 1 : 0;
    return with_exclusion_masked(r, [&]() -> int {
        DeviceBuffer<unsigned long long> dcounter;
        GEMB_CUDA(dcounter.alloc(1));
        if (!(r->top_valid && r->top_und == und && r->top_k == max_k)) {
            int64_t total = 0;
            GEMB_TRY(count_ge(r, und, 1u, dcounter.get(), &total));
            uint32_t bits = 1u;
            int64_t count = total;
            if (max_k >= 0 && total > max_k) {
                // largest bit pattern T with count(>= T) >= max_k:  count(>= lo) >= K  and  count(>= hi) < K
                uint32_t lo = 1u, hi = 0x7f800001u;
                while (hi - lo > 1u) {
                    const uint32_t mid = lo + (hi - lo) / 2u;
                    int64_t cm = 0;
                    GEMB_TRY(count_ge(r, und, mid, dcounter.get(), &cm));
                    if (cm >= std::max<int64_t>(max_k, 1)) { lo = mid; count = cm; } else { hi = mid; }
                }
                bits = lo;
                if (max_k == 0) count = 0;
            }
            r->top_valid = 1; r->top_und = und; r->top_k = max_k; r->top_bits = bits; r->top_count = count;
        }
        *m_out = r->top_count;
        if (cap <= 0 || r->top_count <= 0) return GEMB_OK;
        if (cap < r->top_count) {
            set_error("gemb_recon_top: %lld entries reach the threshold, cap is %lld", (long long)r->top_count, (long long)cap);
            return GEMB_ERR_ARG;
        }
        const int64_t m = r->top_count;
        DeviceBuffer<int32_t> di, dj;
        DeviceBuffer<float> dw;
        GEMB_CUDA(di.alloc((size_t)m));
        GEMB_CUDA(dj.alloc((size_t)m));
        GEMB_CUDA(dw.alloc((size_t)m));
        GEMB_CUDA(cudaMemsetAsync(dcounter.get(), 0, sizeof(unsigned long long), c->stream));
        const int64_t n_panels = r->n_pad / PW;
        GEMB_TRY(launch(c, recon_select_kernel<true>, grid_stride(c, n_panels * r->n * 32, 256, 16), 256, 0, r->n, n_panels, und,
                        r->top_bits, r->adj, dcounter.get(), m, di.get(), dj.get(), dw.get()));
        GEMB_TRY(decode_out(r, m, dw.get()));
        GEMB_CUDA(cudaMemcpyAsync(i_out, di.get(), sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaMemcpyAsync(j_out, dj.get(), sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaMemcpyAsync(w_out, dw.get(), sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaStreamSynchronize(c->stream));
        return GEMB_OK;
    });
}

}  // extern "C"
