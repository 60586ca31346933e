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
//   metrics.py:6-25   computePrecisionCurve: global sort              threshold of the K-th best entry by a radix
//                                                                       select on the float bit pattern (two histogram
//                                                                       passes), then one compaction pass
//   evaluate_graph_reconstruction.py:37-40  weighted error            gemb_recon_pairs gathers a[i][j] of the edges
//
// Layout: A_hat is n x n_pad fp32, n_pad = 64 * ceil(n / 64), PANEL-major: element (i, j) at
// ((j / 64) * n + i) * 64 + j % 64 -- each 64-column panel is the contiguous n x 64 output of one apply launch
// (ldo = 64: the rows of one panel are adjacent).  Padded columns hold 0.
// Roofline: HBM writes of 4 n^2 bytes for the product (k = 64: 32 flop per byte written, far below the tensor
// pipe), HBM reads of 4 n^2 bytes per counting pass.
//
// Blocks: a BLOCK is a run of ppb consecutive panels, contiguous in that layout, produced by exactly the launches that
// produce those panels of the whole matrix (same n, so the same kernel choice and the same bits).  When every panel
// fits in device memory the handle holds one block, made at create and kept.  Otherwise it keeps the factors and one
// block buffer, and every call regenerates the blocks in order (a PASS) and lets each consumer add up its part over
// them: ranks (a gather pass of the true edges' scores, then a counting pass), top (one or two histogram passes for the
// count, one compaction pass for the entries), pairs (the blocks that hold a pair), dense (every block).  Blocks are
// column runs, not row runs: a row block would need one apply launch per (block, panel).
//
// Gaussian kind (LaplacianEigenmaps / LocallyLinearEmbedding, lap.py:39-42, lle.py:37-40: exp(-|x_i - x_j|^2)):
// the panels hold an ORDER KEY instead of the score, key = bits 0x7f800000 - bits(delta) with delta = |x_i - x_j|^2
// (0 when delta > 745.1332f, the last fp32 delta whose fp64 exp(-delta) is > 0).  The key is a positive float that
// orders exactly as the score does, so the counting kernels below run on it unchanged; fp32 exp(-delta) would merge
// distinct distances.  delta is summed in the difference form (recon_sqdist_kernel): exact 0 for equal rows.
//
// Link prediction (evaluation_util.py:39-53 splits the graph; the held-out edges are ranked among the candidates that
// are not training edges): gemb_recon_exclude keeps the offsets of the training edges grouped by block, relative to
// the block.  An entry that holds 0 is not a candidate in any counting kernel (nor, for the Gaussian kind, key 0), so
// ranks and top run unchanged on each block with those entries set to 0: recon_swap_kernel zeroes them and keeps
// their values while the block is counted, and puts them back after (dense and pairs always see the unmasked values).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

struct gemb_recon {
    gemb_ctx *ctx = nullptr;
    int64_t n = 0, n_pad = 0;
    int d = 0, k = 0;
    int kind = 0;             // GEMB_RECON_DOT, _SPLIT or _GAUSS
    int64_t n_panels = 0, ppb = 0, n_blocks = 0;   // panels, panels per block, blocks
    float *blk = nullptr;     // the block buffer: n x (64 ppb), panel-major; the whole matrix when n_blocks == 1
    // factors, kept only when the blocks are regenerated (n_blocks > 1): X (n x d), L (n x k, split kind), Rt (k x n_pad)
    float *X = nullptr, *L = nullptr, *Rt = nullptr;
    // gemb_recon_top cache (the caller asks for the count first, then the entries)
    int top_valid = 0, top_und = 0;
    int64_t top_k = 0, top_count = 0;
    uint32_t top_bits = 0;
    // exclusion (gemb_recon_exclude): offsets relative to their block, block b's at [ex_ptr[b], ex_ptr[b + 1]), and
    // their values while the block has them masked (0 otherwise); nullptr = none
    std::vector<int64_t> ex_ptr;
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

// the diagonal entries that fall in the block of panels [p0, p0 + np) (blk = its first panel)
__global__ void recon_zero_diag_kernel(int64_t n, int64_t p0, int64_t np, float *__restrict__ blk) {
    const int64_t c0 = p0 * PW, c1 = std::min(n, (p0 + np) * PW);
    for (int64_t i = c0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < c1; i += (int64_t)gridDim.x * blockDim.x)
        blk[adj_index(i, i, n) - (size_t)c0 * n] = 0.f;
}

// rows [r0, r0 + rows) of the block's columns [c0, c0 + w), row-major: out[(i - r0) * w + (j - c0)]
__global__ void recon_rowmajor_kernel(int64_t n, int64_t c0, int64_t w, int64_t r0, int64_t rows,
                                      const float *__restrict__ blk, float *__restrict__ out) {
    const int64_t total = rows * w;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t ii = idx / w, jj = idx - ii * w;
        out[idx] = blk[adj_index(r0 + ii, c0 + jj, n) - (size_t)c0 * n];
    }
}

// out[t] = a[pi[t]][pj[t]] (0 on the diagonal) for the pairs whose column lies in the block of panels [p0, p0 + np)
__global__ void recon_pairs_kernel(int64_t n, int64_t p0, int64_t np, int64_t m, const int32_t *__restrict__ pi,
                                   const int32_t *__restrict__ pj, const float *__restrict__ blk, float *__restrict__ out) {
    const int64_t c0 = p0 * PW, c1 = (p0 + np) * PW;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = pi[t], j = pj[t];
        if (j >= c0 && j < c1) out[t] = (i == j) ? 0.f : blk[adj_index(i, j, n) - (size_t)c0 * n];
    }
}

// One warp per row i, over the columns of the block of panels [p0, p0 + np).  Edge e = (i -> j_e) of the true graph is
// in the predicted list iff j_e != i, (undirected: j_e > i) and s_e = a[i][j_e] > 0 (s_e gathered beforehand, so that
// every block compares with the same value); its 1-based position in the list sorted by weight (descending, stable
// in j) is 1 + #{valid j' : a[i][j'] > s_e  or  (a[i][j'] == s_e and j' < j_e)}.  Each block adds its part of that
// count to rank[e] and its predicted entries to n_pred_row[i]; the last block turns rank[e] into the position + 1, or
// 0 for an edge that is not predicted.  Both arrays start at 0.
__global__ void __launch_bounds__(256)
recon_rank_kernel(int64_t n, int64_t p0, int64_t np, int last, const int32_t *__restrict__ indptr,
                  const int32_t *__restrict__ indices, const float *__restrict__ s, int undirected,
                  const float *__restrict__ blk, int32_t *__restrict__ rank, int32_t *__restrict__ n_pred_row) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t c0 = p0 * PW, c1 = std::min(n, (p0 + np) * PW);
    const float *base = blk - (size_t)c0 * n;   // adj_index addresses the block from here
    for (int64_t i = warp; i < n; i += nwarps) {
        const int64_t lo = undirected ? i + 1 : 0;
        const int64_t jlo = std::max(lo, c0);
        const int e_begin = indptr[i], e_end = indptr[i + 1];
        const int nchunks = e_end > e_begin ? (e_end - e_begin + 31) / 32 : 1;   // chunk 0 also counts the row
        for (int ch = 0; ch < nchunks; ch++) {
            const int e = e_begin + ch * 32 + lane;
            long long je = -1;
            float se = -1.f;
            if (e < e_end) {
                je = indices[e];
                if (je != i && je >= lo && s[e] > 0.f) se = s[e];
            }
            const bool any_valid = __any_sync(0xffffffffu, se > 0.f);
            int mine = 0;
            if ((any_valid || ch == 0) && jlo < c1) {
                int cnt[32];
#pragma unroll
                for (int t = 0; t < 32; t++) cnt[t] = 0;
                int npred = 0;
                for (int64_t j0 = jlo & ~(int64_t)31; j0 < c1; j0 += 32) {
                    const int64_t jj = j0 + lane;
                    float v = 0.f;
                    if (jj >= jlo && jj < c1 && jj != i) v = base[adj_index(i, jj, n)];
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
                    if (lane == 0) n_pred_row[i] += npred;
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
            if (e < e_end) {
                if (last) rank[e] = se > 0.f ? rank[e] + mine + 1 : 0;
                else if (mine) rank[e] += mine;
            }
        }
    }
}

// ---- top-k threshold: radix select on the bit pattern of the valid entries (positive floats order like their bits;
// every valid entry is in [1, 0x7f800000]).  Pass 1 counts the entries per high half (bits >> 16, < 2^15 values), pass
// 2 the entries of one high half per low half; the counts are 64-bit and added with integer atomics only.
constexpr int HIST_HI = 1 << 15, HIST_LO = 1 << 16, HIST_THREADS = 1024;

// the valid entry of segment s (panel p0 + s / n, row s % n) at lane position h * 32 + lane, or 0
__device__ __forceinline__ uint32_t valid_bits(int64_t n, int64_t p, int64_t i, int h, int lane, int undirected,
                                               const float *seg, int64_t *j_out) {
    const int64_t j = p * PW + h * 32 + lane;
    const float v = seg[h * 32 + lane];
    *j_out = j;
    return (j < n && j != i && (!undirected || j > i) && v > 0.f) ? __float_as_uint(v) : 0u;
}

// LOW = false: hist[bits >> 16] += 1 for every valid entry of the block (per-CTA 32-bit counts in shared memory: a CTA
// sees fewer than 2^32 entries of one block, as grid >= entries / 2^31).  LOW = true: hist[bits & 0xffff] += 1 for the
// valid entries with bits >> 16 == hi (warp-aggregated global atomics: only the entries of one high half get here).
template <bool LOW>
__global__ void __launch_bounds__(HIST_THREADS)
recon_hist_kernel(int64_t n, int64_t p0, int64_t np, int undirected, uint32_t hi, const float *__restrict__ blk,
                  unsigned long long *__restrict__ hist) {
    extern __shared__ uint32_t sh[];
    const int lane = threadIdx.x & 31;
    if (!LOW) {
        for (int b = threadIdx.x; b < HIST_HI; b += blockDim.x) sh[b] = 0;
        __syncthreads();
    }
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t segs = np * n;             // segment = 64 consecutive floats: panel p0 + s / n, row s % n
    for (int64_t s = warp; s < segs; s += nwarps) {
        const int64_t p = p0 + s / n, i = s % n;
        if (undirected && p * PW + PW - 1 <= i) continue;      // every column of the panel is <= i
        const float *seg = blk + (size_t)s * PW;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            int64_t j;
            const uint32_t b = valid_bits(n, p, i, h, lane, undirected, seg, &j);
            if (!LOW) {
                if (b) atomicAdd(&sh[b >> 16], 1u);
            } else {
                const bool in = b && (b >> 16) == hi;
                const unsigned same = __match_any_sync(0xffffffffu, in ? (b & 0xffffu) : 0x10000u);
                if (in && lane == __ffs(same) - 1) atomicAdd(&hist[b & 0xffffu], (unsigned long long)__popc(same));
            }
        }
    }
    if (!LOW) {
        __syncthreads();
        for (int b = threadIdx.x; b < HIST_HI; b += blockDim.x)
            if (sh[b]) atomicAdd(&hist[b], (unsigned long long)sh[b]);
    }
}

// collect the valid entries of the block whose bit pattern is >= bits (warp-aggregated slots of one counter)
__global__ void __launch_bounds__(256)
recon_select_kernel(int64_t n, int64_t p0, int64_t np, int undirected, uint32_t bits, const float *__restrict__ blk,
                    unsigned long long *__restrict__ counter, int64_t cap, int32_t *__restrict__ oi,
                    int32_t *__restrict__ oj, float *__restrict__ ow) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t segs = np * n;
    for (int64_t s = warp; s < segs; s += nwarps) {
        const int64_t p = p0 + s / n, i = s % n;
        if (undirected && p * PW + PW - 1 <= i) continue;
        const float *seg = blk + (size_t)s * PW;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            int64_t j;
            const uint32_t b = valid_bits(n, p, i, h, lane, undirected, seg, &j);
            const bool valid = b && b >= bits;
            const unsigned mask = __ballot_sync(0xffffffffu, valid);
            if (mask) {
                unsigned long long base = 0;
                if (lane == 0) base = atomicAdd(counter, (unsigned long long)__popc(mask));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (valid) {
                    const int64_t slot = (int64_t)base + __popc(mask & ((1u << lane) - 1u));
                    if (slot < cap) { oi[slot] = (int32_t)i; oj[slot] = (int32_t)j; ow[slot] = __uint_as_float(b); }
                }
            }
        }
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

// One launch over every (128-row x 64-column) tile of the block of panels from p0 (blk = its first panel), tile t =
// panel p0 + t / row_tiles, row tile t % row_tiles: the row tiles of one panel run next to each other and share its 64
// column vectors in L2.  The rows and the panel's columns are staged k-major in shared memory, SQD_KC coordinates at a
// time; each thread keeps an 8 x 4 tile of sum_k (x_ik - x_jk)^2 (FADD + FFMA per term, fp32) and its 16 threads of a
// row write the whole 256-byte panel row.  Diagonal and padded columns get key 0.
__global__ void __launch_bounds__(SQD_THREADS)
recon_sqdist_kernel(int64_t n, int d, int64_t row_tiles, int64_t p0, const float *__restrict__ X, float *__restrict__ blk) {
    __shared__ __align__(16) float xr[SQD_KC][SQD_ROWS + 4];
    __shared__ __align__(16) float xc[SQD_KC][PW + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int64_t pl = (int64_t)blockIdx.x / row_tiles;
    const int64_t i0 = ((int64_t)blockIdx.x - pl * row_tiles) * SQD_ROWS, j0 = (p0 + pl) * PW;
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
        *reinterpret_cast<float4 *>(blk + ((size_t)pl * (size_t)n + (size_t)i) * PW + tx * 4) = make_float4(v[0], v[1], v[2], v[3]);
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
// blk[off[t]] <-> saved[t]: with saved all 0 the first launch masks the excluded entries, the second restores them.
// The offsets are distinct, so no two threads touch one entry.
__global__ void recon_swap_kernel(int64_t m, const int64_t *__restrict__ off, float *__restrict__ saved,
                                  float *__restrict__ blk) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const float v = blk[off[t]];
        blk[off[t]] = saved[t];
        saved[t] = v;
    }
}

// Write the panels [p0, p0 + np) into the block buffer: the launches the whole matrix is made of, for those panels.
static int make_block(gemb_recon *r, int64_t p0, int64_t np) {
    gemb_ctx *c = r->ctx;
    const int64_t n = r->n;
    if (r->kind == GEMB_RECON_GAUSS) {
        const int64_t row_tiles = (n + SQD_ROWS - 1) / SQD_ROWS;
        return launch(c, recon_sqdist_kernel, (unsigned)(row_tiles * np), SQD_THREADS, 0, n, r->d, row_tiles, p0, r->X, r->blk);
    }
    const float *Lp = r->kind == GEMB_RECON_SPLIT ? r->L : r->X;
    for (int64_t p = p0; p < p0 + np; p++)
        GEMB_TRY(apply_launch(c, n, Lp, r->k, r->Rt + p * PW, (int)r->n_pad, PW, r->blk + (size_t)(p - p0) * n * PW, PW));
    return launch(c, recon_zero_diag_kernel, grid_stride(c, np * PW, 256, 16), 256, 0, n, p0, np, r->blk);
}

static int swap_excluded(gemb_recon *r, int64_t b) {
    if (r->ex_nnz == 0) return GEMB_OK;
    const int64_t t0 = r->ex_ptr[b], m = r->ex_ptr[b + 1] - t0;
    if (m == 0) return GEMB_OK;
    return launch(r->ctx, recon_swap_kernel, grid_stride(r->ctx, m, 256, 16), 256, 0, m, r->ex_off + t0, r->ex_saved + t0, r->blk);
}

// body(p0, np) on every block (only those with need[b] when need is given), in order; regenerated first unless the
// handle holds the whole matrix.  masked: the block's excluded entries are 0 while body() runs, and are put back
// whatever body() returns (the first error wins).
template <class F> static int for_each_block(gemb_recon *r, bool masked, const std::vector<char> *need, F body) {
    for (int64_t b = 0; b < r->n_blocks; b++) {
        if (need && !(*need)[b]) continue;
        const int64_t p0 = b * r->ppb, np = std::min(r->ppb, r->n_panels - p0);
        if (r->n_blocks > 1) GEMB_TRY(make_block(r, p0, np));
        if (masked) GEMB_TRY(swap_excluded(r, b));
        const int st = body(p0, np);
        const int st_restore = masked ? swap_excluded(r, b) : GEMB_OK;
        GEMB_TRY(st);
        GEMB_TRY(st_restore);
    }
    return GEMB_OK;
}

// which blocks hold the column of at least one of the m pairs
static std::vector<char> blocks_of(const gemb_recon *r, const int32_t *pj, int64_t m) {
    std::vector<char> need((size_t)r->n_blocks, 0);
    for (int64_t t = 0; t < m; t++) need[(size_t)((pj[t] >> 6) / r->ppb)] = 1;
    return need;
}

// out[t] = the entry (pi[t], pj[t]) as stored (key for the Gaussian kind), exclusion masked when `masked`; pi, pj, out on
// the device, pj_h the host copy of pj
static int gather(gemb_recon *r, bool masked, int64_t m, const int32_t *pj_h, const int32_t *pi, const int32_t *pj,
                  float *out) {
    gemb_ctx *c = r->ctx;
    const std::vector<char> need = blocks_of(r, pj_h, m);
    return for_each_block(r, masked, &need, [&](int64_t p0, int64_t np) {
        return launch(c, recon_pairs_kernel, grid_stride(c, m, 256, 16), 256, 0, r->n, p0, np, m, pi, pj, r->blk, out);
    });
}

// one histogram pass (see recon_hist_kernel) into the 64-bit device array hist of HIST_HI or HIST_LO bins -> host h
static int histogram(gemb_recon *r, bool low, int und, uint32_t hi, unsigned long long *hist, std::vector<unsigned long long> &h) {
    gemb_ctx *c = r->ctx;
    const int bins = low ? HIST_LO : HIST_HI;
    const size_t smem = low ? 0 : sizeof(uint32_t) * HIST_HI;
    const auto kernel = low ? recon_hist_kernel<true> : recon_hist_kernel<false>;
    GEMB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GEMB_CUDA(cudaMemsetAsync(hist, 0, sizeof(unsigned long long) * bins, c->stream));
    GEMB_TRY(for_each_block(r, true, nullptr, [&](int64_t p0, int64_t np) {
        const int64_t entries = np * PW * r->n;
        const int grid = (int)std::max<int64_t>(grid_stride(c, np * r->n * 32, HIST_THREADS, 1), (entries >> 31) + 1);
        return launch(c, kernel, grid, HIST_THREADS, smem, r->n, p0, np, und, hi, r->blk, hist);
    }));
    h.assign((size_t)bins, 0);
    return copy_sync(c, h.data(), hist, sizeof(unsigned long long) * bins, cudaMemcpyDeviceToHost);
}

// Gaussian kind: turn the m keys at w (device) into delta before they are copied out; a no-op for the other kinds
static int decode_out(const gemb_recon *r, int64_t m, float *w) {
    if (r->kind != GEMB_RECON_GAUSS || m == 0) return GEMB_OK;
    return launch(r->ctx, recon_key_to_delta_kernel, grid_stride(r->ctx, m, 256, 16), 256, 0, m, w);
}

}  // namespace gemb

using namespace gemb;

extern "C" {

int gemb_recon_create_blocked(gemb_ctx *c, const float *X, int64_t n, int d, int kind, int64_t panels_per_block,
                              gemb_recon **out) {
    GEMB_ARG(c && X && out, "ctx/X/out");
    GEMB_ARG(n > 0 && n < ((int64_t)1 << 31), "n");
    GEMB_ARG(panels_per_block >= 0, "panels_per_block (0 = automatic)");
    if (kind != GEMB_RECON_DOT && kind != GEMB_RECON_GAUSS) kind = GEMB_RECON_SPLIT;
    const bool split = kind == GEMB_RECON_SPLIT, gauss = kind == GEMB_RECON_GAUSS;
    GEMB_ARG(d > 0 && (!split || d % 2 == 0), "d (even when split)");
    if (gauss) {
        const size_t total = (size_t)n * (size_t)d;
        for (size_t t = 0; t < total; t++)
            GEMB_ARG(std::isfinite(X[t]), "X finite (a NaN or infinite distance has no place in the order)");
    }
    GEMB_CUDA(cudaSetDevice(c->device));
    const int k = split ? d / 2 : d;
    const int64_t n_pad = (n + PW - 1) / PW * PW, n_panels = n_pad / PW;
    size_t free_b = 0, total_b = 0;
    GEMB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // device bytes left for the matrix once X and the factors (L and Rt) are in place
    const double factors = gauss ? 0.0 : 8.0 * (double)n_pad * k;
    const double avail = 0.9 * ((double)free_b + (double)gemb_mem_cached_bytes()) - 4.0 * (double)n * d - factors;
    const double panel_bytes = 4.0 * PW * (double)n;
    int64_t ppb = panels_per_block ? std::min(panels_per_block, n_panels) : n_panels;
    if (!panels_per_block && panel_bytes * n_panels > avail) {
        // blocks: keep room for the scratch of a call (its CSR, ranks and selection: 16 bytes per node and 1 GiB)
        ppb = std::min<int64_t>(n_panels - 1, (int64_t)std::floor((avail - 16.0 * n - (double)(1 << 30)) / panel_bytes));
    }
    if (ppb < 1 || panel_bytes * ppb > avail) {
        set_error("gemb_recon_create: a block of %lld panel(s) of the %lld x %lld reconstruction needs %.1f GB of device "
                  "memory besides the factors, %.1f GB free", (long long)std::max<int64_t>(ppb, 1), (long long)n,
                  (long long)n, panel_bytes * std::max<int64_t>(ppb, 1) / 1e9, (double)free_b / 1e9);
        return GEMB_ERR_NOMEM;
    }
    gemb_recon tmp;
    tmp.ctx = c; tmp.n = n; tmp.n_pad = n_pad; tmp.d = d; tmp.k = k; tmp.kind = kind;
    tmp.n_panels = n_panels; tmp.ppb = ppb; tmp.n_blocks = (n_panels + ppb - 1) / ppb;
    DeviceBuffer<float> dX, L, Rt, blk;
    GEMB_CUDA(dX.upload(X, (size_t)n * d, c->stream));
    if (!gauss) {
        GEMB_CUDA(Rt.alloc((size_t)n_pad * k));
        if (split) {
            GEMB_CUDA(L.alloc((size_t)n * k));
            GEMB_TRY(launch(c, recon_left_kernel, grid_stride(c, n * k, 256, 16), 256, 0, n, d, k, dX.get(), L.get()));
        }
        GEMB_TRY(launch(c, recon_right_t_kernel, dim3((unsigned)((n_pad + 31) / 32), (unsigned)((k + 31) / 32)), dim3(32, 8), 0,
                        n, n_pad, d, k, split ? k : 0, dX.get(), Rt.get()));
    }
    GEMB_CUDA(blk.alloc((size_t)n * PW * ppb));
    tmp.X = dX.get(); tmp.L = L.get(); tmp.Rt = Rt.get(); tmp.blk = blk.get();
    if (tmp.n_blocks == 1) GEMB_TRY(make_block(&tmp, 0, n_panels));   // the whole matrix, kept: the factors go
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    gemb_recon *r = new gemb_recon(tmp);
    r->blk = blk.release();
    if (r->n_blocks == 1) {
        r->X = r->L = r->Rt = nullptr;
    } else {
        r->X = dX.release(); r->L = L.release(); r->Rt = Rt.release();
    }
    *out = r;
    return GEMB_OK;
}

int gemb_recon_create(gemb_ctx *c, const float *X, int64_t n, int d, int kind, gemb_recon **out) {
    return gemb_recon_create_blocked(c, X, n, d, kind, 0, out);
}

int gemb_recon_info(gemb_recon *r, int64_t *panels_per_block, int64_t *blocks) {
    GEMB_ARG(r && panels_per_block && blocks, "recon/panels_per_block/blocks");
    *panels_per_block = r->ppb;
    *blocks = r->n_blocks;
    return GEMB_OK;
}

int gemb_recon_free(gemb_recon *r) {
    if (!r) return GEMB_OK;
    cudaSetDevice(r->ctx->device);
    dfree(r->blk);
    dfree(r->X);
    dfree(r->L);
    dfree(r->Rt);
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
    const int64_t wmax = std::min(n, r->ppb * PW);
    const int64_t rows = std::max<int64_t>(1, std::min<int64_t>(n, ((int64_t)256 << 20) / (4 * wmax)));   // <= 256 MB chunks
    DeviceBuffer<float> buf;
    GEMB_CUDA(buf.alloc((size_t)rows * wmax));
    return for_each_block(r, false, nullptr, [&](int64_t p0, int64_t np) -> int {
        const int64_t c0 = p0 * PW, w = std::min(n, (p0 + np) * PW) - c0;
        for (int64_t r0 = 0; r0 < n; r0 += rows) {
            const int64_t nr = std::min(rows, n - r0);
            GEMB_TRY(launch(c, recon_rowmajor_kernel, grid_stride(c, nr * w, 256, 16), 256, 0, n, c0, w, r0, nr, r->blk, buf.get()));
            GEMB_TRY(decode_out(r, nr * w, buf.get()));
            GEMB_CUDA(cudaMemcpy2DAsync(adj_out + (size_t)r0 * n + c0, sizeof(float) * (size_t)n, buf.get(), sizeof(float) * (size_t)w,
                                        sizeof(float) * (size_t)w, (size_t)nr, cudaMemcpyDeviceToHost, c->stream));
            GEMB_CUDA(cudaStreamSynchronize(c->stream));
        }
        return GEMB_OK;
    });
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
    GEMB_TRY(gather(r, false, m, pj, di.get(), dj.get(), dout.get()));
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
    std::vector<int32_t> rows((size_t)nnz);
    for (int64_t i = 0; i < n; i++)
        for (int64_t t = indptr[i]; t < indptr[i + 1]; t++) rows[(size_t)t] = (int32_t)i;
    DeviceBuffer<int32_t> dp, dix, drow, drank, dnp;
    DeviceBuffer<float> ds;
    GEMB_CUDA(dp.upload(indptr, (size_t)(n + 1), c->stream));
    GEMB_CUDA(dix.upload(indices, (size_t)nnz, c->stream));
    GEMB_CUDA(drow.upload(rows.data(), (size_t)nnz, c->stream));
    GEMB_CUDA(ds.alloc((size_t)std::max<int64_t>(nnz, 1)));
    GEMB_CUDA(drank.alloc((size_t)std::max<int64_t>(nnz, 1)));
    GEMB_CUDA(dnp.alloc((size_t)n));
    GEMB_CUDA(cudaMemsetAsync(drank.get(), 0, sizeof(int32_t) * (size_t)std::max<int64_t>(nnz, 1), c->stream));
    GEMB_CUDA(cudaMemsetAsync(dnp.get(), 0, sizeof(int32_t) * (size_t)n, c->stream));
    // s_e = the score of every true edge with the exclusion applied, then the counting pass
    if (nnz) GEMB_TRY(gather(r, true, nnz, indices, drow.get(), dix.get(), ds.get()));
    const int und = is_undirected ? 1 : 0;
    GEMB_TRY(for_each_block(r, true, nullptr, [&](int64_t p0, int64_t np) {
        return launch(c, recon_rank_kernel, grid_stride(c, n * 32, 256, 16), 256, 0, n, p0, np, p0 + np == r->n_panels ? 1 : 0,
                      dp.get(), dix.get(), ds.get(), und, r->blk, drank.get(), dnp.get());
    }));
    if (nnz) GEMB_CUDA(cudaMemcpyAsync(rank_out, drank.get(), sizeof(int32_t) * (size_t)nnz, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(n_pred_row, dnp.get(), sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

int gemb_recon_exclude(gemb_recon *r, const int32_t *ex_indptr, const int32_t *ex_indices) {
    GEMB_ARG(r, "recon");
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    const int64_t n = r->n, nb = r->n_blocks;
    const size_t blk_floats = (size_t)n * PW * r->ppb;
    std::vector<int64_t> ptr((size_t)nb + 1, 0), off;
    if (ex_indptr) {
        const int64_t nnz = ex_indptr[n];
        GEMB_ARG(ex_indptr[0] == 0 && nnz >= 0 && (nnz == 0 || ex_indices), "exclusion CSR");
        for (int64_t i = 0; i < n; i++) {
            GEMB_ARG(ex_indptr[i + 1] >= ex_indptr[i], "exclusion offsets non-decreasing");
            for (int64_t t = ex_indptr[i]; t < ex_indptr[i + 1]; t++) {
                GEMB_ARG(ex_indices[t] >= 0 && ex_indices[t] < n, "exclusion column id out of range");
                GEMB_ARG(t == ex_indptr[i] || ex_indices[t] > ex_indices[t - 1], "exclusion columns strictly ascending");
                ptr[(size_t)((ex_indices[t] >> 6) / r->ppb) + 1]++;
            }
        }
        for (int64_t b = 0; b < nb; b++) ptr[(size_t)b + 1] += ptr[(size_t)b];
        off.resize((size_t)nnz);
        std::vector<int64_t> fill(ptr.begin(), ptr.end() - 1);
        for (int64_t i = 0; i < n; i++)
            for (int64_t t = ex_indptr[i]; t < ex_indptr[i + 1]; t++) {
                const size_t o = adj_index(i, ex_indices[t], n);   // offset in the whole matrix -> block, offset in it
                off[(size_t)fill[o / blk_floats]++] = (int64_t)(o % blk_floats);
            }
    }
    dfree(r->ex_off);
    dfree(r->ex_saved);
    r->ex_off = nullptr;
    r->ex_saved = nullptr;
    r->ex_nnz = 0;
    r->ex_ptr.clear();
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
    r->ex_ptr = std::move(ptr);
    return GEMB_OK;
}

int gemb_recon_top(gemb_recon *r, int is_undirected, int64_t max_k, int64_t cap, int32_t *i_out, int32_t *j_out,
                   float *w_out, int64_t *m_out) {
    GEMB_ARG(r && m_out, "recon/m_out");
    GEMB_ARG(cap == 0 || (i_out && j_out && w_out), "output arrays");
    gemb_ctx *c = r->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    const int und = is_undirected ? 1 : 0;
    if (!(r->top_valid && r->top_und == und && r->top_k == max_k)) {
        // T = the largest bit pattern with count(>= T) >= K: the high half of T is the largest h with
        // sum_{h' >= h} hist_hi[h'] >= K, its low half the largest l with (that sum above h) + sum_{l' >= l} hist_lo[l'] >= K
        DeviceBuffer<unsigned long long> dhist;
        GEMB_CUDA(dhist.alloc(HIST_LO));
        std::vector<unsigned long long> h;
        GEMB_TRY(histogram(r, false, und, 0, dhist.get(), h));
        int64_t total = 0;
        for (unsigned long long x : h) total += (int64_t)x;
        uint32_t bits = 1u;
        int64_t count = total;
        if (max_k >= 0 && total > max_k) {
            const int64_t K = std::max<int64_t>(max_k, 1);
            int64_t above = 0;
            int hi = HIST_HI - 1;
            while (above + (int64_t)h[(size_t)hi] < K) above += (int64_t)h[(size_t)hi--];
            GEMB_TRY(histogram(r, true, und, (uint32_t)hi, dhist.get(), h));
            int lo = HIST_LO - 1;
            while (above + (int64_t)h[(size_t)lo] < K) above += (int64_t)h[(size_t)lo--];
            bits = ((uint32_t)hi << 16) | (uint32_t)lo;
            count = max_k == 0 ? 0 : above + (int64_t)h[(size_t)lo];
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
    DeviceBuffer<unsigned long long> dcounter;
    DeviceBuffer<int32_t> di, dj;
    DeviceBuffer<float> dw;
    GEMB_CUDA(dcounter.alloc(1));
    GEMB_CUDA(di.alloc((size_t)m));
    GEMB_CUDA(dj.alloc((size_t)m));
    GEMB_CUDA(dw.alloc((size_t)m));
    GEMB_CUDA(cudaMemsetAsync(dcounter.get(), 0, sizeof(unsigned long long), c->stream));
    GEMB_TRY(for_each_block(r, true, nullptr, [&](int64_t p0, int64_t np) {
        return launch(c, recon_select_kernel, grid_stride(c, np * r->n * 32, 256, 16), 256, 0, r->n, p0, np, und, r->top_bits,
                      r->blk, dcounter.get(), m, di.get(), dj.get(), dw.get());
    }));
    GEMB_TRY(decode_out(r, m, dw.get()));
    GEMB_CUDA(cudaMemcpyAsync(i_out, di.get(), sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(j_out, dj.get(), sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(w_out, dw.get(), sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

}  // extern "C"
