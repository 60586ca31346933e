// gem_b200/csrc/spmm.cu -- CSR SpMM  Y = X0 + alpha * A * X  over an fp32 row-major block.
//
// Replaces the dense products hidden in hope.py:31 (inv(I - beta A) . beta A) and inside
// scipy's svds matvecs (hope.py:33): S is never formed, every S.x is a Horner sweep of this kernel.
//
// Mapping (HBM/L2-bound gather, SURVEY 8(d)): a group of G = b/4 threads owns one CSR row; thread
// c of the group owns columns [4c, 4c+4) of the block, so one nonzero = one coalesced 16*G-byte
// read of X[col, :] (320 B for b = 80) and the accumulators never leave registers.  Column ids and
// values of a row are read through the read-only path (same address across the group -> one L1
// broadcast).  The nonzero loop is unrolled by 4 so that each thread keeps 4 independent 16-byte
// gathers in flight.  The Horner epilogue (X0 + alpha * acc) is fused: one extra coalesced read.
#include "common.cuh"
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include "tc_common.cuh"

namespace gemb {

int spmm_heavy_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int b, float alpha, const float *X, float gamma,
                      const float *Xself, float delta, const float *X0, float *Y, const HaloPushArgs *push, int n_loc);

__device__ __forceinline__ void fma4(float4 &a, float v, const float4 &x) {
    a.x = fmaf(v, x.x, a.x);
    a.y = fmaf(v, x.y, a.y);
    a.z = fmaf(v, x.z, a.z);
    a.w = fmaf(v, x.w, a.w);
}

// Y[row] = alpha * (A X)[row] + gamma * Xself[row] + delta * X0[row]
//   Horner / Katz sweep:      gamma = 0, delta = 1, X0 = the sweep's input block
//   Chebyshev three-term step: gamma = -2 s c0 / e (current block), delta = -s s' (previous block)
// HAS_PUSH (multi-GPU, halo.cu): the finished row is also stored into the halo slots of the peers whose shards
// reference it -- 16-byte posted stores over NVLink, issued while the other row groups of the SM are still gathering.
template <bool HAS_VAL, bool HAS_X0, bool HAS_SELF, bool HAS_PUSH, bool HALF>
__global__ void __launch_bounds__(256)
spmm_rowgroup_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                     const float *__restrict__ vals, int64_t n_rows, int G, int rows_per_cta,
                     float alpha, float gamma, float delta, const float4 *__restrict__ X,
                     const float4 *__restrict__ Xself, const float4 *__restrict__ X0,
                     float4 *__restrict__ Y, int heavy_deg, HaloPushArgs P, int n_loc) {
    const int tid = threadIdx.x;
    const int lr = tid / G;
    const int c = tid - lr * G;
    if (lr >= rows_per_cta) return;
    const int64_t row = (int64_t)blockIdx.x * rows_per_cta + lr;
    if (row >= n_rows) return;
    const int s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
    if (heavy_deg > 0 && e - s > heavy_deg) return;   // a heavy row: spmm_heavy_* kernels below
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int i = s;
    for (; i + 4 <= e; i += 4) {
        const int c0 = __ldg(indices + i), c1 = __ldg(indices + i + 1);
        const int c2 = __ldg(indices + i + 2), c3 = __ldg(indices + i + 3);
        float v0 = 1.f, v1 = 1.f, v2 = 1.f, v3 = 1.f;
        if (HAS_VAL) {
            v0 = __ldg(vals + i);
            v1 = __ldg(vals + i + 1);
            v2 = __ldg(vals + i + 2);
            v3 = __ldg(vals + i + 3);
        }
        const float4 x0 = halo_gather<HALF>(X, c0, G, c, n_loc);
        const float4 x1 = halo_gather<HALF>(X, c1, G, c, n_loc);
        const float4 x2 = halo_gather<HALF>(X, c2, G, c, n_loc);
        const float4 x3 = halo_gather<HALF>(X, c3, G, c, n_loc);
        fma4(acc, v0, x0);
        fma4(acc, v1, x1);
        fma4(acc, v2, x2);
        fma4(acc, v3, x3);
    }
    for (; i < e; i++) {
        const int c0 = __ldg(indices + i);
        const float v0 = HAS_VAL ? __ldg(vals + i) : 1.f;
        fma4(acc, v0, halo_gather<HALF>(X, c0, G, c, n_loc));
    }
    float4 r = make_float4(alpha * acc.x, alpha * acc.y, alpha * acc.z, alpha * acc.w);
    if (HAS_SELF) {
        const float4 z = __ldg(Xself + row * G + c);
        r.x = fmaf(gamma, z.x, r.x);
        r.y = fmaf(gamma, z.y, r.y);
        r.z = fmaf(gamma, z.z, r.z);
        r.w = fmaf(gamma, z.w, r.w);
    }
    if (HAS_X0) {
        const float4 z = __ldg(X0 + row * G + c);
        r.x = fmaf(delta, z.x, r.x);
        r.y = fmaf(delta, z.y, r.y);
        r.z = fmaf(delta, z.z, r.z);
        r.w = fmaf(delta, z.w, r.w);
    }
    Y[row * G + c] = r;
    if (HAS_PUSH) halo_push_row(P, row, G, c, r);
}

// ---- heavy rows (degree > SPMM_HEAVY_DEG; the hubs of a power-law graph -- R-MAT scale 21 has a 61 814-neighbour
// row, which one 20-thread group would walk for longer than the whole rest of the sweep takes).  Each chunk of
// SPMM_HEAVY_CHUNK nonzeros is one CTA: its row groups stride over the chunk, the group sums are added in a fixed
// order in shared memory, and the chunk sum goes to a scratch row; a second tiny kernel adds the chunk sums of a row
// in chunk order and applies the fused epilogue.  No atomics: the result is bit-reproducible.
template <bool HAS_VAL, bool HALF>
__global__ void __launch_bounds__(256)
spmm_heavy_partial_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                          const float *__restrict__ vals, const int32_t *__restrict__ item_row,
                          const int32_t *__restrict__ item_beg, int G, int groups, int chunk,
                          const float4 *__restrict__ X, float4 *__restrict__ partial, int n_loc) {
    __shared__ float4 red[256];
    const int tid = threadIdx.x;
    const int lr = tid / G;
    const int c = tid - lr * G;
    const int item = blockIdx.x;
    const int row = __ldg(item_row + item);
    const int beg = __ldg(item_beg + item);
    const int row_end = __ldg(indptr + row + 1);
    const int end = beg + chunk < row_end ? beg + chunk : row_end;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lr < groups) {
        int i = beg + lr;
        for (; i + 3 * groups < end; i += 4 * groups) {
            const int c0 = __ldg(indices + i), c1 = __ldg(indices + i + groups);
            const int c2 = __ldg(indices + i + 2 * groups), c3 = __ldg(indices + i + 3 * groups);
            float v0 = 1.f, v1 = 1.f, v2 = 1.f, v3 = 1.f;
            if (HAS_VAL) {
                v0 = __ldg(vals + i); v1 = __ldg(vals + i + groups);
                v2 = __ldg(vals + i + 2 * groups); v3 = __ldg(vals + i + 3 * groups);
            }
            const float4 x0 = halo_gather<HALF>(X, c0, G, c, n_loc), x1 = halo_gather<HALF>(X, c1, G, c, n_loc);
            const float4 x2 = halo_gather<HALF>(X, c2, G, c, n_loc), x3 = halo_gather<HALF>(X, c3, G, c, n_loc);
            fma4(acc, v0, x0); fma4(acc, v1, x1); fma4(acc, v2, x2); fma4(acc, v3, x3);
        }
        for (; i < end; i += groups) {
            const int c0 = __ldg(indices + i);
            const float v0 = HAS_VAL ? __ldg(vals + i) : 1.f;
            fma4(acc, v0, halo_gather<HALF>(X, c0, G, c, n_loc));
        }
        red[tid] = acc;
    }
    __syncthreads();
    if (lr == 0) {
        float4 sum = red[c];
        for (int g = 1; g < groups; g++) {
            const float4 t = red[g * G + c];
            sum.x += t.x; sum.y += t.y; sum.z += t.z; sum.w += t.w;
        }
        partial[(size_t)item * G + c] = sum;
    }
}

template <bool HAS_X0, bool HAS_SELF>
__global__ void __launch_bounds__(256)
spmm_heavy_finish_kernel(int n_heavy, const int32_t *__restrict__ heavy_row, const int32_t *__restrict__ heavy_first,
                         int G, float alpha, float gamma, float delta, const float4 *__restrict__ partial,
                         const float4 *__restrict__ Xself, const float4 *__restrict__ X0, float4 *__restrict__ Y,
                         bool has_push, HaloPushArgs P) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int h = idx / G, c = idx - h * G;
    if (h >= n_heavy) return;
    const int64_t row = __ldg(heavy_row + h);
    const int f = __ldg(heavy_first + h), l = __ldg(heavy_first + h + 1);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int it = f; it < l; it++) {
        const float4 t = partial[(size_t)it * G + c];
        acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    float4 r = make_float4(alpha * acc.x, alpha * acc.y, alpha * acc.z, alpha * acc.w);
    if (HAS_SELF) {
        const float4 z = __ldg(Xself + row * G + c);
        r.x = fmaf(gamma, z.x, r.x); r.y = fmaf(gamma, z.y, r.y); r.z = fmaf(gamma, z.z, r.z); r.w = fmaf(gamma, z.w, r.w);
    }
    if (HAS_X0) {
        const float4 z = __ldg(X0 + row * G + c);
        r.x = fmaf(delta, z.x, r.x); r.y = fmaf(delta, z.y, r.y); r.z = fmaf(delta, z.z, r.z); r.w = fmaf(delta, z.w, r.w);
    }
    Y[row * G + c] = r;
    if (has_push) halo_push_row(P, row, G, c, r);
}

// ---- v3 (TMA-staged): one CTA per row TILE (passes * rows_per_cta consecutive rows); the tile's slice of the column-id
// (and value) arrays -- one contiguous range of the CSR -- is staged into shared memory by ONE TMA bulk copy
// (cp.async.bulk + mbarrier complete_tx) issued by thread 0 while every row group fetches its row offsets; the other
// resident CTAs of the SM hide the copy's latency.  The row groups then read their column ids from shared memory: the
// dependent chain per row drops from indptr -> indices -> X (three global round trips) to indptr -> X, and the
// ~nnz/4 broadcast LDGs of v1 (one L1 wavefront each) leave the L1 data pipe to the gathers.  scripts/spmm_lab.cu times
// the variants against each other (GEMB_SPMM=v1 and GEMB_SPMM_PASSES select them in the library).  A tile whose
// slice exceeds the staging buffer (hubs) reads its ids from global memory as v1 does; rows above SPMM_HEAVY_DEG still go
// to the chunk kernels.
constexpr int BULK_CAP = 3072;                 // staged ids per tile (+ up to 3 of alignment slack + 4 of over-read)
template <bool HAS_VAL, bool HAS_PUSH, bool HAS_X0, bool HAS_SELF, bool HALF>
__global__ void __launch_bounds__(256)
spmm_bulk_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                 const float *__restrict__ vals, int64_t n_rows, int64_t nnz, int G, int rows_per_cta, int tile_rows,
                 float alpha, float gamma, float delta, const float4 *__restrict__ X,
                 const float4 *__restrict__ Xself, const float4 *__restrict__ X0, float4 *__restrict__ Y,
                 int heavy_deg, HaloPushArgs P, int n_loc) {
    __shared__ __align__(16) int32_t s_idx[BULK_CAP + 8];
    __shared__ __align__(16) float s_val[HAS_VAL ? BULK_CAP + 8 : 4];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ int s_base;                     // first staged nonzero of the tile, or -1: not staged
    const int tid = threadIdx.x;
    const int lr = tid / G;
    const int c = tid - lr * G;
    const int64_t r0 = (int64_t)blockIdx.x * tile_rows;
    const int64_t r1 = r0 + tile_rows < n_rows ? r0 + tile_rows : n_rows;
    const uint32_t bar = tc::smem_u32(&s_bar);
    if (tid == 0) {
        tc::mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const int s = __ldg(indptr + r0), e = __ldg(indptr + r1);
        const int a0 = s & ~3;                                   // 16-byte aligned source
        int cnt = (e - a0 + 3) & ~3;
        if ((int64_t)a0 + cnt > ((nnz + 3) & ~(int64_t)3)) cnt = (int)(((nnz + 3) & ~(int64_t)3) - a0);   // arrays are padded to x4
        if (e > s && cnt <= BULK_CAP + 4) {
            s_base = a0;
            const uint32_t bytes = (uint32_t)cnt * 4u;
            tc::mbar_expect_tx(bar, HAS_VAL ? 2 * bytes : bytes);
            tc::bulk_g2s(tc::smem_u32(&s_idx[0]), indices + a0, bytes, bar);
            if (HAS_VAL) tc::bulk_g2s(tc::smem_u32(&s_val[0]), vals + a0, bytes, bar);
        } else {
            s_base = -1;
            tc::mbar_arrive(bar);                                // an empty transaction completes the phase
        }
    }
    __syncthreads();
    if (lr >= rows_per_cta) return;
    int64_t row = r0 + lr;
    int s = 0, e = 0;
    if (row < r1) { s = __ldg(indptr + row); e = __ldg(indptr + row + 1); }     // in flight together with the bulk copy
    tc::mbar_wait(bar, 0);
    const int base = s_base;
    const int32_t *li = s_idx - base;
    const float *lv = s_val - base;
    for (; row < r1; row += rows_per_cta) {
        if (!(heavy_deg > 0 && e - s > heavy_deg)) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            int i = s;
            if (base >= 0) {
                for (; i + 4 <= e; i += 4) {
                    const int c0 = li[i], c1 = li[i + 1], c2 = li[i + 2], c3 = li[i + 3];
                    const float4 x0 = halo_gather<HALF>(X, c0, G, c, n_loc), x1 = halo_gather<HALF>(X, c1, G, c, n_loc);
                    const float4 x2 = halo_gather<HALF>(X, c2, G, c, n_loc), x3 = halo_gather<HALF>(X, c3, G, c, n_loc);
                    fma4(acc, HAS_VAL ? lv[i] : 1.f, x0); fma4(acc, HAS_VAL ? lv[i + 1] : 1.f, x1);
                    fma4(acc, HAS_VAL ? lv[i + 2] : 1.f, x2); fma4(acc, HAS_VAL ? lv[i + 3] : 1.f, x3);
                }
                for (; i < e; i++) fma4(acc, HAS_VAL ? lv[i] : 1.f, halo_gather<HALF>(X, li[i], G, c, n_loc));
            } else {
                for (; i + 4 <= e; i += 4) {
                    const int c0 = __ldg(indices + i), c1 = __ldg(indices + i + 1);
                    const int c2 = __ldg(indices + i + 2), c3 = __ldg(indices + i + 3);
                    const float4 x0 = halo_gather<HALF>(X, c0, G, c, n_loc), x1 = halo_gather<HALF>(X, c1, G, c, n_loc);
                    const float4 x2 = halo_gather<HALF>(X, c2, G, c, n_loc), x3 = halo_gather<HALF>(X, c3, G, c, n_loc);
                    fma4(acc, HAS_VAL ? __ldg(vals + i) : 1.f, x0); fma4(acc, HAS_VAL ? __ldg(vals + i + 1) : 1.f, x1);
                    fma4(acc, HAS_VAL ? __ldg(vals + i + 2) : 1.f, x2); fma4(acc, HAS_VAL ? __ldg(vals + i + 3) : 1.f, x3);
                }
                for (; i < e; i++) fma4(acc, HAS_VAL ? __ldg(vals + i) : 1.f, halo_gather<HALF>(X, __ldg(indices + i), G, c, n_loc));
            }
            float4 r = make_float4(alpha * acc.x, alpha * acc.y, alpha * acc.z, alpha * acc.w);
            if (HAS_SELF) {
                const float4 z = __ldg(Xself + row * G + c);
                r.x = fmaf(gamma, z.x, r.x); r.y = fmaf(gamma, z.y, r.y); r.z = fmaf(gamma, z.z, r.z); r.w = fmaf(gamma, z.w, r.w);
            }
            if (HAS_X0) {
                const float4 z = __ldg(X0 + row * G + c);
                r.x = fmaf(delta, z.x, r.x); r.y = fmaf(delta, z.y, r.y); r.z = fmaf(delta, z.z, r.z); r.w = fmaf(delta, z.w, r.w);
            }
            Y[row * G + c] = r;
            if (HAS_PUSH) halo_push_row(P, row, G, c, r);
        }
        const int64_t nrow = row + rows_per_cta;
        if (nrow < r1) { s = __ldg(indptr + nrow); e = __ldg(indptr + nrow + 1); }
    }
}

static int spmm_variant() {   // GEMB_SPMM=v1 selects the round-1 kernel (A/B runs); default v3
    static int v = -1;
    if (v < 0) { const char *e = getenv("GEMB_SPMM"); v = (e && e[0] == 'v' && e[1] == '1') ? 1 : 3; }
    return v;
}
static int spmm_tile_passes() {   // rows per tile = passes * (256 / G)
    static int t = -1;
    if (t < 0) { const char *e = getenv("GEMB_SPMM_PASSES"); t = e ? atoi(e) : 4; if (t < 1) t = 1; if (t > 16) t = 16; }
    return t;
}
int spmm_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, float alpha,
                const float *X, const float *X0, float *Y) {
    return spmm3_launch(ctx, A, n_rows, b, alpha, X, 0.f, nullptr, 1.f, X0, Y, nullptr);
}

int spmm3_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, float alpha, const float *X,
                 float gamma, const float *Xself, float delta, const float *X0, float *Y, const HaloPushArgs *push,
                 int64_t half_from) {
    GEMB_ARG(b > 0 && b % 4 == 0 && b <= 1024, "block width must be a multiple of 4, <= 1024");
    GEMB_ARG(half_from >= 0 && half_from < (int64_t)2147483647, "half_from");
    const int n_loc = (int)half_from;     // > 0: halo rows of X (column ids >= n_loc) are fp16 slots
    if (n_rows == 0) return GEMB_OK;
    const int G = b / 4;
    const int rows_per_cta = 256 / G;
    if (spmm_variant() == 3 && G <= 256 && n_rows >= 4096) {
        const int tile_rows = rows_per_cta * spmm_tile_passes();
        const int64_t n_tiles = (n_rows + tile_rows - 1) / tile_rows;
        GEMB_ARG(n_tiles < (int64_t)2147483647, "grid too large");
        const bool heavy3 = A.n_items > 0;
        const int hd = heavy3 ? SPMM_HEAVY_DEG : 0;
        HaloPushArgs PA3;
        memset(&PA3, 0, sizeof PA3);
        if (push) PA3 = *push;
        const float4 *X4 = (const float4 *)X, *X04 = (const float4 *)X0, *XS4 = (const float4 *)Xself;
        float4 *Y4 = (float4 *)Y;
#define LAUNCH3H(V, PU, Z, S, H)                                                                                         \
        spmm_bulk_kernel<V, PU, Z, S, H><<<(unsigned)n_tiles, 256, 0, ctx->stream>>>(A.indptr, A.indices, A.data, n_rows, A.nnz, G, rows_per_cta, \
                                                                                     tile_rows, alpha, gamma, delta, X4, XS4, X04, Y4, hd, PA3, n_loc)
#define LAUNCH3(V, PU, Z, S) do { if (n_loc > 0) LAUNCH3H(V, PU, Z, S, true); else LAUNCH3H(V, PU, Z, S, false); } while (0)
#define LAUNCH3B(V, PU)                                                                                                  \
        do {                                                                                                             \
            if (X0 && Xself) LAUNCH3(V, PU, true, true); else if (X0) LAUNCH3(V, PU, true, false);                       \
            else if (Xself) LAUNCH3(V, PU, false, true); else LAUNCH3(V, PU, false, false);                              \
        } while (0)
        if (A.data) { if (push) LAUNCH3B(true, true); else LAUNCH3B(true, false); }
        else { if (push) LAUNCH3B(false, true); else LAUNCH3B(false, false); }
#undef LAUNCH3B
#undef LAUNCH3
#undef LAUNCH3H
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        if (!heavy3) return GEMB_OK;
        return spmm_heavy_launch(ctx, A, b, alpha, X, gamma, Xself, delta, X0, Y, push, n_loc);
    }
    const int64_t grid = (n_rows + rows_per_cta - 1) / rows_per_cta;
    GEMB_ARG(grid < (int64_t)2147483647, "grid too large");
    dim3 g((unsigned)grid), t(256);
    const float4 *X4 = (const float4 *)X, *X04 = (const float4 *)X0, *XS4 = (const float4 *)Xself;
    float4 *Y4 = (float4 *)Y;
    const bool heavy = A.n_items > 0 && G <= 256;
    const int heavy_deg = heavy ? SPMM_HEAVY_DEG : 0;
    HaloPushArgs PA;
    memset(&PA, 0, sizeof PA);
    if (push) PA = *push;
#define LAUNCH1(V, Z, S, PU, H)                                                                                        \
    spmm_rowgroup_kernel<V, Z, S, PU, H><<<g, t, 0, ctx->stream>>>(A.indptr, A.indices, A.data, n_rows, G, rows_per_cta,      \
                                                                   alpha, gamma, delta, X4, XS4, X04, Y4, heavy_deg, PA, n_loc)
#define LAUNCH(V, Z, S)                                                                                      \
    do {                                                                                                     \
        if (push) { if (n_loc > 0) LAUNCH1(V, Z, S, true, true); else LAUNCH1(V, Z, S, true, false); }       \
        else { if (n_loc > 0) LAUNCH1(V, Z, S, false, true); else LAUNCH1(V, Z, S, false, false); }          \
    } while (0)
    const int sel = (A.data ? 4 : 0) | (X0 ? 2 : 0) | (Xself ? 1 : 0);
    switch (sel) {
        case 0: LAUNCH(false, false, false); break;
        case 1: LAUNCH(false, false, true); break;
        case 2: LAUNCH(false, true, false); break;
        case 3: LAUNCH(false, true, true); break;
        case 4: LAUNCH(true, false, false); break;
        case 5: LAUNCH(true, false, true); break;
        case 6: LAUNCH(true, true, false); break;
        default: LAUNCH(true, true, true); break;
    }
#undef LAUNCH
#undef LAUNCH1
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    if (heavy) return spmm_heavy_launch(ctx, A, b, alpha, X, gamma, Xself, delta, X0, Y, push, n_loc);
    return GEMB_OK;
}

int spmm_heavy_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int b, float alpha, const float *X, float gamma,
                      const float *Xself, float delta, const float *X0, float *Y, const HaloPushArgs *push, int n_loc) {
    const int G = b / 4;
    const int rows_per_cta = 256 / G;
    const float4 *X4 = (const float4 *)X, *X04 = (const float4 *)X0, *XS4 = (const float4 *)Xself;
    float4 *Y4 = (float4 *)Y;
    HaloPushArgs PA;
    memset(&PA, 0, sizeof PA);
    if (push) PA = *push;
    {
        const size_t need = sizeof(float) * (size_t)A.n_items * b;
        if (ctx->spmm_scratch_bytes < need) {
            GEMB_CUDA(dfree(ctx->spmm_scratch));
            ctx->spmm_scratch = nullptr; ctx->spmm_scratch_bytes = 0;
            GEMB_CUDA(dmalloc(&ctx->spmm_scratch, need));
            ctx->spmm_scratch_bytes = need;
        }
        float4 *P4 = (float4 *)ctx->spmm_scratch;
#define HP(V, H) spmm_heavy_partial_kernel<V, H><<<A.n_items, 256, 0, ctx->stream>>>(A.indptr, A.indices, A.data, A.item_row, A.item_beg, \
                                                                                  G, rows_per_cta, SPMM_HEAVY_CHUNK, X4, P4, n_loc)
        if (A.data) { if (n_loc > 0) HP(true, true); else HP(true, false); }
        else { if (n_loc > 0) HP(false, true); else HP(false, false); }
#undef HP
        GEMB_CUDA(cudaGetLastError());
        const int fgrid = (int)(((int64_t)A.n_heavy * G + 255) / 256);
#define FIN(Z, S) spmm_heavy_finish_kernel<Z, S><<<fgrid, 256, 0, ctx->stream>>>(A.n_heavy, A.heavy_row, A.heavy_first, G, alpha, gamma, \
                                                                               delta, P4, XS4, X04, Y4, push != nullptr, PA)
        if (X0 && Xself) FIN(true, true);
        else if (X0) FIN(true, false);
        else if (Xself) FIN(false, true);
        else FIN(false, false);
#undef FIN
        GEMB_CUDA(cudaGetLastError());
        count_launch(2);
    }
    return GEMB_OK;
}

}  // namespace gemb

using namespace gemb;

extern "C" int gemb_spmm(gemb_graph *g, int transpose, int b, float alpha, const float *X,
                         const float *X0, float *Y) {
    GEMB_ARG(g && X && Y, "graph/X/Y");
    GEMB_ARG(b > 0 && b % 4 == 0, "b must be a positive multiple of 4");
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    float *dX = nullptr, *dX0 = nullptr, *dY = nullptr;
    const size_t full = sizeof(float) * (size_t)g->n * b, shard = sizeof(float) * (size_t)g->n_local * b;
    GEMB_CUDA(dmalloc(&dX, full ? full : 4));
    GEMB_CUDA(dmalloc(&dY, shard ? shard : 4));
    if (X0) GEMB_CUDA(dmalloc(&dX0, shard ? shard : 4));
    GEMB_CUDA(cudaMemcpyAsync(dX, X, full, cudaMemcpyHostToDevice, c->stream));
    if (X0) GEMB_CUDA(cudaMemcpyAsync(dX0, X0, shard, cudaMemcpyHostToDevice, c->stream));
    int s = spmm_launch(c, transpose ? g->AT : g->A, g->n_local, b, alpha, dX, dX0, dY);
    if (s == GEMB_OK) {
        cudaError_t e = cudaMemcpyAsync(Y, dY, shard, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) {
            set_error("gemb_spmm: %s", cudaGetErrorString(e));
            s = GEMB_ERR_CUDA;
        }
    }
    dfree(dX);
    dfree(dY);
    dfree(dX0);
    return s;
}
