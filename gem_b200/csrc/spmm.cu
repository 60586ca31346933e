// gem_b200/csrc/spmm.cu -- CSR SpMM  Y = alpha * A * X  over an fp32 row-major block, with a fused epilogue that adds up
// to three more row blocks (SpmmEpilogue, common.cuh).
//
// Replaces the dense products hidden in hope.py:31 (inv(I - beta A) . beta A) and inside
// scipy's svds matvecs (hope.py:33): S is never formed, every S.x is a Horner sweep of this kernel.
//
// Mapping (HBM/L2-bound gather, SURVEY 8(d)): a group of G = b/4 threads owns one CSR row; thread
// c of the group owns columns [4c, 4c+4) of the block, so one nonzero = one coalesced 16*G-byte
// read of X[col, :] (320 B for b = 80) and the accumulators never leave registers.  Column ids and
// values of a row tile are staged in shared memory (spmm_bulk_kernel below).  The nonzero loop is
// unrolled by 4 so that each thread keeps 4 independent 16-byte gathers in flight.  The epilogue
// (the Horner step: X0 + alpha * acc) is fused: one extra coalesced read per operand.
#include "common.cuh"
#include <string.h>
#include <algorithm>
#include "tc_common.cuh"

namespace gemb {

__device__ __forceinline__ void fma4(float4 &a, float v, const float4 &x) {
    a.x = fmaf(v, x.x, a.x);
    a.y = fmaf(v, x.y, a.y);
    a.z = fmaf(v, x.z, a.z);
    a.w = fmaf(v, x.w, a.w);
}

// The epilogue of one finished row chunk (SpmmEpilogue): a * acc with a = alpha (HAS_SCALE: alpha * rscale[row]), then
// gamma * Xself, delta * X0 and eps * X1 added in this order by one fmaf each -- the order fixes the rounding.
template <bool HAS_X0, bool HAS_SELF, bool HAS_X1, bool HAS_SCALE>
__device__ __forceinline__ float4 spmm_epilogue(const float4 &acc, int64_t row, int G, int c, float alpha, float gamma,
                                                float delta, float eps, const float4 *__restrict__ Xself,
                                                const float4 *__restrict__ X0, const float4 *__restrict__ X1,
                                                const float *__restrict__ rscale) {
    const float a = HAS_SCALE ? alpha * __ldg(rscale + row) : alpha;
    float4 r = make_float4(a * acc.x, a * acc.y, a * acc.z, a * acc.w);
    if (HAS_SELF) fma4(r, gamma, __ldg(Xself + row * G + c));
    if (HAS_X0) fma4(r, delta, __ldg(X0 + row * G + c));
    if (HAS_X1) fma4(r, eps, __ldg(X1 + row * G + c));
    return r;
}

// ---- heavy rows (degree > SPMM_HEAVY_DEG; the hubs of a power-law graph -- R-MAT scale 21 has a 61 814-neighbour
// row, which one 20-thread group would walk for longer than the whole rest of the sweep takes).  Each chunk of
// SPMM_HEAVY_CHUNK nonzeros is one CTA: its row groups stride over the chunk, the group sums are added in a fixed
// order in shared memory, and the chunk sum goes to a scratch row; a second tiny kernel adds the chunk sums of a row
// in chunk order and applies the fused epilogue.  No atomics: the result is bit-reproducible.
template <bool HAS_VAL>
__global__ void __launch_bounds__(256)
spmm_heavy_partial_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                          const float *__restrict__ vals, const int32_t *__restrict__ item_row,
                          const int32_t *__restrict__ item_beg, int G, int groups, int chunk,
                          const float4 *__restrict__ X, float4 *__restrict__ partial) {
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
            const float4 x0 = __ldg(X + (int64_t)c0 * G + c), x1 = __ldg(X + (int64_t)c1 * G + c);
            const float4 x2 = __ldg(X + (int64_t)c2 * G + c), x3 = __ldg(X + (int64_t)c3 * G + c);
            fma4(acc, v0, x0); fma4(acc, v1, x1); fma4(acc, v2, x2); fma4(acc, v3, x3);
        }
        for (; i < end; i += groups) {
            const int c0 = __ldg(indices + i);
            const float v0 = HAS_VAL ? __ldg(vals + i) : 1.f;
            fma4(acc, v0, __ldg(X + (int64_t)c0 * G + c));
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

template <bool HAS_X0, bool HAS_SELF, bool HAS_X1, bool HAS_SCALE>
__global__ void __launch_bounds__(256)
spmm_heavy_finish_kernel(int n_heavy, const int32_t *__restrict__ heavy_row, const int32_t *__restrict__ heavy_first,
                         int G, float alpha, float gamma, float delta, const float4 *__restrict__ partial,
                         const float4 *__restrict__ Xself, const float4 *__restrict__ X0, float4 *__restrict__ Y,
                         bool has_push, HaloPushArgs P, float eps, const float4 *__restrict__ X1,
                         const float *__restrict__ rscale) {
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
    const float4 r =
        spmm_epilogue<HAS_X0, HAS_SELF, HAS_X1, HAS_SCALE>(acc, row, G, c, alpha, gamma, delta, eps, Xself, X0, X1, rscale);
    Y[row * G + c] = r;
    if (has_push) halo_push_row(P, row, G, c, r);
}

// Y[row] = alpha * (A X)[row] + gamma * Xself[row] + delta * X0[row] (+ eps * X1[row])
//   HAS_SCALE: alpha * rscale[row] multiplies the row's sum instead of alpha (Y = alpha diag(s) A X; the first sweep of
//   the Adamic-Adar operator A D A, hope.cu, spectral_mode 4)
//   Horner / Katz sweep:      gamma = 0, delta = 1, X0 = the sweep's input block
//   Chebyshev three-term step: gamma = -2 s c0 / e (current block), delta = -s s' (previous block)
//   the same step on the composite operator -M^T M, M = I - A (hope.cu, spectral_mode 2): the second sweep gathers
//   T = X - A X through A^T and needs T, the current and the previous block: Xself = T, X0 = current, X1 = previous
// One CTA per row TILE (SPMM_TILE_PASSES * rows_per_cta consecutive rows); the tile's slice of the column-id (and value)
// arrays -- one contiguous range of the CSR -- is staged into shared memory by ONE TMA bulk copy (cp.async.bulk +
// mbarrier complete_tx) issued by thread 0 while every row group fetches its row offsets; the other resident CTAs of the
// SM hide the copy's latency.  The row groups then read their column ids from shared memory: the dependent chain per row
// drops from indptr -> indices -> X (three global round trips) to indptr -> X, and the ~nnz/4 broadcast LDGs of reading
// the ids through the read-only path (one L1 wavefront each) leave the L1 data pipe to the gathers.  scripts/spmm_lab.cu
// times variants of this layout against each other.  A tile whose slice exceeds the staging buffer (hubs) reads its ids
// from global memory; rows above SPMM_HEAVY_DEG go to the chunk kernels.
// HAS_PUSH (multi-GPU, halo.cu): the finished row is also stored into the halo slots of the peers whose shards
// reference it -- 16-byte posted stores over NVLink, issued while the other row groups of the SM are still gathering.
constexpr int BULK_CAP = 3072;                 // staged ids per tile (+ up to 3 of alignment slack + 4 of over-read)
constexpr int SPMM_TILE_PASSES = 4;            // rows per tile = passes * (256 / G)
template <bool HAS_VAL, bool HAS_PUSH, bool HAS_X0, bool HAS_SELF, bool HAS_X1, bool HAS_SCALE = false>
__global__ void __launch_bounds__(256)
spmm_bulk_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                 const float *__restrict__ vals, int64_t n_rows, int64_t nnz, int G, int rows_per_cta, int tile_rows,
                 float alpha, float gamma, float delta, const float4 *__restrict__ X,
                 const float4 *__restrict__ Xself, const float4 *__restrict__ X0, float4 *__restrict__ Y,
                 int heavy_deg, HaloPushArgs P, float eps, const float4 *__restrict__ X1,
                 const float *__restrict__ rscale) {
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
                    const float4 x0 = __ldg(X + (int64_t)c0 * G + c), x1 = __ldg(X + (int64_t)c1 * G + c);
                    const float4 x2 = __ldg(X + (int64_t)c2 * G + c), x3 = __ldg(X + (int64_t)c3 * G + c);
                    fma4(acc, HAS_VAL ? lv[i] : 1.f, x0); fma4(acc, HAS_VAL ? lv[i + 1] : 1.f, x1);
                    fma4(acc, HAS_VAL ? lv[i + 2] : 1.f, x2); fma4(acc, HAS_VAL ? lv[i + 3] : 1.f, x3);
                }
                for (; i < e; i++) fma4(acc, HAS_VAL ? lv[i] : 1.f, __ldg(X + (int64_t)li[i] * G + c));
            } else {
                for (; i + 4 <= e; i += 4) {
                    const int c0 = __ldg(indices + i), c1 = __ldg(indices + i + 1);
                    const int c2 = __ldg(indices + i + 2), c3 = __ldg(indices + i + 3);
                    const float4 x0 = __ldg(X + (int64_t)c0 * G + c), x1 = __ldg(X + (int64_t)c1 * G + c);
                    const float4 x2 = __ldg(X + (int64_t)c2 * G + c), x3 = __ldg(X + (int64_t)c3 * G + c);
                    fma4(acc, HAS_VAL ? __ldg(vals + i) : 1.f, x0); fma4(acc, HAS_VAL ? __ldg(vals + i + 1) : 1.f, x1);
                    fma4(acc, HAS_VAL ? __ldg(vals + i + 2) : 1.f, x2); fma4(acc, HAS_VAL ? __ldg(vals + i + 3) : 1.f, x3);
                }
                for (; i < e; i++) fma4(acc, HAS_VAL ? __ldg(vals + i) : 1.f, __ldg(X + (int64_t)__ldg(indices + i) * G + c));
            }
            const float4 r = spmm_epilogue<HAS_X0, HAS_SELF, HAS_X1, HAS_SCALE>(acc, row, G, c, alpha, gamma, delta, eps,
                                                                                Xself, X0, X1, rscale);
            Y[row * G + c] = r;
            if (HAS_PUSH) halo_push_row(P, row, G, c, r);
        }
        const int64_t nrow = row + rows_per_cta;
        if (nrow < r1) { s = __ldg(indptr + nrow); e = __ldg(indptr + nrow + 1); }
    }
}

// One sweep with the epilogue's operand set fixed at compile time: the bulk kernel over every row tile, then, when A has
// heavy rows, their chunk sums (into ctx->spmm_scratch, grown on demand) and the finish kernel with the same epilogue.
template <bool HAS_PUSH, bool HAS_X0, bool HAS_SELF, bool HAS_X1, bool HAS_SCALE>
static int spmm_sweep(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, const float *X, float *Y,
                      const SpmmEpilogue &e) {
    const int G = b / 4;
    const int rows_per_cta = 256 / G;
    const int tile_rows = rows_per_cta * SPMM_TILE_PASSES;
    const int64_t n_tiles = (n_rows + tile_rows - 1) / tile_rows;
    GEMB_ARG(n_tiles < (int64_t)2147483647, "grid too large");
    const bool heavy = A.n_items > 0;
    HaloPushArgs PA;
    memset(&PA, 0, sizeof PA);
    if (HAS_PUSH) PA = *e.push;
    const float4 *X4 = (const float4 *)X, *XS4 = (const float4 *)e.Xself, *X04 = (const float4 *)e.X0;
    const float4 *X14 = (const float4 *)e.X1;
    float4 *Y4 = (float4 *)Y;
    auto bulk = A.data ? spmm_bulk_kernel<true, HAS_PUSH, HAS_X0, HAS_SELF, HAS_X1, HAS_SCALE>
                       : spmm_bulk_kernel<false, HAS_PUSH, HAS_X0, HAS_SELF, HAS_X1, HAS_SCALE>;
    GEMB_TRY(launch(ctx, bulk, (unsigned)n_tiles, 256, 0, A.indptr, A.indices, A.data, n_rows, A.nnz, G, rows_per_cta, tile_rows,
                    e.alpha, e.gamma, e.delta, X4, XS4, X04, Y4, heavy ? SPMM_HEAVY_DEG : 0, PA, e.eps, X14, e.rscale));
    if (!heavy) return GEMB_OK;
    const size_t need = sizeof(float) * (size_t)A.n_items * b;
    if (ctx->spmm_scratch_bytes < need) {
        GEMB_CUDA(dfree(ctx->spmm_scratch));
        ctx->spmm_scratch = nullptr; ctx->spmm_scratch_bytes = 0;
        GEMB_CUDA(dmalloc(&ctx->spmm_scratch, need));
        ctx->spmm_scratch_bytes = need;
    }
    float4 *P4 = (float4 *)ctx->spmm_scratch;
    auto partial = A.data ? spmm_heavy_partial_kernel<true> : spmm_heavy_partial_kernel<false>;
    GEMB_TRY(launch(ctx, partial, A.n_items, 256, 0, A.indptr, A.indices, A.data, A.item_row, A.item_beg, G, rows_per_cta,
                    SPMM_HEAVY_CHUNK, X4, P4));
    const int fgrid = (int)(((int64_t)A.n_heavy * G + 255) / 256);
    return launch(ctx, spmm_heavy_finish_kernel<HAS_X0, HAS_SELF, HAS_X1, HAS_SCALE>, fgrid, 256, 0, A.n_heavy, A.heavy_row,
                  A.heavy_first, G, e.alpha, e.gamma, e.delta, P4, XS4, X04, Y4, HAS_PUSH, PA, e.eps, X14, e.rscale);
}

int spmm_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, const float *X, float *Y,
                const SpmmEpilogue &e) {
    GEMB_ARG(!e.X1 || (e.Xself && e.X0), "the fourth epilogue operand needs Xself and X0");
    GEMB_ARG(!e.X1 || !e.push, "the fourth epilogue operand is single-GPU");
    GEMB_ARG(!e.rscale || (!e.Xself && !e.X0 && !e.X1 && !e.push), "the row scale takes no other epilogue operand");
    GEMB_ARG(b > 0 && b % 4 == 0 && b <= 1024, "block width must be a multiple of 4, <= 1024");
    if (n_rows == 0) return GEMB_OK;
    //                                    PUSH   X0     SELF   X1     SCALE
    if (e.rscale) return spmm_sweep<false, false, false, false, true>(ctx, A, n_rows, b, X, Y, e);
    if (e.X1) return spmm_sweep<false, true, true, true, false>(ctx, A, n_rows, b, X, Y, e);
    if (e.push) {
        if (e.X0 && e.Xself) return spmm_sweep<true, true, true, false, false>(ctx, A, n_rows, b, X, Y, e);
        if (e.X0) return spmm_sweep<true, true, false, false, false>(ctx, A, n_rows, b, X, Y, e);
        if (e.Xself) return spmm_sweep<true, false, true, false, false>(ctx, A, n_rows, b, X, Y, e);
        return spmm_sweep<true, false, false, false, false>(ctx, A, n_rows, b, X, Y, e);
    }
    if (e.X0 && e.Xself) return spmm_sweep<false, true, true, false, false>(ctx, A, n_rows, b, X, Y, e);
    if (e.X0) return spmm_sweep<false, true, false, false, false>(ctx, A, n_rows, b, X, Y, e);
    if (e.Xself) return spmm_sweep<false, false, true, false, false>(ctx, A, n_rows, b, X, Y, e);
    return spmm_sweep<false, false, false, false, false>(ctx, A, n_rows, b, X, Y, e);
}

// The sweep of the test hooks from host memory: X (all n rows) and the epilogue's blocks (the shard's rows) to the
// device, one sweep of A or A^T over the shard, Y back.
static int spmm_host(gemb_graph *g, int transpose, int b, const float *X, SpmmEpilogue e, float *Y) {
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    DeviceBuffer<float> dX, dY, dXs, dX0, dX1, dS;
    const size_t shard = (size_t)g->n_local * b;
    GEMB_CUDA(dX.upload(X, (size_t)g->n * b, c->stream));
    if (e.Xself) GEMB_CUDA(dXs.upload(e.Xself, shard, c->stream));   // an absent operand stays a null pointer
    if (e.X0) GEMB_CUDA(dX0.upload(e.X0, shard, c->stream));
    if (e.X1) GEMB_CUDA(dX1.upload(e.X1, shard, c->stream));
    if (e.rscale) GEMB_CUDA(dS.upload(e.rscale, (size_t)g->n_local, c->stream));
    GEMB_CUDA(dY.alloc(shard));
    e.Xself = dXs.get(); e.X0 = dX0.get(); e.X1 = dX1.get(); e.rscale = dS.get();
    GEMB_TRY(spmm_launch(c, transpose ? g->AT : g->A, g->n_local, b, dX.get(), dY.get(), e));
    return copy_sync(c, Y, dY.get(), sizeof(float) * shard, cudaMemcpyDeviceToHost);
}

}  // namespace gemb

using namespace gemb;

extern "C" int gemb_spmm(gemb_graph *g, int transpose, int b, float alpha, const float *X, float gamma,
                         const float *Xself, float delta, const float *X0, float *Y) {
    return gemb_spmm4(g, transpose, b, alpha, X, gamma, Xself, delta, X0, 0.f, nullptr, Y);
}

extern "C" int gemb_spmm4(gemb_graph *g, int transpose, int b, float alpha, const float *X, float gamma,
                          const float *Xself, float delta, const float *X0, float eps, const float *X1, float *Y) {
    GEMB_ARG(g && X && Y, "graph/X/Y");
    GEMB_ARG(b > 0 && b % 4 == 0, "b must be a positive multiple of 4");
    GEMB_ARG(!X1 || (Xself && X0), "X1 needs Xself and X0");
    GEMB_ARG(!X1 || g->n_local == g->n, "the fourth epilogue operand is single-GPU");
    return spmm_host(g, transpose, b, X,
                     {.alpha = alpha, .gamma = gamma, .Xself = Xself, .delta = delta, .X0 = X0, .eps = eps, .X1 = X1}, Y);
}

extern "C" int gemb_spmm_scaled(gemb_graph *g, int transpose, int b, float alpha, const float *X, const float *rscale,
                                float *Y) {
    GEMB_ARG(g && X && rscale && Y, "graph/X/rscale/Y");
    GEMB_ARG(b > 0 && b % 4 == 0, "b must be a positive multiple of 4");
    gemb_ctx *c = g->ctx;
    GEMB_ARG(c->nranks == 1 && g->n_local == g->n, "gemb_spmm_scaled is single-GPU");
    return spmm_host(g, transpose, b, X, {.alpha = alpha, .rscale = rscale}, Y);
}
