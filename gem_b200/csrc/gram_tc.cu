// gem_b200/csrc/gram_tc.cu -- the tall-skinny Gram contraction G = P^T Q on the Hopper tensor cores (wgmma).
//
// This is the ONE dense contraction of the HOPE solver (CholeskyQR Gram and the Rayleigh-Ritz
// projection; replaces numpy.linalg.qr / svd inside scipy svds, _svds.py:508-533).  It is memory bound
// (read n*b fp32 once), so the kernel is a persistent streaming design, one CTA per SM, three warpgroups:
//
//   loader (warpgroup 2)   : thread 256 issues the TMA bulk copies -- a stage of <= 64 rows is one contiguous piece of
//                            the row-major block, three raw stages in flight, mbarrier complete_tx.  The four warps
//                            read each raw stage (lane -> column, 4 consecutive rows: conflict-free LDS.32), split
//                            x = hi + lo with hi = rna_tf32(x), lo = rna_tf32(x - hi), and write two STS.128 into the
//                            K-major / no-swizzle wgmma layout (element (mn, k) -> (mn/8)*SBO + (mn%8)*16 + (k/4)*LBO
//                            + (k%4)*4) of one of two tile buffers
//   MMA (warpgroups 0, 1)  : warpgroup w owns rows 64w .. 64w+63 of the G block; per 8-row k-block three
//                            wgmma.mma_async m64nNk8 tf32 (hi*hi + hi*lo + lo*hi = "3xTF32", ~fp32 accuracy), N = 32..128
// A launch computes one block G[m0 : m0+mb, n0 : n0+nb] (mb, nb <= 128) from whole raw rows; wider blocks take several
// launches.  Every CTA stores its partial block, and the partials are added in a fixed order (sum_partials_launch).
// The contraction index is the ROW index of the row-major blocks, i.e. A = P^T and B = Q^T arrive MN-major; wgmma takes
// tf32 operands K-major only, so the loader transposes on the way into shared memory.
#include "tc_common.cuh"

namespace gemb {

struct GramTcParams {
    int64_t n;
    const float *P, *Q;
    int ldp, ldq;        // columns of the raw rows of P and Q
    int m0, n0, mb, nb;  // the block: columns m0 .. m0+mb-1 of P against n0 .. n0+nb-1 of Q (of P when Q is not staged)
    double *part;        // partials: part[cta * part_stride + row * ldg + col] of the whole G
    int ldg;
    int64_t part_stride;
    int stage_rows;      // multiple of 8
    uint32_t tile_bytes_a, tile_bytes_b;   // bytes of one (hi or lo) tile
    uint32_t raw_bytes_p, raw_bytes_q;     // bytes of one raw (row-major fp32) stage
};

// one unit = 4 rows x 32 columns of the RAW stage (row-major fp32, as it lies in global memory): lane -> column
// mn = j32*32 + lane reads rows k4*4 .. k4*4+3 (four conflict-free LDS.32), i.e. exactly the 16-byte K chunk the
// K-major tile wants -- no register transpose.  Rows >= valid_rows read as zero.
// Columns c0 .. c0+w-1 of raw rows of `ld` floats.
__device__ __forceinline__ void transform_unit(const char *raw, int ld, int c0, int w, int valid_rows, int k4, int j32,
                                               int lane, char *tile_hi, char *tile_lo, uint32_t lbo, uint32_t sbo) {
    const int mn = j32 * 32 + lane;
    if (mn >= w) return;
    const int k0 = k4 * 4;
    const float *src = (const float *)raw + (size_t)k0 * ld + c0 + mn;
    float4 v;
    v.x = (k0 + 0 < valid_rows) ? src[0] : 0.f;
    v.y = (k0 + 1 < valid_rows) ? src[(size_t)ld] : 0.f;
    v.z = (k0 + 2 < valid_rows) ? src[2 * (size_t)ld] : 0.f;
    v.w = (k0 + 3 < valid_rows) ? src[3 * (size_t)ld] : 0.f;
    uint4 hi, lo;
    tc::split_tf32(v, hi, lo);
    const uint32_t off = (uint32_t)(mn >> 3) * sbo + (uint32_t)(mn & 7) * 16u + (uint32_t)k4 * lbo;
    *(uint4 *)(tile_hi + off) = hi;
    *(uint4 *)(tile_lo + off) = lo;
}

// QRAW: the raw stages hold rows of Q after those of P (cross Gram).  BSEP: the B tile is built separately (cross Gram or an
// off-diagonal block); otherwise B = A.  NPAD = accumulator width (N of the MMA, >= nb).  Hand-offs are mbarriers:
//   s_full[3]       TMA complete_tx -> loader warps        (raw stage landed)
//   s_tile_full[2]  loader warps (4 arrivals) -> MMA       (hi / lo tiles written)
//   s_tile_free[2]  MMA warps (8 arrivals) -> loader warps (the MMAs that read the tiles are complete)
// A raw slot is refilled by thread 256 once the four loader warps passed named barrier 1 after reading it.
// Accumulation is two-level: every stage (<= 64 rows) accumulates into a FRESH register accumulator (the tensor core
// does not round its fp32 additions to nearest, which biases long sums of positive terms such as the diagonal), and the
// finished stage is folded into a second fp32 accumulator with round-to-nearest adds while the loader prepares the next.
template <bool QRAW, bool BSEP, int NPAD>
__global__ void __launch_bounds__(384, 1) gram_tc_kernel(GramTcParams p) {
    extern __shared__ __align__(128) char smem[];
    __shared__ __align__(8) uint64_t s_full[3], s_tile_full[2], s_tile_free[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int kblocks = p.stage_rows / 8;              // MMA k-steps (K = 8 rows) per stage
    const int kquads = p.stage_rows / 4;               // 16-byte K chunks per stage
    const uint32_t lbo = 128u;                         // consecutive K chunks of one 8-column group are adjacent
    const uint32_t sbo = (uint32_t)kquads * 128u;      // stride between 8-column (MN) groups
    // shared memory: 3 raw stages [P | (Q)] filled by TMA bulk copies, then 2 tile stages [P_hi | P_lo | (Q_hi | Q_lo)]
    const uint32_t raw_stage = p.raw_bytes_p + (QRAW ? p.raw_bytes_q : 0);
    const uint32_t stage_bytes = 2 * p.tile_bytes_a + (BSEP ? 2 * p.tile_bytes_b : 0);
    char *raw_base = smem;
    char *tile_base = smem + 3 * (size_t)raw_stage;

    if (tid == 0) {
        for (int i = 0; i < 2; i++) { tc::mbar_init(tc::smem_u32(&s_tile_full[i]), 4); tc::mbar_init(tc::smem_u32(&s_tile_free[i]), 8); }
        for (int i = 0; i < 3; i++) tc::mbar_init(tc::smem_u32(&s_full[i]), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // contiguous row range of this CTA, in whole stages
    const int64_t stages_total = (p.n + p.stage_rows - 1) / p.stage_rows;
    const int64_t per_cta = (stages_total + gridDim.x - 1) / gridDim.x;
    const int64_t s_begin = (int64_t)blockIdx.x * per_cta;
    const int64_t s_end = s_begin + per_cta < stages_total ? s_begin + per_cta : stages_total;
    const int nst = (int)(s_end > s_begin ? s_end - s_begin : 0);

    if (warp >= 8) {
        // ================= loader warpgroup: TMA producer (thread 256) + raw -> hi / lo tiles =================
        const int lw = warp - 8;
        auto issue = [&](int it) {
            const int slot = it % 3;
            const int64_t row0 = (s_begin + it) * p.stage_rows;
            const int64_t vr = p.n - row0 < p.stage_rows ? p.n - row0 : p.stage_rows;
            const uint32_t bytes_p = (uint32_t)(vr * p.ldp * 4), bytes_q = QRAW ? (uint32_t)(vr * p.ldq * 4) : 0u;
            const uint32_t bar = tc::smem_u32(&s_full[slot]);
            char *dst = raw_base + (size_t)slot * raw_stage;
            tc::mbar_expect_tx(bar, bytes_p + bytes_q);
            tc::bulk_g2s(tc::smem_u32(dst), p.P + row0 * p.ldp, bytes_p, bar);
            if (QRAW) tc::bulk_g2s(tc::smem_u32(dst + p.raw_bytes_p), p.Q + row0 * p.ldq, bytes_q, bar);
        };
        if (tid == 256)
            for (int it = 0; it < 3 && it < nst; it++) issue(it);
        for (int it = 0; it < nst; it++) {
            const int st = it & 1, slot = it % 3;
            char *base = tile_base + (size_t)st * stage_bytes;
            const char *raw = raw_base + (size_t)slot * raw_stage;
            tc::mbar_wait(tc::smem_u32(&s_full[slot]), (uint32_t)(it / 3) & 1);                // stage `it` has landed
            if (it >= 2) tc::mbar_wait(tc::smem_u32(&s_tile_free[st]), (uint32_t)((it >> 1) - 1) & 1);   // MMAs of it-2 done
            const int64_t row0 = (s_begin + it) * p.stage_rows;
            const int vr = (int)(p.n - row0 < p.stage_rows ? p.n - row0 : p.stage_rows);
            const int units_a = kquads * ((p.mb + 31) / 32);
#pragma unroll 3
            for (int u = lw; u < units_a; u += 4)
                transform_unit(raw, p.ldp, p.m0, p.mb, vr, u % kquads, u / kquads, lane, base, base + p.tile_bytes_a, lbo, sbo);
            if (BSEP) {
                const int units_b = kquads * ((p.nb + 31) / 32);
                char *qb = base + 2 * p.tile_bytes_a;
                const char *rb = QRAW ? raw + p.raw_bytes_p : raw;
                const int ldb = QRAW ? p.ldq : p.ldp;
#pragma unroll 3
                for (int u = lw; u < units_b; u += 4)
                    transform_unit(rb, ldb, p.n0, p.nb, vr, u % kquads, u / kquads, lane, qb, qb + p.tile_bytes_b, lbo, sbo);
            }
            tc::fence_proxy_async();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(tc::smem_u32(&s_tile_full[st]));
            tc::named_sync(1, 128);                                                              // raw slot fully read
            if (tid == 256 && it + 3 < nst) issue(it + 3);
        }
    } else {
        // ================= MMA warpgroups 0, 1: rows 64*wg .. 64*wg + 63 of G =================
        const int wg = warp >> 2;
        const bool active = wg * 64 < p.mb;                 // warpgroup-uniform
        float acc[NPAD / 2], racc[NPAD / 2];
#pragma unroll
        for (int i = 0; i < NPAD / 2; i++) racc[i] = 0.f;
        for (int it = 0; it < nst; it++) {
            const int st = it & 1;
            tc::mbar_wait(tc::smem_u32(&s_tile_full[st]), (uint32_t)(it >> 1) & 1);            // tiles of stage `it` written
            if (active) {
                const uint32_t a_hi = tc::smem_u32(tile_base + (size_t)st * stage_bytes), a_lo = a_hi + p.tile_bytes_a;
                const uint32_t b_hi = BSEP ? a_hi + 2 * p.tile_bytes_a : a_hi;
                const uint32_t b_lo = BSEP ? b_hi + p.tile_bytes_b : a_lo;
                const uint32_t a_off = (uint32_t)wg * 8u * sbo;                                   // this warpgroup's 64 rows
                uint64_t dah = tc::make_desc(a_hi + a_off, lbo, sbo), dal = tc::make_desc(a_lo + a_off, lbo, sbo);
                uint64_t dbh = tc::make_desc(b_hi, lbo, sbo), dbl = tc::make_desc(b_lo, lbo, sbo);
                const uint64_t step = (uint64_t)((2u * lbo) >> 4);                                // one MMA consumes two K chunks
                tc::wgmma_fence();
                for (int kb = 0; kb < kblocks; kb++) {
                    tc::wgmma_tf32<NPAD>(acc, dah, dbh, kb > 0 ? 1u : 0u);
                    tc::wgmma_tf32<NPAD>(acc, dah, dbl, 1u);
                    tc::wgmma_tf32<NPAD>(acc, dal, dbh, 1u);
                    dah += step; dal += step; dbh += step; dbl += step;
                }
                tc::wgmma_commit();
                tc::wgmma_wait_all();
            }
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(tc::smem_u32(&s_tile_free[st]));
            if (active) {
#pragma unroll
                for (int i = 0; i < NPAD / 2; i++) racc[i] += acc[i];
            }
        }
        if (active) {                                         // every CTA stores its block (zeros when it had no rows)
            const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
            double *dst = p.part + (size_t)blockIdx.x * p.part_stride + (size_t)p.m0 * p.ldg + p.n0;
#pragma unroll
            for (int i = 0; i < NPAD / 2; i++) {
                const int row = r0 + ((i >> 1) & 1) * 8, col = (i >> 2) * 8 + (lane & 3) * 2 + (i & 1);
                if (row < p.mb && col < p.nb) dst[(size_t)row * p.ldg + col] = (double)racc[i];
            }
        }
    }
}

template <bool QRAW, bool BSEP, int NPAD>
static int gram_tc_launch_t(gemb_ctx *ctx, const GramTcParams &p, int grid, size_t smem_bytes) {
    static size_t attr_bytes = 0;
    if (attr_bytes < smem_bytes) {
        GEMB_CUDA(cudaFuncSetAttribute(gram_tc_kernel<QRAW, BSEP, NPAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
        attr_bytes = smem_bytes;
    }
    return launch(ctx, gram_tc_kernel<QRAW, BSEP, NPAD>, grid, 384, smem_bytes, p);
}

template <bool QRAW, bool BSEP>
static int gram_tc_dispatch(gemb_ctx *ctx, const GramTcParams &p, int grid, size_t smem_bytes) {
    // accumulator width: one of 32 / 64 / 80 / 96 / 128 columns
    if (p.nb <= 32) return gram_tc_launch_t<QRAW, BSEP, 32>(ctx, p, grid, smem_bytes);
    if (p.nb <= 64) return gram_tc_launch_t<QRAW, BSEP, 64>(ctx, p, grid, smem_bytes);
    if (p.nb <= 80) return gram_tc_launch_t<QRAW, BSEP, 80>(ctx, p, grid, smem_bytes);
    if (p.nb <= 96) return gram_tc_launch_t<QRAW, BSEP, 96>(ctx, p, grid, smem_bytes);
    return gram_tc_launch_t<QRAW, BSEP, 128>(ctx, p, grid, smem_bytes);
}

// returns GEMB_ERR_UNSUPPORTED (without setting an error) when the shape does not fit this kernel
int gram_tc_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G) {
    const bool cross = (P != Q);
    if (b1 % 4 || b2 % 4 || n <= 0) return GEMB_ERR_UNSUPPORTED;
    // G is computed in blocks of <= 128 x 128; all launches share one stage size (hence one grid and one partial layout)
    const int bm = (b1 + 127) / 128, bn = (b2 + 127) / 128;
    const size_t cols_raw = (size_t)b1 + (cross ? b2 : 0);
    size_t cols_tile = 0;
    for (int i = 0; i < bm; i++)
        for (int j = 0; j < bn; j++) {
            const int mb = std::min(128, b1 - 128 * i), nb = std::min(128, b2 - 128 * j);
            const bool bsep = cross || i != j;
            cols_tile = std::max(cols_tile, (size_t)(mb + 7) / 8 * 8 + (bsep ? (size_t)(nb + 7) / 8 * 8 : 0));
        }
    // stage rows: largest multiple of 8 (<= 64) such that 3 raw stages + 2 tile stages (hi + lo) fit in ~176 KB
    const size_t bytes_per_row = 3 * 4 * cols_raw + 2 * 2 * 4 * cols_tile;
    int rows = (int)((176 * 1024) / bytes_per_row) / 8 * 8;
    if (rows > 64) rows = 64;
    if (rows < 8) return GEMB_ERR_UNSUPPORTED;
    const size_t sbo = (size_t)(rows / 4) * 128;
    const size_t raw_stage = (size_t)rows * cols_raw * 4;
    // the MMAs read 16 column groups of A (two warpgroups x 64 rows) and NPAD/8 <= 16 groups of B even where the block is
    // narrower: keep those (ignored) reads inside the allocation
    const size_t smem_bytes = 3 * raw_stage + 2 * cols_tile / 8 * 2 * sbo + 16 * sbo + 1024;
    if (smem_bytes > 226 * 1024) return GEMB_ERR_UNSUPPORTED;   // + ~64 B of static shared memory <= 227 KB
    const int64_t stages_total = (n + rows - 1) / rows;
    int grid = ctx->sm_count;
    if (grid > stages_total) grid = (int)stages_total;
    double *part = nullptr;
    GEMB_TRY(red_scratch(ctx, (size_t)grid * b1 * b2, &part));
    GramTcParams p;
    p.n = n; p.P = P; p.Q = Q; p.ldp = b1; p.ldq = b2;
    p.part = part; p.ldg = b2; p.part_stride = (int64_t)b1 * b2;
    p.stage_rows = rows;
    p.raw_bytes_p = (uint32_t)(rows * b1 * 4);
    p.raw_bytes_q = (uint32_t)(rows * b2 * 4);
    for (int i = 0; i < bm; i++)
        for (int j = 0; j < bn; j++) {
            p.m0 = 128 * i; p.mb = std::min(128, b1 - p.m0);
            p.n0 = 128 * j; p.nb = std::min(128, b2 - p.n0);
            p.tile_bytes_a = (uint32_t)((p.mb + 7) / 8) * (uint32_t)(rows / 4) * 128u;
            p.tile_bytes_b = (uint32_t)((p.nb + 7) / 8) * (uint32_t)(rows / 4) * 128u;
            if (cross) GEMB_TRY((gram_tc_dispatch<true, true>(ctx, p, grid, smem_bytes)));
            else if (i != j) GEMB_TRY((gram_tc_dispatch<false, true>(ctx, p, grid, smem_bytes)));
            else GEMB_TRY((gram_tc_dispatch<false, false>(ctx, p, grid, smem_bytes)));
        }
    return sum_partials_launch(ctx, grid, (int64_t)b1 * b2, part, G);
}

}  // namespace gemb
