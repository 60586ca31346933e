// gem_b200/csrc/apply_tc.cu -- the tall-skinny product Out = Q * M (n x b1 times b1 x b2) on the Hopper tensor cores
// (wgmma): the second half of CholeskyQR (Q R^-1) and the Ritz rotation (replaces the GEMMs inside numpy.linalg.qr /
// svd of scipy svds, _svds.py:508-533).  Memory bound (read n*b1, write n*b2 fp32), persistent, one CTA per SM, three
// warpgroups, tiles of TILE_M = 128 rows (64 where shared memory is short: then warpgroup 1 has no MMA work):
//
//   loader (warpgroup 2) : thread 256 issues a TMA bulk copy of TILE_M consecutive rows of Q (one contiguous piece of the
//                          row-major block) into a 2-slot raw ring; the four warps turn the raw rows into the K-major /
//                          no-swizzle wgmma tile, splitting x = hi + lo (rna_tf32) on the way -- for A = Q the 16-byte K
//                          chunk is 4 consecutive floats of a row, i.e. a straight copy
//   MMA (warpgroups 0, 1): warpgroup w owns rows 64w .. 64w+63 of the tile: 3 * b1/8 wgmma.mma_async m64nNk8 tf32
//                          (hi*hi + hi*lo + lo*hi, "3xTF32"), N = 32..128, accumulator in registers, then the epilogue
//                          stores its fragment straight from registers (8-byte stores, whole 32-byte sectors per row)
//   B = M^T (K-major) is split once per CTA and stays resident in shared memory.  Out columns beyond what one B tile
//   holds are computed by further launches over column blocks of M and Out.
#include "tc_common.cuh"

namespace gemb {

struct ApplyTcParams {
    int64_t n;
    const float *Q;      // n x b1
    const float *M;      // b1 x b2, leading dimension ldm
    float *Out;          // n x b2, leading dimension ldo (>= b2, even)
    int b1, b2, ldm, ldo;
    uint32_t a_lbo;      // byte stride between 16-byte K chunks of the A tile (16 * TILE_M + 16: bank-conflict free stores)
    uint32_t a_tile;     // bytes of one (hi or lo) A tile
    uint32_t b_tile;     // bytes of one (hi or lo) B tile
    uint32_t raw_slot;   // bytes of one raw slot
};

// Hand-offs (mbarriers): s_full[2] TMA complete_tx -> loader warps; s_tile_full loader warps (4 arrivals) -> MMA;
// s_tile_free MMA warps (8 arrivals) -> loader warps (the MMAs that read the single A tile are complete).
template <int TILE_M, int NPAD>
__global__ void __launch_bounds__(384, 1) apply_tc_kernel(ApplyTcParams p) {
    extern __shared__ __align__(128) char smem[];
    __shared__ __align__(8) uint64_t s_full[2], s_tile_full, s_tile_free;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int kchunks = p.b1 / 4;                 // 16-byte K chunks per row
    const int ksteps = p.b1 / 8;                  // MMAs (K = 8) per split product
    const uint32_t a_sbo = 128u;                  // 8-row groups of the A tile are adjacent
    const uint32_t b_lbo = 128u;                  // B tile: consecutive K chunks of one 8-column group are adjacent
    const uint32_t b_sbo = (uint32_t)kchunks * 128u;
    // shared memory: [raw 0 | raw 1 | A_hi | A_lo | B_hi | B_lo]
    char *raw_base = smem;
    char *a_hi = smem + 2 * (size_t)p.raw_slot, *a_lo = a_hi + p.a_tile;
    char *b_hi = a_lo + p.a_tile, *b_lo = b_hi + p.b_tile;

    if (tid == 0) {
        for (int i = 0; i < 2; i++) tc::mbar_init(tc::smem_u32(&s_full[i]), 1);
        tc::mbar_init(tc::smem_u32(&s_tile_full), 4);
        tc::mbar_init(tc::smem_u32(&s_tile_free), 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // ---- B = M^T, K-major: element (n, k) = M[k][n]  ->  (n/8)*b_sbo + (n%8)*16 + (k/4)*b_lbo + (k%4)*4
    for (int idx = tid; idx < NPAD * kchunks; idx += blockDim.x) {
        const int nn = idx % NPAD, kc = idx / NPAD;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (nn < p.b2) {
            const float *m = p.M + (size_t)(4 * kc) * p.ldm + nn;
            v = make_float4(__ldg(m), __ldg(m + p.ldm), __ldg(m + 2 * (size_t)p.ldm), __ldg(m + 3 * (size_t)p.ldm));
        }
        uint4 hi, lo;
        tc::split_tf32(v, hi, lo);
        const uint32_t off = (uint32_t)(nn >> 3) * b_sbo + (uint32_t)(nn & 7) * 16u + (uint32_t)kc * b_lbo;
        *(uint4 *)(b_hi + off) = hi;
        *(uint4 *)(b_lo + off) = lo;
    }
    tc::fence_proxy_async();
    __syncthreads();

    const int64_t tiles_total = (p.n + TILE_M - 1) / TILE_M;
    const int nt = (int)((tiles_total - blockIdx.x + gridDim.x - 1) / gridDim.x);   // tiles blockIdx.x, + grid, ...
    auto tile_row0 = [&](int t) { return ((int64_t)blockIdx.x + (int64_t)t * gridDim.x) * TILE_M; };
    auto tile_rows = [&](int t) { const int64_t r0 = tile_row0(t); return (int)(p.n - r0 < TILE_M ? p.n - r0 : TILE_M); };

    if (warp >= 8) {
        // ================= loader warpgroup: TMA producer (thread 256) + raw rows -> K-major hi / lo tile =================
        auto issue = [&](int t) {
            const int slot = t & 1;
            const uint32_t bytes = (uint32_t)tile_rows(t) * (uint32_t)p.b1 * 4u;
            const uint32_t bar = tc::smem_u32(&s_full[slot]);
            tc::mbar_expect_tx(bar, bytes);
            tc::bulk_g2s(tc::smem_u32(raw_base + (size_t)slot * p.raw_slot), p.Q + tile_row0(t) * p.b1, bytes, bar);
        };
        if (tid == 256) {
            if (nt > 0) issue(0);
            if (nt > 1) issue(1);
        }
        const int ltid = tid - 256;
        for (int t = 0; t < nt; t++) {
            const int slot = t & 1;
            const char *raw = raw_base + (size_t)slot * p.raw_slot;
            tc::mbar_wait(tc::smem_u32(&s_full[slot]), (uint32_t)(t >> 1) & 1);           // rows of tile t have landed
            if (t >= 1) tc::mbar_wait(tc::smem_u32(&s_tile_free), (uint32_t)(t - 1) & 1);  // MMAs of tile t-1 are done
            // lane -> chunk (conflict-free LDS), store with the padded LBO
            const int vr = tile_rows(t);
            for (int idx = ltid; idx < TILE_M * kchunks; idx += 128) {
                const int m = idx / kchunks, kc = idx - m * kchunks;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (m < vr) v = *(const float4 *)(raw + ((size_t)m * p.b1 + 4 * kc) * 4);
                uint4 hi, lo;
                tc::split_tf32(v, hi, lo);
                const uint32_t off = (uint32_t)(m >> 3) * a_sbo + (uint32_t)(m & 7) * 16u + (uint32_t)kc * p.a_lbo;
                *(uint4 *)(a_hi + off) = hi;
                *(uint4 *)(a_lo + off) = lo;
            }
            tc::fence_proxy_async();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(tc::smem_u32(&s_tile_full));
            tc::named_sync(1, 128);                                                         // raw slot fully read
            if (tid == 256 && t + 2 < nt) issue(t + 2);
        }
    } else {
        // ================= MMA warpgroups 0, 1: rows 64*wg .. 64*wg + 63 of every tile, then the epilogue =================
        const int wg = warp >> 2;
        const bool active = wg * 64 < TILE_M;               // warpgroup-uniform
        float acc[NPAD / 2];
        const uint32_t a_off = (uint32_t)wg * 8u * a_sbo;
        for (int t = 0; t < nt; t++) {
            tc::mbar_wait(tc::smem_u32(&s_tile_full), (uint32_t)t & 1);                    // A tile of `t` is written
            __syncwarp();
            uint64_t dah = tc::make_desc(tc::smem_u32(a_hi) + a_off, p.a_lbo, a_sbo), dal = tc::make_desc(tc::smem_u32(a_lo) + a_off, p.a_lbo, a_sbo);
            uint64_t dbh = tc::make_desc(tc::smem_u32(b_hi), b_lbo, b_sbo), dbl = tc::make_desc(tc::smem_u32(b_lo), b_lbo, b_sbo);
            const uint64_t a_step = (uint64_t)((2u * p.a_lbo) >> 4), b_step = (uint64_t)((2u * b_lbo) >> 4);
            if (active) {
                tc::wgmma_fence();
                for (int ks = 0; ks < ksteps; ks++) {
                    tc::wgmma_tf32<NPAD>(acc, dah, dbh, ks > 0 ? 1u : 0u);
                    tc::wgmma_tf32<NPAD>(acc, dah, dbl, 1u);
                    tc::wgmma_tf32<NPAD>(acc, dal, dbh, 1u);
                    dah += a_step; dal += a_step; dbh += b_step; dbl += b_step;
                }
                tc::wgmma_commit();
                tc::wgmma_wait_all();
            }
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(tc::smem_u32(&s_tile_free));                    // the loader may refill the A tile
            if (!active) continue;
            // epilogue (overlaps the loader's work on tile t+1): fragment -> Out, 2 consecutive floats per store
            const int vr = tile_rows(t);
            const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
            float *orow = p.Out + tile_row0(t) * p.ldo;
#pragma unroll
            for (int j = 0; j < NPAD / 8; j++) {
                const int col = j * 8 + (lane & 3) * 2;
                if (col < p.b2) {
                    if (r0 < vr) *(float2 *)(orow + (size_t)r0 * p.ldo + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
                    if (r0 + 8 < vr) *(float2 *)(orow + (size_t)(r0 + 8) * p.ldo + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
                }
            }
        }
    }
}

template <int TILE_M, int NPAD>
static int apply_tc_launch_t(gemb_ctx *ctx, const ApplyTcParams &p, int grid, size_t smem_bytes) {
    static size_t attr_bytes = 0;
    if (attr_bytes < smem_bytes) {
        GEMB_CUDA(cudaFuncSetAttribute(apply_tc_kernel<TILE_M, NPAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
        attr_bytes = smem_bytes;
    }
    return launch(ctx, apply_tc_kernel<TILE_M, NPAD>, grid, 384, smem_bytes, p);
}

template <int TILE_M>
static int apply_tc_dispatch(gemb_ctx *ctx, const ApplyTcParams &p, int npad, int grid, size_t smem_bytes) {
    switch (npad) {
        case 32: return apply_tc_launch_t<TILE_M, 32>(ctx, p, grid, smem_bytes);
        case 64: return apply_tc_launch_t<TILE_M, 64>(ctx, p, grid, smem_bytes);
        case 80: return apply_tc_launch_t<TILE_M, 80>(ctx, p, grid, smem_bytes);
        case 96: return apply_tc_launch_t<TILE_M, 96>(ctx, p, grid, smem_bytes);
        default: return apply_tc_launch_t<TILE_M, 128>(ctx, p, grid, smem_bytes);
    }
}

static int pad_width(int b) {   // accumulator width: one of 32 / 64 / 80 / 96 / 128 columns
    const int widths[5] = {32, 64, 80, 96, 128};
    for (int w : widths) if (w >= b) return w;
    return 128;
}

static size_t apply_smem_bytes(int tile_m, int b1, int npad) {
    const size_t raw_slot = (size_t)tile_m * b1 * 4, a_tile = (size_t)(b1 / 4) * (16 * tile_m + 16);
    const size_t b_tile = (size_t)(npad / 8) * (b1 / 4) * 128;
    return 2 * raw_slot + 2 * a_tile + 2 * b_tile + 256;
}

// returns GEMB_ERR_UNSUPPORTED (without setting an error) when the shape does not fit this kernel
int apply_tc_launch(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int ldm, int b2, float *Out, int ldo) {
    if (b1 % 8 || b2 % 4 || b1 > 128 || ldo < b2 || ldo % 4 || ((uintptr_t)Out & 15) || n <= 0) return GEMB_ERR_UNSUPPORTED;
    // the first configuration that fits in shared memory: 128-row tiles and all columns in one launch, then 64-row tiles,
    // then column blocks of 64 / 32 (one launch each)
    const int cfg[5][2] = {{128, 128}, {64, 128}, {128, 64}, {64, 64}, {64, 32}};
    int tile_m = 0, nbw = 0;
    for (const auto &c : cfg) {
        const int w = std::min(c[1], b2);
        if (apply_smem_bytes(c[0], b1, pad_width(w)) <= 226 * 1024) { tile_m = c[0]; nbw = w; break; }
    }
    if (!tile_m) return GEMB_ERR_UNSUPPORTED;
    const int64_t tiles = (n + tile_m - 1) / tile_m;
    int grid = ctx->sm_count;
    if (grid > tiles) grid = (int)tiles;
    for (int n0 = 0; n0 < b2; n0 += nbw) {
        ApplyTcParams p;
        const int w = std::min(nbw, b2 - n0), npad = pad_width(w);
        p.n = n; p.Q = Q; p.M = M + n0; p.Out = Out + n0; p.b1 = b1; p.b2 = w; p.ldm = ldm; p.ldo = ldo;
        p.a_lbo = 16u * (uint32_t)tile_m + 16u;
        p.a_tile = (uint32_t)(b1 / 4) * p.a_lbo;
        p.b_tile = (uint32_t)(npad / 8) * (uint32_t)(b1 / 4) * 128u;
        p.raw_slot = (uint32_t)((size_t)tile_m * b1 * 4);
        const size_t smem_bytes = apply_smem_bytes(tile_m, b1, npad);
        if (tile_m == 128) GEMB_TRY(apply_tc_dispatch<128>(ctx, p, npad, grid, smem_bytes));
        else GEMB_TRY(apply_tc_dispatch<64>(ctx, p, npad, grid, smem_bytes));
    }
    return GEMB_OK;
}

}  // namespace gemb
