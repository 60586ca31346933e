// gem_b200/csrc/dense.cu -- tall-skinny dense kernels of the HOPE solver (round-1 CUDA-core version).
//
//   gram   : G = P^T Q      (n x b1, n x b2 -> b1 x b2), the CholeskyQR / Rayleigh-Ritz contraction
//   apply  : Out = Q * M    (n x b1 times b1 x b2)
//   chol_inverse, eigh : single-CTA fp64 factorizations of the b x b matrices, one kernel each; the working matrices
//                        live in shared memory where they fit and in global memory (L2 resident) beyond
// These replace numpy.linalg.qr / svd inside scipy's svds (hope.py:33 -> _svds.py:508-533).
// fp32 data, fp32 FMA inside a CTA's partial sums, fp64 across CTAs and in the b x b algebra.
#include "common.cuh"
#include <algorithm>

namespace gemb {

// ------------------------------------------------------------------------------------ gram
// Output tile (16*TM) x (16*TM) per blockIdx.y, rows strided over blockIdx.x in chunks of KC; the partial sums of
// blockIdx.x go to Gpart[blockIdx.x][b1][b2] (added in a fixed order afterwards).
template <int TM>
__global__ void __launch_bounds__(256)
gram_kernel(int64_t n, const float *__restrict__ P, int b1, const float *__restrict__ Q, int b2,
            double *__restrict__ Gpart, int tiles_n) {
    constexpr int BT = 16 * TM;
    constexpr int KC = 32;
    __shared__ float sP[KC][BT];
    __shared__ float sQ[KC][BT];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int tile_m = blockIdx.y / tiles_n, tile_n = blockIdx.y % tiles_n;
    const int m0 = tile_m * BT, n0 = tile_n * BT;
    float acc[TM][TM];
#pragma unroll
    for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TM; j++) acc[i][j] = 0.f;

    for (int64_t r0 = (int64_t)blockIdx.x * KC; r0 < n; r0 += (int64_t)gridDim.x * KC) {
        for (int idx = tid; idx < KC * BT; idx += 256) {
            const int kk = idx / BT, col = idx - kk * BT;
            const int64_t r = r0 + kk;
            float vp = 0.f, vq = 0.f;
            if (r < n) {
                if (m0 + col < b1) vp = __ldg(P + r * b1 + m0 + col);
                if (n0 + col < b2) vq = __ldg(Q + r * b2 + n0 + col);
            }
            sP[kk][col] = vp;
            sQ[kk][col] = vq;
        }
        __syncthreads();
#pragma unroll 4
        for (int kk = 0; kk < KC; kk++) {
            float a[TM], bb[TM];
#pragma unroll
            for (int i = 0; i < TM; i++) a[i] = sP[kk][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TM; j++) bb[j] = sQ[kk][tx * TM + j];
#pragma unroll
            for (int i = 0; i < TM; i++)
#pragma unroll
                for (int j = 0; j < TM; j++) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TM; i++) {
        const int gm = m0 + ty * TM + i;
        if (gm >= b1) continue;
#pragma unroll
        for (int j = 0; j < TM; j++) {
            const int gn = n0 + tx * TM + j;
            if (gn < b2) Gpart[(size_t)blockIdx.x * b1 * b2 + (size_t)gm * b2 + gn] = (double)acc[i][j];
        }
    }
}

static int pick_tm(int b) {
    // tile edge 16*TM for TM in {4,5,6,8}: minimise padded area, prefer fewer tiles on ties
    int best = 4;
    long best_cost = -1;
    const int cand[4] = {4, 5, 6, 8};
    for (int t = 0; t < 4; t++) {
        int bt = 16 * cand[t];
        long tiles = (b + bt - 1) / bt;
        long cost = tiles * bt;
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = cand[t]; }
    }
    return best;
}

int gram_tc_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G);

int gram_fp32_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G);

int gram_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G) {
    if (n >= 4096) {
        const int s = gram_tc_launch(ctx, n, P, b1, Q, b2, G);
        if (s != GEMB_ERR_UNSUPPORTED) return s;
    }
    return gram_fp32_launch(ctx, n, P, b1, Q, b2, G);
}

int red_scratch(gemb_ctx *ctx, size_t doubles, double **out) {
    const size_t need = sizeof(double) * std::max<size_t>(doubles, 1);
    if (ctx->red_scratch_bytes < need) {
        GEMB_CUDA(dfree(ctx->red_scratch));
        ctx->red_scratch = nullptr; ctx->red_scratch_bytes = 0;
        GEMB_CUDA(dmalloc(&ctx->red_scratch, need));
        ctx->red_scratch_bytes = need;
    }
    *out = ctx->red_scratch;
    return GEMB_OK;
}

// block (32, 8): 32 consecutive outputs; warp y adds parts y, y + 8, ... (coalesced rows), then the 8 sums in order
__global__ void __launch_bounds__(256) sum_partials_kernel(int parts, int64_t count, const double *__restrict__ part,
                                                           double *__restrict__ out) {
    __shared__ double s_sum[8][33];
    const int tx = threadIdx.x, ty = threadIdx.y;
    for (int64_t i0 = (int64_t)blockIdx.x * 32; i0 < count; i0 += (int64_t)gridDim.x * 32) {
        const int64_t i = i0 + tx;
        double s = 0.0;
        if (i < count)
            for (int c = ty; c < parts; c += 8) s += part[(size_t)c * count + i];
        s_sum[ty][tx] = s;
        __syncthreads();
        if (ty == 0 && i < count) {
            double t = 0.0;
            for (int y = 0; y < 8; y++) t += s_sum[y][tx];
            out[i] = t;
        }
        __syncthreads();
    }
}

int sum_partials_launch(gemb_ctx *ctx, int parts, int64_t count, const double *part, double *out) {
    if (count == 0) return GEMB_OK;
    return launch(ctx, sum_partials_kernel, grid_stride(ctx, count, 32, 16), dim3(32, 8), 0, parts, count, part, out);
}

int gram_fp32_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G) {
    if (n == 0) {
        GEMB_CUDA(cudaMemsetAsync(G, 0, sizeof(double) * (size_t)b1 * b2, ctx->stream));
        return GEMB_OK;
    }
    const int bmax = b1 > b2 ? b1 : b2;
    const int TM = pick_tm(bmax);
    const int BT = 16 * TM;
    const int tiles_m = (b1 + BT - 1) / BT, tiles_n = (b2 + BT - 1) / BT;
    int64_t chunks = (n + 31) / 32;
    int gx = ctx->sm_count * 4 / (tiles_m * tiles_n);
    if (gx < 1) gx = 1;
    if (gx > chunks) gx = (int)chunks;
    dim3 grid(gx, tiles_m * tiles_n), block(256);
    double *part = nullptr;
    GEMB_TRY(red_scratch(ctx, (size_t)gx * b1 * b2, &part));
    const auto kernel = TM == 4 ? gram_kernel<4> : TM == 5 ? gram_kernel<5> : TM == 6 ? gram_kernel<6> : gram_kernel<8>;
    GEMB_TRY(launch(ctx, kernel, grid, block, 0, n, P, b1, Q, b2, part, tiles_n));
    return sum_partials_launch(ctx, gx, (int64_t)b1 * b2, part, G);
}

// ------------------------------------------------------------------------------------ apply
// Out[r, n0 + ..] = sum_k Q[r, k] * M[k, ..];  CTA tile: 64 rows x (16*TN) columns, K chunks of 16.
template <int TN>
__global__ void __launch_bounds__(256)
apply_kernel(int64_t n, const float *__restrict__ Q, int b1, const float *__restrict__ M, int ldm,
             int b2, float *__restrict__ Out, int ldo) {
    constexpr int BN = 16 * TN;
    constexpr int BM = 64, BK = 16;
    __shared__ float sA[BK][BM + 1];
    __shared__ float sB[BK][BN];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;  // ty -> 4 rows, tx -> TN columns
    const int64_t r0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    float acc[4][TN];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < b1; k0 += BK) {
        for (int idx = tid; idx < BM * BK; idx += 256) {
            const int rr = idx / BK, kk = idx - rr * BK;
            const int64_t r = r0 + rr;
            sA[kk][rr] = (r < n && k0 + kk < b1) ? __ldg(Q + r * b1 + k0 + kk) : 0.f;
        }
        for (int idx = tid; idx < BK * BN; idx += 256) {
            const int kk = idx / BN, col = idx - kk * BN;
            sB[kk][col] = (k0 + kk < b1 && n0 + col < b2) ? __ldg(M + (size_t)(k0 + kk) * ldm + n0 + col) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; kk++) {
            float a[4], bb[TN];
#pragma unroll
            for (int i = 0; i < 4; i++) a[i] = sA[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < TN; j++) bb[j] = sB[kk][tx * TN + j];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < TN; j++) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int64_t r = r0 + ty * 4 + i;
        if (r >= n) continue;
#pragma unroll
        for (int j = 0; j < TN; j++) {
            const int col = n0 + tx * TN + j;
            if (col < b2) Out[r * ldo + col] = acc[i][j];
        }
    }
}

int apply_tc_launch(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int ldm, int b2, float *Out, int ldo);

int apply_launch(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int ldm, int b2,
                 float *Out, int ldo) {
    if (n == 0 || b2 == 0) return GEMB_OK;
    if (n >= 4096) {
        const int s = apply_tc_launch(ctx, n, Q, b1, M, ldm, b2, Out, ldo);
        if (s != GEMB_ERR_UNSUPPORTED) return s;
    }
    return apply_fp32_launch(ctx, n, Q, b1, M, ldm, b2, Out, ldo);
}

int apply_fp32_launch(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int ldm, int b2,
                      float *Out, int ldo) {
    const int TN = pick_tm(b2);
    const int BN = 16 * TN;
    dim3 grid((unsigned)((n + 63) / 64), (b2 + BN - 1) / BN), block(256);
    const auto kernel = TN == 4 ? apply_kernel<4> : TN == 5 ? apply_kernel<5> : TN == 6 ? apply_kernel<6> : apply_kernel<8>;
    return launch(ctx, kernel, grid, block, 0, n, Q, b1, M, ldm, b2, Out, ldo);
}

// ------------------------------------------------------------------------------------ chol_inverse
// G (b x b fp64, symmetric) -> Minv = R^-1 (fp32, upper triangular) with G = R^T R.
// Work on the diagonally scaled matrix D^-1/2 G D^-1/2 (unit diagonal) so that the rank test is
// scale free.  A pivot below PIV_EPS marks the column numerically dependent: its column of Minv is
// zero (the orthonormalised block then carries a zero column, which stays zero under S).
#define GEMB_PIV_EPS 1e-5
// Two block barriers per Cholesky column (the <= 3 warps that own the column compute the pivot themselves), and the
// triangular inverse without block barriers -- each column of L^-1 belongs to 8 lanes of one warp that split the dot
// products.  Index walks are division free.  Since b <= 1024, one thread per row of a column of L.
// SMEM: the scaled matrix lives in shared memory with an odd leading dimension (column walks are bank-conflict free),
// and G is only read.  Otherwise the kernel works in place in G (leading dimension b) and overwrites it.
// Gg is not __restrict__: without SMEM it is the work matrix that other threads write between barriers, and with
// __restrict__ nvcc once kept a pivot G[j][j] that every thread had loaded before another thread replaced it by its
// root across the barrier (a column of L was divided by the pivot, not its root).
template <bool SMEM>
__global__ void __launch_bounds__(1024)
chol_inverse_kernel(int b, double *Gg, float *__restrict__ Minv, double *__restrict__ Minv64,
                    int *__restrict__ rank_out) {
    extern __shared__ double sh[];
    const int ld = SMEM ? (b | 1) : b;
    double *dscale = sh;           // b : 1/sqrt(G_jj) (0 if G_jj <= 0)
    double *ldiag = sh + b;        // b : L_jj (0 if the column was dropped)
    double *colj = sh + 2 * b;     // b : scaled column j of L
    double *G = SMEM ? sh + 3 * b : Gg;   // b x ld
    const double *__restrict__ Gin = Gg;  // read only, and only when SMEM: its loads may take the read-only data path
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int j = tid; j < b; j += nt) {
        const double d = (SMEM ? Gin : Gg)[(size_t)j * b + j];
        dscale[j] = d > 0.0 ? rsqrt(d) : 0.0;
    }
    __syncthreads();
    for (int idx = tid; idx < b * b; idx += nt) {
        const int i = idx / b, j = idx - i * b;
        G[i * ld + j] = (SMEM ? Gin : Gg)[idx] * dscale[i] * dscale[j];
    }
    __syncthreads();
    const int gi0 = tid / b, gk0 = tid - gi0 * b, gdi = nt / b, gdk = nt - gdi * b;
    int si = gi0, sk = gk0;   // where the walk starts; in global memory it skips the rows <= j, which hold no update
    for (int j = 0; j < b; j++) {
        const int m = b - j - 1;
        if (tid < m || tid == 0) {   // the column's owners each derive the pivot (no broadcast barrier)
            const double d = G[j * ld + j];
            const bool ok = d > GEMB_PIV_EPS;
            const double ljj = ok ? sqrt(d) : 0.0;
            const double inv = ok ? 1.0 / ljj : 0.0;
            if (tid == 0) ldiag[j] = ljj;
            if (tid < m) {
                const int i = j + 1 + tid;
                const double v = G[i * ld + j] * inv;
                colj[i] = v;
                G[i * ld + j] = v;
            }
        }
        __syncthreads();
        // every thread owns the same (i, k) positions of the b x b grid in all steps (no index division)
        if (!SMEM) while (si <= j) { sk += gdk; si += gdi; if (sk >= b) { sk -= b; si++; } }
        for (int i = si, k = sk; i < b;) {
            if (k > j && k <= i) G[i * ld + k] -= colj[i] * colj[k];
            k += gdk; i += gdi;
            if (k >= b) { k -= b; i++; }
        }
        __syncthreads();
    }
    // X = L^-1 by rows; column c of X is kept in the free strict upper triangle G[c][i] = X[i][c]
    const int lane8 = tid & 7, grp = tid >> 3, ngrp = nt >> 3;
    const unsigned gmask = 0xffu << ((tid & 31) & ~7);
    for (int c = grp; c < b; c += ngrp) {
        const double lcc = ldiag[c];
        const bool okc = lcc > 0.0;
        const double xc = okc ? 1.0 / lcc : 0.0;
        for (int i = c + 1; i < b; i++) {
            const double lii = ldiag[i];
            double sum = 0.0;
            if (okc && lii > 0.0) {
                for (int k = c + 1 + lane8; k < i; k += 8) sum += G[i * ld + k] * G[c * ld + k];
                sum += __shfl_xor_sync(gmask, sum, 4, 8);
                sum += __shfl_xor_sync(gmask, sum, 2, 8);
                sum += __shfl_xor_sync(gmask, sum, 1, 8);
                sum = -(sum + G[i * ld + c] * xc) / lii;
            }
            __syncwarp(gmask);
            if (lane8 == 0) G[c * ld + i] = sum;
            __syncwarp(gmask);
        }
    }
    __syncthreads();
    int rank = 0;
    for (int idx = tid; idx < b * b; idx += nt) {
        const int r = idx / b, c = idx - r * b;  // Minv[r][c] = dscale[r] * X[c][r], r <= c
        double v = 0.0;
        if (r == c) { v = ldiag[r] > 0.0 ? dscale[r] / ldiag[r] : 0.0; }
        else if (r < c) v = G[r * ld + c] * dscale[r];
        Minv[idx] = (float)v;
        if (Minv64) Minv64[idx] = v;
    }
    if (tid == 0 && rank_out) {
        for (int j = 0; j < b; j++) rank += ldiag[j] > 0.0;
        *rank_out = rank;
    }
}

int chol_inverse_launch(gemb_ctx *ctx, int b, double *G, float *Minv, int *rank_out_dev, double *Minv64) {
    const size_t vecs = sizeof(double) * 3 * (size_t)b;
    const size_t smem = vecs + sizeof(double) * (size_t)b * (b | 1);
    static int optin = 0;    // the device's per-block opt-in limit (227 KB on H100: b <= 168 in shared memory)
    if (!optin) {
        int v = 0;
        GEMB_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
        GEMB_CUDA(cudaFuncSetAttribute(chol_inverse_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
        optin = v;
    }
    const bool in_smem = smem <= (size_t)optin;
    return launch(ctx, in_smem ? chol_inverse_kernel<true> : chol_inverse_kernel<false>, 1, 1024, in_smem ? smem : vecs,
                  b, G, Minv, Minv64, rank_out_dev);
}

// ------------------------------------------------------------------------------------ eigh
// Two-sided cyclic Jacobi with round-robin (circle-method) pair ordering, one CTA, fp64: w ascending, Z column j <->
// w[j].  Zt is b x b scratch.  b <= 1024: one rotation pair per thread.
//   * the two-sided update A <- J^T A J is done per 2x2 BLOCK {p,q} x {r,s} of two rotation pairs by one thread
//     (4 loads, both rotations in registers, 4 stores): half the A traffic and one block barrier per round less
//     than a column phase followed by a row phase;
//   * the eigenvector accumulator is kept transposed so that its update is a row walk;
//   * (pair, column) indices advance incrementally (no division in the loops), rotation parameters are one
//     16-byte and one 8-byte load, the shared-memory leading dimension is odd (conflict-free row and column walks).
// Where the matrices live (eigh_launch takes the first that fits in shared memory):
//   JAC_SHARED     A and Z^T in shared memory (b <= 117);
//   JAC_ZT_GLOBAL  A alone fills the shared memory (b <= 167, e.g. the Rayleigh-Ritz matrix of the thick-restart
//                  Lanczos solver); Z^T is Zt (L2 resident, 200 KB), updated by coalesced row walks;
//   JAC_GLOBAL     A is G itself (leading dimension b, destroyed) and Z^T is Zt.
// symmetrize: the decomposition is that of (G + G^T) / 2, formed while the matrix is loaded (a Rayleigh-Ritz matrix
// V^T (A V) is symmetric only up to rounding).
// G and Zt are not __restrict__: in global memory they are written by other threads between barriers.
enum JacobiStore { JAC_SHARED, JAC_ZT_GLOBAL, JAC_GLOBAL };
template <JacobiStore STORE>
__global__ void __launch_bounds__(1024)
eigh_jacobi_kernel(int b, double *Ag, double *__restrict__ w, double *__restrict__ Z, double *Ztg, int max_sweeps,
                   double rel_tol, bool symmetrize) {
    constexpr bool A_GLOBAL = STORE == JAC_GLOBAL, ZT_GLOBAL = STORE != JAC_SHARED;
    extern __shared__ __align__(16) unsigned char sh_fast[];
    double *sh = (double *)sh_fast;
    const int m = (b + 1) & ~1;
    const int half = m / 2;
    const int ld = A_GLOBAL ? b : (b | 1);
    double2 *csn = (double2 *)sh;                 // half : (c, s)
    int2 *pq = (int2 *)(sh + 2 * half);           // half : (p, q), q = -1 for the dummy partner
    double *A = A_GLOBAL ? Ag : sh + 3 * half + 2;       // b x ld
    double *ZT = ZT_GLOBAL ? Ztg : A + (size_t)b * ld;   // ZT[j][k] = component k of eigenvector j
    const int ldz = ZT_GLOBAL ? b : ld;
    __shared__ double s_woff[32], s_wdiag[32];   // per-warp partials, added in warp order (same result every run)
    const int tid = threadIdx.x, nt = blockDim.x;
    const double *__restrict__ Ain = Ag;          // read only, and only when A is in shared memory (read-only data path)
    for (int idx = tid; idx < b * b; idx += nt) {
        const int i = idx / b, j = idx - i * b;
        if (!A_GLOBAL) A[i * ld + j] = (symmetrize && i != j) ? 0.5 * (Ain[idx] + Ain[j * b + i]) : Ain[idx];
        else if (symmetrize && i < j) Ag[idx] = Ag[j * b + i] = 0.5 * (Ag[idx] + Ag[j * b + i]);   // the pair's only owner
        ZT[i * ldz + j] = (i == j) ? 1.0 : 0.0;
    }
    // incremental (pair, column) walks: idx = tid + t * nt  ->  (idx / div, idx % div)
    const int zb_i0 = tid / b, zb_k0 = tid - zb_i0 * b, zb_di = nt / b, zb_dk = nt - zb_di * b;
    const int bl_i0 = tid / half, bl_j0 = tid - bl_i0 * half, bl_di = nt / half, bl_dj = nt - bl_di * half;
    __syncthreads();
    for (int sweep = 0; sweep < max_sweeps; sweep++) {
        __syncthreads();                 // the previous sweep has read s_woff / s_wdiag
        double off = 0.0, dg = 0.0;
        for (int i = zb_i0, j = zb_k0; i < b;) {
            const double v = A[i * ld + j];
            if (i == j) dg += v * v; else off += v * v;
            j += zb_dk; i += zb_di;
            if (j >= b) { j -= b; i++; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            off += __shfl_xor_sync(0xffffffffu, off, o);
            dg += __shfl_xor_sync(0xffffffffu, dg, o);
        }
        if ((tid & 31) == 0) { s_woff[tid >> 5] = off; s_wdiag[tid >> 5] = dg; }
        __syncthreads();
        double s_off = 0.0, s_diag = 0.0;
        for (int w = 0; w < (nt >> 5); w++) { s_off += s_woff[w]; s_diag += s_wdiag[w]; }
        if (s_off <= rel_tol * rel_tol * (s_diag + s_off) || s_diag + s_off == 0.0) break;
        for (int r = 0; r < m - 1; r++) {
            if (tid < half) {
                int p, q;
                if (tid == 0) { p = m - 1; q = r % (m - 1); }
                else { p = (r + tid) % (m - 1); q = (r + m - 1 - tid) % (m - 1); }
                if (p > q) { int t = p; p = q; q = t; }
                double c = 1.0, s = 0.0;
                if (q < b) {
                    const double apq = A[p * ld + q];
                    if (apq != 0.0) {
                        const double app = A[p * ld + p], aqq = A[q * ld + q];
                        const double theta = (aqq - app) / (2.0 * apq);
                        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                        c = rsqrt(t * t + 1.0);
                        s = t * c;
                    }
                } else { q = -1; }
                pq[tid] = make_int2(p, q);
                csn[tid] = make_double2(c, s);
            }
            __syncthreads();
            // A <- J^T A J, one 2x2 block {p,q} x {r2,s2} per thread
            for (int pi = bl_i0, rj = bl_j0; pi < half;) {
                const double2 r1 = csn[pi], r2 = csn[rj];
                if (r1.y != 0.0 || r2.y != 0.0) {
                    const int2 a = pq[pi], c2 = pq[rj];
                    const bool hq = a.y >= 0, hs = c2.y >= 0;
                    double *row_p = A + a.x * ld, *row_q = A + (hq ? a.y : a.x) * ld;
                    const int cr = c2.x, cs2 = hs ? c2.y : c2.x;
                    const double apr = row_p[cr], aps = hs ? row_p[cs2] : 0.0;
                    const double aqr = hq ? row_q[cr] : 0.0, aqs = (hq && hs) ? row_q[cs2] : 0.0;
                    const double tpr = r1.x * apr - r1.y * aqr, tqr = r1.y * apr + r1.x * aqr;
                    const double tps = r1.x * aps - r1.y * aqs, tqs = r1.y * aps + r1.x * aqs;
                    row_p[cr] = r2.x * tpr - r2.y * tps;
                    if (hs) row_p[cs2] = r2.y * tpr + r2.x * tps;
                    if (hq) {
                        row_q[cr] = r2.x * tqr - r2.y * tqs;
                        if (hs) row_q[cs2] = r2.y * tqr + r2.x * tqs;
                    }
                }
                rj += bl_dj; pi += bl_di;
                if (rj >= half) { rj -= half; pi++; }
            }
            // Z^T <- J^T Z^T (rows p, q; consecutive threads = consecutive columns)
            if (ZT_GLOBAL) {
                // global (L2) accumulator: batches of 4 independent element pairs -- all 8 loads are issued before the
                // first store, otherwise every element pays a full L2 round trip in sequence
                int pi = zb_i0, k = zb_k0;
                while (pi < half) {
                    double *xp[4], *yp[4];
                    double2 rt[4];
                    double x[4], y[4];
                    bool on[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        on[u] = false;
                        if (pi < half) {
                            rt[u] = csn[pi];
                            const int2 a = pq[pi];
                            if (a.y >= 0 && rt[u].y != 0.0) {
                                on[u] = true;
                                xp[u] = ZT + a.x * ldz + k; yp[u] = ZT + a.y * ldz + k;
                            }
                            k += zb_dk; pi += zb_di;
                            if (k >= b) { k -= b; pi++; }
                        }
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) if (on[u]) { x[u] = __ldcg(xp[u]); y[u] = __ldcg(yp[u]); }
#pragma unroll
                    for (int u = 0; u < 4; u++) if (on[u]) {
                        __stcg(xp[u], rt[u].x * x[u] - rt[u].y * y[u]);
                        __stcg(yp[u], rt[u].y * x[u] + rt[u].x * y[u]);
                    }
                }
            } else {
                for (int pi = zb_i0, k = zb_k0; pi < half;) {
                    const double2 rt = csn[pi];
                    const int2 a = pq[pi];
                    if (a.y >= 0 && rt.y != 0.0) {
                        double *xp = ZT + a.x * ldz + k, *yp = ZT + a.y * ldz + k;
                        const double x = *xp, y = *yp;
                        *xp = rt.x * x - rt.y * y;
                        *yp = rt.y * x + rt.x * y;
                    }
                    k += zb_dk; pi += zb_di;
                    if (k >= b) { k -= b; pi++; }
                }
            }
            __syncthreads();
        }
    }
    __syncthreads();
    const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
    for (int j = warp; j < b; j += nwarps) {
        const double wj = A[j * ld + j];
        int rank = 0;
        for (int i = lane; i < b; i += 32) {
            const double wi = A[i * ld + i];
            rank += (wi < wj) || (wi == wj && i < j);
        }
        for (int o = 16; o > 0; o >>= 1) rank += __shfl_xor_sync(0xffffffffu, rank, o);
        if (lane == 0) w[rank] = wj;
        for (int k = lane; k < b; k += 32) Z[(size_t)k * b + rank] = ZT_GLOBAL ? __ldcg(ZT + j * ldz + k) : ZT[j * ldz + k];
    }
}

int eigh_launch(gemb_ctx *ctx, int b, double *G, double *w, double *Z, double *Zscratch, double rel_tol, bool symmetrize) {
    const int half = ((b + 1) & ~1) / 2;
    const size_t base = sizeof(double) * (3 * half + 2);
    const size_t cap = 220 * 1024;
    const size_t mat = sizeof(double) * (size_t)b * (b | 1);
    static bool attr_set = false;
    if (!attr_set) {
        GEMB_CUDA(cudaFuncSetAttribute(eigh_jacobi_kernel<JAC_SHARED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cap));
        GEMB_CUDA(cudaFuncSetAttribute(eigh_jacobi_kernel<JAC_ZT_GLOBAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cap));
        attr_set = true;
    }
    auto kernel = eigh_jacobi_kernel<JAC_GLOBAL>;
    size_t smem = base;
    if (base + 2 * mat <= cap) { kernel = eigh_jacobi_kernel<JAC_SHARED>; smem = base + 2 * mat; }
    else if (base + mat <= cap) { kernel = eigh_jacobi_kernel<JAC_ZT_GLOBAL>; smem = base + mat; }
    return launch(ctx, kernel, 1, 1024, smem, b, G, w, Z, Zscratch, 30, rel_tol, symmetrize);
}

// ------------------------------------------------------------------------------------ small b x b products
// C = op(A) * B, all b x b fp64 row-major (one CTA; used for the Ritz rotation of Gram matrices)
__global__ void __launch_bounds__(1024)
small_gemm_kernel(int b, const double *__restrict__ A, int transA, const double *__restrict__ B,
                  double *__restrict__ C, float *__restrict__ C32) {
    for (int idx = threadIdx.x; idx < b * b; idx += blockDim.x) {
        const int i = idx / b, j = idx - i * b;
        double acc = 0.0;
        if (transA) for (int k = 0; k < b; k++) acc += A[(size_t)k * b + i] * B[(size_t)k * b + j];
        else for (int k = 0; k < b; k++) acc += A[(size_t)i * b + k] * B[(size_t)k * b + j];
        if (C) C[idx] = acc;
        if (C32) C32[idx] = (float)acc;
    }
}

int small_gemm_launch(gemb_ctx *ctx, int b, const double *A, int transA, const double *B, double *C, float *C32) {
    return launch(ctx, small_gemm_kernel, 1, 1024, 0, b, A, transA, B, C, C32);
}

// ------------------------------------------------------------------------------------ misc
__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// standard normal per (global row, column): independent of the sharding
__global__ void randn_kernel(int64_t n, int b, uint64_t seed, uint64_t row_offset, float *__restrict__ X) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * b) return;
    const int64_t r = idx / b;
    const int c = (int)(idx - r * b);
    const uint64_t h = splitmix64(seed ^ splitmix64(((uint64_t)(r + row_offset) << 12) ^ (uint64_t)c));
    const uint32_t u1 = (uint32_t)(h >> 32), u2 = (uint32_t)h;
    const float f1 = ((float)u1 + 1.0f) * 2.3283064365386963e-10f;  // (0,1]
    const float f2 = (float)u2 * 2.3283064365386963e-10f;
    X[idx] = sqrtf(-2.0f * logf(f1)) * cospif(2.0f * f2);
}

int randn_launch(gemb_ctx *ctx, int64_t n, int b, uint64_t seed, uint64_t row_offset, float *X) {
    const int64_t tot = n * b;
    if (tot == 0) return GEMB_OK;
    return launch(ctx, randn_kernel, (unsigned)((tot + 255) / 256), 256, 0, n, b, seed, row_offset, X);
}

// block sums of squares -> part[blockIdx.x] (blockDim.x = 256)
__global__ void sumsq_kernel(int64_t count, const float *__restrict__ X, double *__restrict__ part) {
    __shared__ double s_w[8];
    double acc = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count;
         i += (int64_t)gridDim.x * blockDim.x) {
        const double v = X[i];
        acc += v * v;
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int w = 0; w < 8; w++) s += s_w[w];
        part[blockIdx.x] = s;
    }
}

int sumsq_launch(gemb_ctx *ctx, int64_t count, const float *X, double *out_dev) {
    if (count == 0) {
        GEMB_CUDA(cudaMemsetAsync(out_dev, 0, sizeof(double), ctx->stream));
        return GEMB_OK;
    }
    const int grid = grid_stride(ctx, count, 256, 8);
    double *part = nullptr;
    GEMB_TRY(red_scratch(ctx, (size_t)grid, &part));
    GEMB_TRY(launch(ctx, sumsq_kernel, grid, 256, 0, count, X, part));
    return sum_partials_launch(ctx, grid, 1, part, out_dev);
}

__global__ void scale_kernel(int64_t count, float s, float *__restrict__ X) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count;
         i += (int64_t)gridDim.x * blockDim.x)
        X[i] *= s;
}

int scale_launch(gemb_ctx *ctx, int64_t count, float s, float *X) {
    if (count == 0) return GEMB_OK;
    return launch(ctx, scale_kernel, grid_stride(ctx, count, 256, 8), 256, 0, count, s, X);
}

// Y += a * X over count floats
__global__ void axpy_kernel(int64_t count, float a, const float *__restrict__ X, float *__restrict__ Y) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        Y[i] = fmaf(a, X[i], Y[i]);
}

int axpy_launch(gemb_ctx *ctx, int64_t count, float a, const float *X, float *Y) {
    return launch(ctx, axpy_kernel, ctx->sm_count * 8, 256, 0, count, a, X, Y);
}

}  // namespace gemb

extern "C" int gemb_gram(gemb_ctx *c, int64_t n, const float *P, int b1, const float *Q, int b2,
                         int use_tensor_cores, double *G_out) {
    using namespace gemb;
    GEMB_ARG(c && P && G_out && n >= 0 && b1 > 0 && b2 > 0, "ctx/P/G/n/b");
    GEMB_CUDA(cudaSetDevice(c->device));
    DeviceBuffer<float> dP, dQ;
    DeviceBuffer<double> dG;
    GEMB_CUDA(dP.upload(P, (size_t)n * b1, c->stream));
    if (Q) GEMB_CUDA(dQ.upload(Q, (size_t)n * b2, c->stream));
    GEMB_CUDA(dG.alloc((size_t)b1 * b2));
    const float *dQP = Q ? dQ.get() : dP.get();
    const int s = use_tensor_cores ? gram_tc_launch(c, n, dP.get(), b1, dQP, b2, dG.get())
                                   : gram_fp32_launch(c, n, dP.get(), b1, dQP, b2, dG.get());
    if (s == GEMB_ERR_UNSUPPORTED) set_error("gemb_gram: shape (n=%lld, b1=%d, b2=%d) not supported by the tensor-core kernel", (long long)n, b1, b2);
    if (s != GEMB_OK) return s;
    GEMB_CUDA(cudaMemcpyAsync(G_out, dG.get(), sizeof(double) * (size_t)b1 * b2, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

// The b x b hooks run the solvers' own launchers, so b picks the kernel variant exactly as in a solve.  b is limited to
// the solvers' block limit (gemb_hope: b <= 1024), which both kernels rely on (one thread per row of a column of L, one
// rotation pair per thread).
extern "C" int gemb_chol_inverse(gemb_ctx *c, int b, const double *G, double *Minv64_out, float *Minv32_out,
                                 int *rank_out) {
    using namespace gemb;
    GEMB_ARG(c && G && Minv64_out && Minv32_out && rank_out && b > 0 && b <= 1024, "ctx/G/Minv/rank/b");
    GEMB_CUDA(cudaSetDevice(c->device));
    const size_t bb = (size_t)b * b;
    DeviceBuffer<double> dG, dM64;
    DeviceBuffer<float> dM32;
    DeviceBuffer<int> dRank;
    GEMB_CUDA(dG.upload(G, bb, c->stream));
    GEMB_CUDA(dM64.alloc(bb));
    GEMB_CUDA(dM32.alloc(bb));
    GEMB_CUDA(dRank.alloc(1));
    GEMB_TRY(chol_inverse_launch(c, b, dG.get(), dM32.get(), dRank.get(), dM64.get()));
    GEMB_CUDA(cudaMemcpyAsync(Minv64_out, dM64.get(), sizeof(double) * bb, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(Minv32_out, dM32.get(), sizeof(float) * bb, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(rank_out, dRank.get(), sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

extern "C" int gemb_eigh(gemb_ctx *c, int b, const double *G, double rel_tol, double *w_out, double *Z_out) {
    using namespace gemb;
    GEMB_ARG(c && G && w_out && Z_out && b > 0 && b <= 1024 && rel_tol >= 0.0, "ctx/G/w/Z/b/rel_tol");
    GEMB_CUDA(cudaSetDevice(c->device));
    const size_t bb = (size_t)b * b;
    DeviceBuffer<double> dG, dw, dZ, dZs;
    GEMB_CUDA(dG.upload(G, bb, c->stream));
    GEMB_CUDA(dw.alloc(b));
    GEMB_CUDA(dZ.alloc(bb));
    GEMB_CUDA(dZs.alloc(bb));
    GEMB_TRY(eigh_launch(c, b, dG.get(), dw.get(), dZ.get(), dZs.get(), rel_tol));
    GEMB_CUDA(cudaMemcpyAsync(w_out, dw.get(), sizeof(double) * b, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(Z_out, dZ.get(), sizeof(double) * bb, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

extern "C" int gemb_apply(gemb_ctx *c, int64_t n, const float *Q, int b1, const float *M, int b2,
                          int use_tensor_cores, float *Out) {
    using namespace gemb;
    GEMB_ARG(c && Q && M && Out && n >= 0 && b1 > 0 && b2 > 0, "ctx/Q/M/Out/n/b");
    GEMB_CUDA(cudaSetDevice(c->device));
    DeviceBuffer<float> dQ, dM, dO;
    GEMB_CUDA(dQ.upload(Q, (size_t)n * b1, c->stream));
    GEMB_CUDA(dM.upload(M, (size_t)b1 * b2, c->stream));
    GEMB_CUDA(dO.alloc((size_t)std::max<int64_t>(n, 1) * b2));
    const int s = use_tensor_cores ? apply_tc_launch(c, n, dQ.get(), b1, dM.get(), b2, b2, dO.get(), b2)
                                   : apply_fp32_launch(c, n, dQ.get(), b1, dM.get(), b2, b2, dO.get(), b2);
    if (s == GEMB_ERR_UNSUPPORTED) set_error("gemb_apply: shape (n=%lld, b1=%d, b2=%d) not supported by the tensor-core kernel", (long long)n, b1, b2);
    if (s != GEMB_OK) return s;
    GEMB_CUDA(cudaMemcpyAsync(Out, dO.get(), sizeof(float) * (size_t)n * b2, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}
