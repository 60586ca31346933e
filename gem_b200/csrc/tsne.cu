// gem_b200/csrc/tsne.cu -- t-SNE to two dimensions: sklearn 1.9's TSNE(n_components=2) with its defaults (init='pca',
// method='barnes_hut', metric='euclidean'), the step the reference's plot_embedding2D runs
// (gem/evaluation/visualize_embedding.py:7-12).  Each stage restates one sklearn function:
//
//   1. kNN          NearestNeighbors(algorithm='auto').kneighbors_graph: for d > 15 sklearn is brute force, so the k
//                   nearest rows are exact.  tsne_knn_kernel streams candidate tiles past a block of 64 query rows and
//                   keeps each row's k best (d^2, index) pairs, lexicographically ascending, in shared memory; the
//                   query row itself is excluded.  d^2 is summed in the difference form sum_c (x_c - y_c)^2 (fp32), so
//                   equal rows give exactly 0; the k selected d^2 are then summed again in fp64 (tsne_refine_kernel).
//                   n x n is never stored.
//   2. calibration  _utils.pyx _binary_search_perplexity, one warp per row in fp64 on the fp32 d^2.
//   3. symmetrise   _joint_probabilities_nn: P = (P_cond + P_cond^T) / sum.  Both (i, j, p) and (j, i, p) are emitted,
//                   radix-sorted on the key i << 32 | j, equal keys added (at most two), zeros dropped as scipy's
//                   sparse sum drops them, and the total added in a fixed order.
//   4. PCA start    PCA(n_components=2) (covariance_eigh / full: both the exact top two right singular vectors of the
//                   centred X): X^T X of the centred rows (gram_launch), Jacobi eigh (eigh_launch), svd_flip's sign rule,
//                   projection, and the first column scaled to standard deviation 1e-4.
//   5. gradient     _barnes_hut_tsne.pyx gradient on the cells of _quad_tree.pyx.  The quadtree is built compressed
//                   from the points' cell paths (Morton keys, CUB sort, Karras' binary radix tree): a binary node whose
//                   longest common prefix is delta bits lies in the quadtree cell of depth delta / 2, the deepest cell
//                   holding exactly its points.  sklearn tests the cells of such a one-child chain from the top with the
//                   same barycentre and count, and its acceptance test squared_max_width / d^2 < angle^2 only gets
//                   easier down the chain, so testing the deepest cell of the chain decides the same way.  A binary
//                   node in the same quadtree cell as its parent (a split on the cell's second bit) is not a quadtree
//                   cell and is passed through untested.  A cell is a leaf when all its points lie within 1e-6 of its
//                   lowest-index point (sklearn inserts in index order, so that point is its leaf's barycentre).  Points
//                   whose 32-level paths are equal but which are not such duplicates (a root wider than ~2^32 * 1e-6)
//                   are not a leaf: the walk goes on through the index-split nodes below, all in the same depth-32 cell
//                   and so untested, to the single points, as sklearn's deeper cells separate them.
//                   Counts, barycentres and bounding boxes are combined bottom-up, left child first (integer visit
//                   counters, no floating-point atomics), and every sum is in a fixed order: two runs give the same bits.
//   6. optimiser    _gradient_descent / TSNE._tsne: 250 iterations at momentum 0.5 with P exaggerated, then momentum 0.8;
//                   gains +0.2 / x0.8 by the sign of update . grad, floor 0.01; KL error, n_iter_without_progress and
//                   min_grad_norm checked every 50 iterations -- the only device-to-host reads of the loop.
//
// gemb_launch_count counts this file's own kernels; the CUB sorts and scan it calls are not counted.
#include "common.cuh"
#include <cub/cub.cuh>
#include <chrono>
#include <climits>
#include <cmath>
#include <vector>

namespace gemb {

constexpr int KNN_QB = 64, KNN_CB = 128, KNN_KC = 32;   // query rows per CTA, candidate columns per tile, dims per stage
constexpr int TSNE_KMAX = 320;                          // the row lists of a CTA fit in shared memory up to here
constexpr int TSNE_DMAX = 1024;                         // the PCA start's eigh_launch: one Jacobi rotation pair per thread
constexpr int TSNE_STACK = 128;                         // traversal depth: 64 key bits + 32 index bits of tie-break
constexpr float TSNE_DUP_EPS = 1e-6f;                   // _quad_tree.pyx EPSILON
constexpr float FLOAT32_TINY = 1.17549435e-38f;         // np.finfo(np.float32).tiny

__device__ __forceinline__ bool nb_less(float a, int ia, float b, int ib) { return a < b || (a == b && ia < ib); }

// warp sum in xor-butterfly order: every lane holds the same bits
__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------------ 1. exact kNN
// Block: 256 threads; thread (tr, tc) = (tid / 16, tid % 16) computes rows 4 tr .. 4 tr + 3 against columns tc + 16 c,
// c < 8, of the 64 x 128 tile.  Warp w then merges rows w, w + 8, ... of the tile into their lists: candidates below the
// row's current k-th pair are inserted one at a time (lane order = column order).  Dynamic shared memory: the tile
// and the lists.
__global__ void __launch_bounds__(256) tsne_knn_kernel(int64_t n, int d, int k, const float *__restrict__ X,
                                                       int32_t *__restrict__ idx_out, float *__restrict__ d2_out) {
    extern __shared__ __align__(16) unsigned char knn_smem[];
    float (*tile)[KNN_CB + 1] = (float (*)[KNN_CB + 1])knn_smem;    // KNN_QB x (KNN_CB + 1)
    float *ld = (float *)knn_smem + KNN_QB * (KNN_CB + 1);            // KNN_QB x k
    int *li = (int *)(ld + (size_t)KNN_QB * k);                        // KNN_QB x k
    __shared__ float xq[KNN_KC][KNN_QB + 1];
    __shared__ float xc[KNN_KC][KNN_CB + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tr = tid >> 4, tc = tid & 15;
    const int64_t i0 = (int64_t)blockIdx.x * KNN_QB;
    for (int t = tid; t < KNN_QB * k; t += 256) { ld[t] = INFINITY; li[t] = INT_MAX; }
    for (int64_t j0 = 0; j0 < n; j0 += KNN_CB) {
        float acc[4][8];
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int c = 0; c < 8; c++) acc[r][c] = 0.f;
        for (int k0 = 0; k0 < d; k0 += KNN_KC) {
            const int kc = min(KNN_KC, d - k0);
            __syncthreads();
            for (int t = tid; t < KNN_QB * KNN_KC; t += 256) {
                const int r = t / KNN_KC, kk = t % KNN_KC;
                const int64_t i = i0 + r;
                xq[kk][r] = (i < n && kk < kc) ? X[i * d + k0 + kk] : 0.f;
            }
            for (int t = tid; t < KNN_CB * KNN_KC; t += 256) {
                const int c = t / KNN_KC, kk = t % KNN_KC;
                const int64_t j = j0 + c;
                xc[kk][c] = (j < n && kk < kc) ? X[j * d + k0 + kk] : 0.f;
            }
            __syncthreads();
            for (int kk = 0; kk < kc; kk++) {
                float a[4], b[8];
#pragma unroll
                for (int r = 0; r < 4; r++) a[r] = xq[kk][4 * tr + r];
#pragma unroll
                for (int c = 0; c < 8; c++) b[c] = xc[kk][tc + 16 * c];
#pragma unroll
                for (int r = 0; r < 4; r++)
#pragma unroll
                    for (int c = 0; c < 8; c++) {
                        const float df = a[r] - b[c];
                        acc[r][c] = fmaf(df, df, acc[r][c]);
                    }
            }
        }
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int c = 0; c < 8; c++) tile[4 * tr + r][tc + 16 * c] = acc[r][c];
        __syncthreads();
        for (int r = warp; r < KNN_QB; r += 8) {
            const int64_t i = i0 + r;
            if (i >= n) break;
            float *rd = ld + (size_t)r * k;
            int *ri = li + (size_t)r * k;
            for (int h = 0; h < KNN_CB / 32; h++) {
                const int c = lane + 32 * h;
                const int64_t j = j0 + c;
                const float v = tile[r][c];
                const bool valid = j < n && j != i;
                const unsigned m0 = __ballot_sync(0xffffffffu, valid && nb_less(v, (int)j, rd[k - 1], ri[k - 1]));
                for (unsigned m = m0; m; m &= m - 1) {
                    const int src = __ffs(m) - 1;
                    const float cv = __shfl_sync(0xffffffffu, v, src);
                    const int cj = __shfl_sync(0xffffffffu, (int)j, src);
                    if (!nb_less(cv, cj, rd[k - 1], ri[k - 1])) continue;    // the k-th pair moved down meanwhile
                    int below = 0;
                    for (int t = lane; t < k; t += 32) below += nb_less(rd[t], ri[t], cv, cj);
                    const int pos = __reduce_add_sync(0xffffffffu, below);
                    for (int top = k - 1; top > pos; top -= 32) {          // entries pos .. k-2 move up by one
                        const int t = top - lane;
                        float sv = 0.f;
                        int si = 0;
                        if (t > pos) { sv = rd[t - 1]; si = ri[t - 1]; }
                        __syncwarp();
                        if (t > pos) { rd[t] = sv; ri[t] = si; }
                        __syncwarp();
                    }
                    if (lane == 0) { rd[pos] = cv; ri[pos] = cj; }
                    __syncwarp();
                }
            }
        }
    }
    __syncthreads();
    for (int t = tid; t < KNN_QB * k; t += 256) {
        const int64_t i = i0 + t / k;
        if (i < n) { idx_out[i0 * k + t] = li[t]; d2_out[i0 * k + t] = ld[t]; }
    }
}

// The selected pairs' d^2 again in fp64 (difference form), rounded to fp32 as sklearn rounds its fp64 distances before
// the calibration, and each row re-sorted by (d^2, index).  The fp32 sums of the selection are within a few ulp, but
// exp(-beta d^2) turns that into ~5e-5 of P; the fp64 sums make P agree with sklearn's to ~1e-10.  One warp per row.
__global__ void __launch_bounds__(256) tsne_refine_kernel(int64_t n, int d, int k, const float *__restrict__ X,
                                                          int32_t *__restrict__ idx, float *__restrict__ d2) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = (int64_t)gridDim.x * 8;
    for (int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += nw) {
        int32_t *ri = idx + i * k;
        float *rd = d2 + i * k;
        for (int t = 0; t < k; t++) {
            const int64_t j = ri[t];
            double s = 0.0;
            for (int c = lane; c < d; c += 32) {
                const double df = (double)X[i * d + c] - (double)X[j * d + c];
                s += df * df;
            }
            s = warp_sum(s);
            if (lane == 0) rd[t] = (float)s;
        }
        __syncwarp();
        if (lane == 0)
            for (int t = 1; t < k; t++) {
                const float v = rd[t];
                const int32_t w = ri[t];
                int u = t;
                for (; u > 0 && nb_less(v, w, rd[u - 1], ri[u - 1]); u--) { rd[u] = rd[u - 1]; ri[u] = ri[u - 1]; }
                rd[u] = v;
                ri[u] = w;
            }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------ 2. calibration
// _binary_search_perplexity: beta = 1, at most 100 bisection steps, stop when |H - log(perplexity)| <= 1e-5; the row
// sum floored at 1e-8 (both sklearn's float constants).

__global__ void __launch_bounds__(256) tsne_calibrate_kernel(int64_t n, int k, const float *__restrict__ d2,
                                                             double desired_entropy, double *__restrict__ P) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = (int64_t)gridDim.x * 8;
    const double eps_row = (double)1e-8f, tol = (double)1e-5f;
    for (int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += nw) {
        const float *di = d2 + i * k;
        double *pi = P + i * k;
        double beta = 1.0, beta_min = -INFINITY, beta_max = INFINITY;
        for (int step = 0; step < 100; step++) {
            double s = 0.0;
            for (int t = lane; t < k; t += 32) s += exp(-(double)di[t] * beta);
            double sum_p = warp_sum(s);
            if (sum_p == 0.0) sum_p = eps_row;
            double sd = 0.0;
            for (int t = lane; t < k; t += 32) {
                const double p = exp(-(double)di[t] * beta) / sum_p;
                pi[t] = p;
                sd += (double)di[t] * p;
            }
            const double entropy = log(sum_p) + beta * warp_sum(sd);
            const double diff = entropy - desired_entropy;
            if (fabs(diff) <= tol) break;
            if (diff > 0.0) {
                beta_min = beta;
                beta = beta_max == INFINITY ? beta * 2.0 : (beta + beta_max) / 2.0;
            } else {
                beta_max = beta;
                beta = beta_min == -INFINITY ? beta / 2.0 : (beta + beta_min) / 2.0;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ 3. symmetrise
__global__ void tsne_emit_kernel(int64_t n, int k, const int32_t *__restrict__ idx, const double *__restrict__ Pc,
                                 uint64_t *__restrict__ keys, double *__restrict__ vals) {
    const int64_t m = n * k;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t i = (uint64_t)(t / k), j = (uint64_t)idx[t];
        keys[2 * t] = i << 32 | j;
        keys[2 * t + 1] = j << 32 | i;
        vals[2 * t] = vals[2 * t + 1] = Pc[t];
    }
}

// keep[t] = 1 where t starts a run of equal keys whose sum (at most two entries) is not 0; sum[t] = that sum
__global__ void tsne_runs_kernel(int64_t m, const uint64_t *__restrict__ keys, const double *__restrict__ vals,
                                 int *__restrict__ keep, double *__restrict__ sum) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        const bool head = t == 0 || keys[t] != keys[t - 1];
        const double s = vals[t] + ((t + 1 < m && keys[t + 1] == keys[t]) ? vals[t + 1] : 0.0);
        keep[t] = head && s != 0.0;
        sum[t] = s;
    }
}

__global__ void tsne_compact_kernel(int64_t m, const uint64_t *__restrict__ keys, const int *__restrict__ keep,
                                    const int *__restrict__ pos, const double *__restrict__ sum, int32_t *__restrict__ rows,
                                    int32_t *__restrict__ cols, double *__restrict__ val) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) {
        if (!keep[t]) continue;
        const int p = pos[t];
        rows[p] = (int32_t)(keys[t] >> 32);
        cols[p] = (int32_t)(keys[t] & 0xffffffffu);
        val[p] = sum[t];
    }
}

// indptr[r] = first entry of row r (rows ascending); indptr[n] = nnz
__global__ void tsne_indptr_kernel(int64_t n, int64_t nnz, const int32_t *__restrict__ rows, int64_t *__restrict__ indptr) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= nnz; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t lo = t == 0 ? -1 : rows[t - 1], hi = t == nnz ? n - 1 : rows[t];
        for (int64_t r = lo + 1; r <= hi; r++) indptr[r] = t;
        if (t == nnz) indptr[n] = nnz;
    }
}

// block sum (256 threads) in a fixed order; thread 0 holds it
__device__ __forceinline__ double block_sum(double v, double *red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < 8; w++) t += red[w];
    return t;
}

// part[blockIdx.x] = sum of v[t] over the block's grid-stride share (added by sum_partials_launch in a fixed order)
__global__ void __launch_bounds__(256) tsne_sum_kernel(int64_t m, const double *__restrict__ v, double *__restrict__ part) {
    __shared__ double red[8];
    double s = 0.0;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) s += v[t];
    s = block_sum(s, red);
    if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void tsne_scale_kernel(int64_t m, const double *__restrict__ total, double *__restrict__ v) {
    const double s = fmax(*total, 2.220446049250313e-16);        // np.maximum(P.sum(), MACHINE_EPSILON)
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += (int64_t)gridDim.x * blockDim.x) v[t] /= s;
}

// ------------------------------------------------------------------------------------------------ 4. PCA start
// part[blk * d + c] = sum of X[i, c] over the block's rows
__global__ void tsne_colsum_kernel(int64_t n, int d, const float *__restrict__ X, double *__restrict__ part) {
    for (int c = threadIdx.x; c < d; c += blockDim.x) {
        double s = 0.0;
        for (int64_t i = blockIdx.x; i < n; i += gridDim.x) s += X[i * d + c];
        part[(size_t)blockIdx.x * d + c] = s;
    }
}

__global__ void tsne_center_kernel(int64_t n, int d, const float *__restrict__ X, const double *__restrict__ colsum,
                                   float *__restrict__ Xc) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n * d; t += (int64_t)gridDim.x * blockDim.x)
        Xc[t] = (float)((double)X[t] - colsum[t % d] / (double)n);
}

// V (d x 2): the eigenvectors of the two largest eigenvalues (Z's last two columns), each signed so that its
// largest-magnitude entry (the first on a tie) is positive -- svd_flip(u_based_decision=False)
__global__ void tsne_components_kernel(int d, const double *__restrict__ Z, double *__restrict__ V) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    for (int q = 0; q < 2; q++) {
        const int col = d - 1 - q;
        if (col < 0) {                           // d = 1: a single component
            for (int r = 0; r < d; r++) V[r * 2 + q] = 0.0;
            continue;
        }
        int arg = 0;
        for (int r = 1; r < d; r++)
            if (fabs(Z[(size_t)r * d + col]) > fabs(Z[(size_t)arg * d + col])) arg = r;
        const double s = Z[(size_t)arg * d + col] < 0.0 ? -1.0 : 1.0;
        for (int r = 0; r < d; r++) V[r * 2 + q] = s * Z[(size_t)r * d + col];
    }
}

// Y[i] = (float) (Xc[i] . V), one warp per row
__global__ void __launch_bounds__(256) tsne_project_kernel(int64_t n, int d, const float *__restrict__ Xc,
                                                           const double *__restrict__ V, float *__restrict__ Y) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = (int64_t)gridDim.x * 8;
    for (int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += nw) {
        double a = 0.0, b = 0.0;
        for (int c = lane; c < d; c += 32) {
            const double x = Xc[i * d + c];
            a += x * V[2 * c];
            b += x * V[2 * c + 1];
        }
        a = warp_sum(a);
        b = warp_sum(b);
        if (lane == 0) { Y[2 * i] = (float)a; Y[2 * i + 1] = (float)b; }
    }
}

// part[blk] / part[grid + blk]: sums of y0 and y0^2 (two passes would need the mean first; the spread of the PCA
// scores is far from cancellation at the 1e-4 precision asked of the start)
__global__ void __launch_bounds__(256) tsne_moments_kernel(int64_t n, const float *__restrict__ Y, double *__restrict__ part) {
    __shared__ double red[8];
    double s = 0.0, q = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const double y = Y[2 * i];
        s += y;
        q += y * y;
    }
    s = block_sum(s, red);
    q = block_sum(q, red);
    if (threadIdx.x == 0) { part[blockIdx.x] = s; part[gridDim.x + blockIdx.x] = q; }
}

// X_embedded / np.std(X_embedded[:, 0]) * 1e-4, in fp32 as numpy does it
__global__ void tsne_pca_scale_kernel(int64_t n, const double *__restrict__ mom, float *__restrict__ Y) {
    const double mean = mom[0] / n, var = fmax(mom[1] / n - mean * mean, 0.0);
    const float sd = (float)sqrt(var);
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < 2 * n; t += (int64_t)gridDim.x * blockDim.x)
        Y[t] = Y[t] / sd * 1e-4f;
}

// ------------------------------------------------------------------------------------------------ 5. quadtree
// Nodes 0 .. n-2: internal nodes of the binary radix tree (0 = root); n-1 .. 2n-2: the points in key order.
struct TsneTree {
    int64_t n;
    uint64_t *keys;       // sorted cell paths
    int32_t *perm;        // point of each sorted position
    int32_t *child;       // 2 (n - 1): left, right
    int32_t *parent;      // 2n - 1 (root: -1)
    int32_t *first;       // n - 1: first sorted position of the node's range
    int32_t *delta;       // n - 1: longest common prefix of the range (bits; > 64 for equal keys)
    int32_t *visit;       // n - 1: bottom-up arrival counters
    int32_t *cnt, *minidx;        // 2n - 1
    double2 *sum;                 // 2n - 1
    float4 *bbox;                 // 2n - 1: (min x, min y, max x, max y)
    float4 *node;                 // 2n - 1: (barycentre x, y, squared_max_width, cumulative_size)
    uint8_t *leaf, *testable;     // 2n - 1
    float4 *root;                 // (min x, min y, max x, max y) of the root cell
};

__global__ void __launch_bounds__(256) tsne_bbox_kernel(int64_t n, const float *__restrict__ Y, float4 *__restrict__ part) {
    __shared__ float4 red[256];
    float4 b = make_float4(INFINITY, INFINITY, -INFINITY, -INFINITY);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = Y[2 * i], y = Y[2 * i + 1];
        b = make_float4(fminf(b.x, x), fminf(b.y, y), fmaxf(b.z, x), fmaxf(b.w, y));
    }
    red[threadIdx.x] = b;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            const float4 o = red[threadIdx.x + s];
            b = make_float4(fminf(b.x, o.x), fminf(b.y, o.y), fmaxf(b.z, o.z), fmaxf(b.w, o.w));
            red[threadIdx.x] = b;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = b;
}

// the root cell of QuadTree.build_tree: [min, M] with M = max(M (1 + 1e-3 sign M), M + 1e-3), in fp32
__device__ __forceinline__ float tsne_widen(float M) {
    const float sg = M > 0.f ? 1.f : (M < 0.f ? -1.f : 0.f);
    return fmaxf(M * (1.f + 1e-3f * sg), M + 1e-3f);
}

__global__ void tsne_root_kernel(int parts, const float4 *__restrict__ part, float4 *__restrict__ root) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float4 b = part[0];
    for (int p = 1; p < parts; p++) {
        const float4 o = part[p];
        b = make_float4(fminf(b.x, o.x), fminf(b.y, o.y), fmaxf(b.z, o.z), fmaxf(b.w, o.w));
    }
    *root = make_float4(b.x, b.y, tsne_widen(b.z), tsne_widen(b.w));
}

// The cell path of a point: at each of 32 levels the child _select_child picks, point >= (lo + hi) / 2 per axis
// (x then y), the bounds halved in fp32 exactly as the tree's cells are.
__global__ void tsne_morton_kernel(int64_t n, const float *__restrict__ Y, const float4 *__restrict__ root,
                                   uint64_t *__restrict__ keys, int32_t *__restrict__ perm) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 r = *root;
    float lx = r.x, ly = r.y, hx = r.z, hy = r.w;
    const float x = Y[2 * i], y = Y[2 * i + 1];
    uint64_t key = 0;
    for (int l = 0; l < 32; l++) {
        const float cx = (lx + hx) * 0.5f, cy = (ly + hy) * 0.5f;
        const int bx = x >= cx, by = y >= cy;
        if (bx) lx = cx; else hx = cx;
        if (by) ly = cy; else hy = cy;
        key = key << 2 | (uint64_t)(bx << 1 | by);
    }
    keys[i] = key;
    perm[i] = (int32_t)i;
}

__device__ __forceinline__ int tsne_delta(const uint64_t *keys, int64_t n, int64_t i, int64_t j) {
    if (j < 0 || j >= n) return -1;
    const uint64_t a = keys[i], b = keys[j];
    return a != b ? __clzll(a ^ b) : 64 + __clz((unsigned)(i ^ j));
}

// Karras (2012): internal node i covers the sorted range [min(i, j), max(i, j)] and splits at gamma
__global__ void tsne_karras_kernel(TsneTree T) {
    const int64_t n = T.n;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n - 1) return;
    const uint64_t *K = T.keys;
    const int dir = tsne_delta(K, n, i, i + 1) - tsne_delta(K, n, i, i - 1) >= 0 ? 1 : -1;
    const int dmin = tsne_delta(K, n, i, i - dir);
    int64_t lmax = 2;
    while (tsne_delta(K, n, i, i + lmax * dir) > dmin) lmax *= 2;
    int64_t l = 0;
    for (int64_t t = lmax / 2; t >= 1; t /= 2)
        if (tsne_delta(K, n, i, i + (l + t) * dir) > dmin) l += t;
    const int64_t j = i + l * dir;
    const int dnode = tsne_delta(K, n, i, j);
    int64_t s = 0;
    for (int64_t div = 2;; div *= 2) {
        const int64_t t = (l + div - 1) / div;
        if (tsne_delta(K, n, i, i + (s + t) * dir) > dnode) s += t;
        if (t == 1) break;
    }
    const int64_t gamma = i + s * dir + (dir < 0 ? -1 : 0);
    const int64_t lo = i < j ? i : j, hi = i < j ? j : i;
    const int32_t left = (int32_t)(lo == gamma ? n - 1 + gamma : gamma);
    const int32_t right = (int32_t)(hi == gamma + 1 ? n - 1 + gamma + 1 : gamma + 1);
    T.child[2 * i] = left;
    T.child[2 * i + 1] = right;
    T.parent[left] = (int32_t)i;
    T.parent[right] = (int32_t)i;
    T.first[i] = (int32_t)lo;
    T.delta[i] = dnode;
    T.visit[i] = 0;
    if (i == 0) { T.parent[0] = -1; T.testable[0] = 1; }
}

__device__ __forceinline__ int tsne_depth(int delta) { return min(delta, 64) / 2; }

// squared_max_width of the depth-L cell on the path `key`
__device__ __forceinline__ float tsne_cell_sqw(float4 r, uint64_t key, int L) {
    float lx = r.x, ly = r.y, hx = r.z, hy = r.w;
    for (int l = 0; l < L; l++) {
        const float cx = (lx + hx) * 0.5f, cy = (ly + hy) * 0.5f;
        const int b = (int)(key >> (62 - 2 * l)) & 3;
        if (b & 2) lx = cx; else hx = cx;
        if (b & 1) ly = cy; else hy = cy;
    }
    const float wx = hx - lx, wy = hy - ly;
    return fmaxf(fmaxf(0.f, wx * wx), wy * wy);
}

// One thread per point: its leaf, then up the tree; the second thread to arrive at a node combines the two children
// (left first) and goes on.  Stores are published with a fence before the arrival counter is incremented.
__global__ void tsne_bottom_up_kernel(TsneTree T, const float *__restrict__ Y) {
    const int64_t n = T.n;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const int32_t p = T.perm[t];
    const float x = Y[2 * p], y = Y[2 * p + 1];
    const int64_t leaf = n - 1 + t;
    T.cnt[leaf] = 1;
    T.minidx[leaf] = p;
    T.sum[leaf] = make_double2(x, y);
    T.bbox[leaf] = make_float4(x, y, x, y);
    T.node[leaf] = make_float4(x, y, 0.f, 1.f);
    T.leaf[leaf] = 1;
    T.testable[leaf] = 1;
    __threadfence();
    int32_t v = T.parent[leaf];
    const float4 r = *T.root;
    while (v >= 0) {
        if (atomicAdd(&T.visit[v], 1) == 0) return;
        __threadfence();
        const int32_t a = T.child[2 * v], b = T.child[2 * v + 1];
        const int ca = __ldcg(&T.cnt[a]), cb = __ldcg(&T.cnt[b]);
        const int ma = __ldcg(&T.minidx[a]), mb = __ldcg(&T.minidx[b]);
        const double2 sa = __ldcg(&T.sum[a]), sb = __ldcg(&T.sum[b]);
        const float4 ba = __ldcg(&T.bbox[a]), bb = __ldcg(&T.bbox[b]);
        const int c = ca + cb, m = min(ma, mb);
        const double2 s = make_double2(sa.x + sb.x, sa.y + sb.y);
        const float4 bx = make_float4(fminf(ba.x, bb.x), fminf(ba.y, bb.y), fmaxf(ba.z, bb.z), fmaxf(ba.w, bb.w));
        const int dl = T.delta[v], L = tsne_depth(dl);
        const float px = Y[2 * m], py = Y[2 * m + 1];
        const bool dup = bx.z - px <= TSNE_DUP_EPS && px - bx.x <= TSNE_DUP_EPS && bx.w - py <= TSNE_DUP_EPS &&
                         py - bx.y <= TSNE_DUP_EPS;
        const bool lf = dup;      // equal keys alone are not a leaf: below 32 levels sklearn splits until points separate
        const float sqw = tsne_cell_sqw(r, T.keys[T.first[v]], L);
        T.cnt[v] = c;
        T.minidx[v] = m;
        T.sum[v] = s;
        T.bbox[v] = bx;
        T.node[v] = lf ? make_float4(px, py, sqw, (float)c) : make_float4((float)(s.x / c), (float)(s.y / c), sqw, (float)c);
        T.leaf[v] = lf;
        if (a < n - 1) T.testable[a] = tsne_depth(T.delta[a]) > L;
        if (b < n - 1) T.testable[b] = tsne_depth(T.delta[b]) > L;
        __threadfence();
        v = T.parent[v];
    }
}

// The repulsive half of _barnes_hut_tsne.compute_gradient_negative for every point, by a depth-first walk of the
// compressed tree (left child first).  One thread per sorted position; part[blk]: the block's sum of sum_Q.
__global__ void __launch_bounds__(256) tsne_repulsive_kernel(TsneTree T, const float *__restrict__ Y, float theta2,
                                                             float2 *__restrict__ negf, double *__restrict__ part) {
    __shared__ double red[8];
    const int64_t n = T.n;
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double sq = 0.0;
    if (t < n) {
        const int32_t p = T.perm[t];
        const float px = Y[2 * p], py = Y[2 * p + 1];
        float fx = 0.f, fy = 0.f;
        int stack[TSNE_STACK];
        int sp = 0;
        stack[sp++] = 0;
        while (sp > 0) {
            const int v = stack[--sp];
            if (!T.testable[v]) {
                stack[sp++] = T.child[2 * v + 1];
                stack[sp++] = T.child[2 * v];
                continue;
            }
            const float4 c = T.node[v];
            const float dx = px - c.x, dy = py - c.y;
            const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
            const bool lf = T.leaf[v];
            if (lf && fabsf(dx) <= TSNE_DUP_EPS && fabsf(dy) <= TSNE_DUP_EPS) continue;   // no self interaction
            if (lf || c.z / d2 < theta2) {
                const double q = (double)(1.f / (1.f + d2));
                sq += (double)c.w * q;
                const float mult = (float)((double)c.w * q * q);
                fx = fmaf(mult, dx, fx);
                fy = fmaf(mult, dy, fy);
            } else {
                stack[sp++] = T.child[2 * v + 1];
                stack[sp++] = T.child[2 * v];
            }
        }
        negf[p] = make_float2(fx, fy);
    }
    sq = block_sum(sq, red);
    if (threadIdx.x == 0) part[blockIdx.x] = sq;
}

// ------------------------------------------------------------------------------------------------ gradient + step
// One thread per point: the attractive term over its row of P (compute_gradient_positive, in CSR order), the
// gradient 4 (pos - neg / sum_Q) (fp32, as sklearn stores it), and then either the gradient is written out (grad != 0)
// or one step of _gradient_descent is taken from Y into Ynext.  part[blk] = KL terms, part[grid + blk] = |gains * grad|^2 (fp64).
struct TsneStep {
    float momentum;
    double learning_rate;
    double *update;     // n x 2 (fp64: update = momentum * update - learning_rate * grad, learning_rate a float64)
    float *gains;       // n x 2
};

__global__ void __launch_bounds__(256) tsne_step_kernel(int64_t n, const int64_t *__restrict__ indptr,
                                                        const int32_t *__restrict__ indices, const double *__restrict__ pval,
                                                        double exaggeration, const float2 *__restrict__ negf,
                                                        const double *__restrict__ sum_q, int compute_error,
                                                        const float *__restrict__ Y, float *__restrict__ Ynext,
                                                        float *__restrict__ grad, TsneStep st, double *__restrict__ part) {
    __shared__ double red[8];
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    double err = 0.0, gn = 0.0;
    const double sQ = fmax(*sum_q, 2.220446049250313e-16);     // compute_gradient_negative's floor (FLOAT64_EPS)
    float g[2] = {0.f, 0.f};
    if (i < n) {
        const float xi = Y[2 * i], yi = Y[2 * i + 1];
        float fx = 0.f, fy = 0.f;
        for (int64_t e = indptr[i]; e < indptr[i + 1]; e++) {
            const int32_t j = indices[e];
            const float pij = (float)(exaggeration * pval[e]);
            const float bx = xi - Y[2 * j], by = yi - Y[2 * j + 1];
            const float dij = __fadd_rn(__fmul_rn(bx, bx), __fmul_rn(by, by));
            const float qij = 1.f / (1.f + dij);
            const float w = pij * qij;
            if (compute_error) {
                const float qn = (float)((double)qij / sQ);
                err += (double)pij * log((double)(fmaxf(pij, FLOAT32_TINY) / fmaxf(qn, FLOAT32_TINY)));
            }
            fx = fmaf(w, bx, fx);
            fy = fmaf(w, by, fy);
        }
        const float2 nf = negf[i];
        g[0] = (float)((double)fx - (double)nf.x / sQ) * 4.f;
        g[1] = (float)((double)fy - (double)nf.y / sQ) * 4.f;
    }
    if (i < n) {
        if (grad) {
            grad[2 * i] = g[0];
            grad[2 * i + 1] = g[1];
        } else {
            for (int a = 0; a < 2; a++) {
                const int64_t o = 2 * i + a;
                double u = st.update[o];
                float gain = st.gains[o];
                gain = u * (double)g[a] < 0.0 ? gain + 0.2f : gain * 0.8f;
                gain = fmaxf(gain, 0.01f);
                st.gains[o] = gain;
                const float ga = g[a] * gain;
                gn += (double)ga * ga;
                u = (double)st.momentum * u - st.learning_rate * (double)ga;
                st.update[o] = u;
                Ynext[o] = (float)((double)Y[o] + u);
            }
        }
    }
    err = block_sum(err, red);
    gn = block_sum(gn, red);
    if (threadIdx.x == 0) { part[blockIdx.x] = err; part[gridDim.x + blockIdx.x] = gn; }
}

}  // namespace gemb

using namespace gemb;

namespace {

using Clock = std::chrono::steady_clock;
double ms_since(Clock::time_point t0) { return std::chrono::duration<double, std::milli>(Clock::now() - t0).count(); }

int tsne_k(int64_t n, double perplexity) { return (int)std::min<int64_t>(n - 1, (int64_t)(3.0 * perplexity + 1.0)); }

int tsne_check_x(int64_t n, int d, const float *X) {
    GEMB_ARG(X && n >= 2 && d >= 1, "X, n >= 2, d >= 1");
    for (int64_t t = 0; t < n * d; t++) GEMB_ARG(std::isfinite(X[t]), "X finite");
    return GEMB_OK;
}

// Stages 1-3 on the device.  Out: knn idx / d2 (n x k), conditional P (n x k), joint P as CSR (nnz entries).
struct Affinities {
    int k = 0;
    int64_t nnz = 0;
    DeviceBuffer<int32_t> idx, rows, cols;
    DeviceBuffer<float> d2;
    DeviceBuffer<double> pcond, val;
    DeviceBuffer<int64_t> indptr;
};

int tsne_affinities(gemb_ctx *ctx, int64_t n, int d, const float *dX, double perplexity, Affinities &A, double *knn_ms,
                    double *calib_ms, double *sym_ms) {
    const int k = tsne_k(n, perplexity);
    A.k = k;
    cudaStream_t st = ctx->stream;
    auto t0 = Clock::now();
    const size_t smem = sizeof(float) * KNN_QB * (KNN_CB + 1) + (size_t)KNN_QB * k * 8;
    GEMB_CUDA(cudaFuncSetAttribute(tsne_knn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    GEMB_CUDA(A.idx.alloc((size_t)n * k));
    GEMB_CUDA(A.d2.alloc((size_t)n * k));
    GEMB_TRY(launch(ctx, tsne_knn_kernel, (unsigned)((n + KNN_QB - 1) / KNN_QB), 256, smem, n, d, k, dX, A.idx.get(), A.d2.get()));
    GEMB_TRY(launch(ctx, tsne_refine_kernel, grid_stride(ctx, n, 8, 16), 256, 0, n, d, k, dX, A.idx.get(), A.d2.get()));
    GEMB_CUDA(cudaStreamSynchronize(st));
    if (knn_ms) *knn_ms = ms_since(t0);

    t0 = Clock::now();
    GEMB_CUDA(A.pcond.alloc((size_t)n * k));
    GEMB_TRY(launch(ctx, tsne_calibrate_kernel, grid_stride(ctx, n, 8, 16), 256, 0, n, k, A.d2.get(),
                    std::log((double)(float)perplexity), A.pcond.get()));
    GEMB_CUDA(cudaStreamSynchronize(st));
    if (calib_ms) *calib_ms = ms_since(t0);

    t0 = Clock::now();
    const int64_t m = 2 * n * k;
    GEMB_ARG(m < ((int64_t)1 << 31), "2 n k < 2^31 (the symmetrised pairs are sorted in one CUB call)");
    DeviceBuffer<uint64_t> k0, k1;
    DeviceBuffer<double> v0, v1, sum;
    DeviceBuffer<int> keep, pos;
    GEMB_CUDA(k0.alloc(m)); GEMB_CUDA(k1.alloc(m));
    GEMB_CUDA(v0.alloc(m)); GEMB_CUDA(v1.alloc(m));
    const int g = grid_stride(ctx, m, 256, 8);
    GEMB_TRY(launch(ctx, tsne_emit_kernel, grid_stride(ctx, n * k, 256, 8), 256, 0, n, k, A.idx.get(), A.pcond.get(), k0.get(), v0.get()));
    {
        size_t tb = 0;
        GEMB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k0.get(), k1.get(), v0.get(), v1.get(), (int)m, 0, 64, st));
        DeviceBuffer<unsigned char> tmp;
        GEMB_CUDA(tmp.alloc(tb));
        GEMB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.get(), tb, k0.get(), k1.get(), v0.get(), v1.get(), (int)m, 0, 64, st));
    }
    v0.reset();
    GEMB_CUDA(sum.alloc(m)); GEMB_CUDA(keep.alloc(m)); GEMB_CUDA(pos.alloc(m));
    GEMB_TRY(launch(ctx, tsne_runs_kernel, g, 256, 0, m, k1.get(), v1.get(), keep.get(), sum.get()));
    {
        size_t tb = 0;
        GEMB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, keep.get(), pos.get(), (int)m, st));
        DeviceBuffer<unsigned char> tmp;
        GEMB_CUDA(tmp.alloc(tb));
        GEMB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb, keep.get(), pos.get(), (int)m, st));
    }
    int last[2];
    GEMB_CUDA(cudaMemcpyAsync(&last[0], pos.get() + m - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(&last[1], keep.get() + m - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    const int64_t nnz = (int64_t)last[0] + last[1];
    A.nnz = nnz;
    GEMB_CUDA(A.rows.alloc(nnz)); GEMB_CUDA(A.cols.alloc(nnz)); GEMB_CUDA(A.val.alloc(nnz));
    GEMB_CUDA(A.indptr.alloc(n + 1));
    GEMB_TRY(launch(ctx, tsne_compact_kernel, g, 256, 0, m, k1.get(), keep.get(), pos.get(), sum.get(), A.rows.get(),
                    A.cols.get(), A.val.get()));
    GEMB_TRY(launch(ctx, tsne_indptr_kernel, grid_stride(ctx, nnz + 1, 256, 8), 256, 0, n, nnz, A.rows.get(), A.indptr.get()));
    const int gs = grid_stride(ctx, nnz, 256, 4);
    double *part = nullptr;
    GEMB_TRY(red_scratch(ctx, gs, &part));
    GEMB_TRY(launch(ctx, tsne_sum_kernel, gs, 256, 0, nnz, A.val.get(), part));
    GEMB_TRY(sum_partials_launch(ctx, gs, 1, part, sum.get()));
    GEMB_TRY(launch(ctx, tsne_scale_kernel, grid_stride(ctx, nnz, 256, 8), 256, 0, nnz, sum.get(), A.val.get()));
    GEMB_CUDA(cudaStreamSynchronize(st));
    if (sym_ms) *sym_ms = ms_since(t0);
    return GEMB_OK;
}

int tsne_pca(gemb_ctx *ctx, int64_t n, int d, const float *dX, float *dY) {
    DeviceBuffer<float> Xc;
    DeviceBuffer<double> colsum, G, w, Z, Zs, V, mom;
    GEMB_CUDA(Xc.alloc((size_t)n * d));
    GEMB_CUDA(colsum.alloc(d)); GEMB_CUDA(G.alloc((size_t)d * d)); GEMB_CUDA(w.alloc(d));
    GEMB_CUDA(Z.alloc((size_t)d * d)); GEMB_CUDA(Zs.alloc((size_t)d * d)); GEMB_CUDA(V.alloc(2 * (size_t)d)); GEMB_CUDA(mom.alloc(2));
    const int gc = (int)std::min<int64_t>(n, (int64_t)ctx->sm_count * 4);
    double *part = nullptr;
    GEMB_TRY(red_scratch(ctx, (size_t)gc * d, &part));
    GEMB_TRY(launch(ctx, tsne_colsum_kernel, gc, 256, 0, n, d, dX, part));
    GEMB_TRY(sum_partials_launch(ctx, gc, d, part, colsum.get()));
    GEMB_TRY(launch(ctx, tsne_center_kernel, grid_stride(ctx, n * d, 256, 8), 256, 0, n, d, dX, colsum.get(), Xc.get()));
    GEMB_TRY(gram_launch(ctx, n, Xc.get(), d, Xc.get(), d, G.get()));
    GEMB_TRY(eigh_launch(ctx, d, G.get(), w.get(), Z.get(), Zs.get()));
    GEMB_TRY(launch(ctx, tsne_components_kernel, 1, 32, 0, d, Z.get(), V.get()));
    GEMB_TRY(launch(ctx, tsne_project_kernel, grid_stride(ctx, n, 8, 16), 256, 0, n, d, Xc.get(), V.get(), dY));
    const int gm = grid_stride(ctx, n, 256, 4);
    GEMB_TRY(red_scratch(ctx, 2 * (size_t)gm, &part));
    GEMB_TRY(launch(ctx, tsne_moments_kernel, gm, 256, 0, n, dY, part));
    GEMB_TRY(sum_partials_launch(ctx, gm, 1, part, mom.get()));
    GEMB_TRY(sum_partials_launch(ctx, gm, 1, part + gm, mom.get() + 1));
    return launch(ctx, tsne_pca_scale_kernel, grid_stride(ctx, 2 * n, 256, 8), 256, 0, n, mom.get(), dY);
}

// The tree's device blocks, allocated once per call
struct TreeBuffers {
    DeviceBuffer<uint64_t> keys_in, keys;
    DeviceBuffer<int32_t> perm_in, perm, child, parent, first, delta, visit, cnt, minidx;
    DeviceBuffer<double2> sum;
    DeviceBuffer<float4> bbox, node, bpart, root;
    DeviceBuffer<uint8_t> leaf, testable;
    DeviceBuffer<unsigned char> sort_tmp;
    size_t sort_bytes = 0;
    TsneTree T{};
    int bbox_grid = 1;

    int alloc(gemb_ctx *ctx, int64_t n) {
        const size_t nn = 2 * n - 1;
        GEMB_CUDA(keys_in.alloc(n)); GEMB_CUDA(keys.alloc(n)); GEMB_CUDA(perm_in.alloc(n)); GEMB_CUDA(perm.alloc(n));
        GEMB_CUDA(child.alloc(2 * (n - 1))); GEMB_CUDA(parent.alloc(nn)); GEMB_CUDA(first.alloc(n - 1));
        GEMB_CUDA(delta.alloc(n - 1)); GEMB_CUDA(visit.alloc(n - 1)); GEMB_CUDA(cnt.alloc(nn)); GEMB_CUDA(minidx.alloc(nn));
        GEMB_CUDA(sum.alloc(nn)); GEMB_CUDA(bbox.alloc(nn)); GEMB_CUDA(node.alloc(nn));
        GEMB_CUDA(leaf.alloc(nn)); GEMB_CUDA(testable.alloc(nn));
        bbox_grid = grid_stride(ctx, n, 256, 2);
        GEMB_CUDA(bpart.alloc(bbox_grid)); GEMB_CUDA(root.alloc(1));
        GEMB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, keys_in.get(), keys.get(), perm_in.get(), perm.get(),
                                                  (int)n, 0, 64, ctx->stream));
        GEMB_CUDA(sort_tmp.alloc(sort_bytes));
        T.n = n; T.keys = keys.get(); T.perm = perm.get(); T.child = child.get(); T.parent = parent.get();
        T.first = first.get(); T.delta = delta.get(); T.visit = visit.get(); T.cnt = cnt.get(); T.minidx = minidx.get();
        T.sum = sum.get(); T.bbox = bbox.get(); T.node = node.get(); T.leaf = leaf.get(); T.testable = testable.get();
        T.root = root.get();
        return GEMB_OK;
    }

    int build(gemb_ctx *ctx, const float *dY) {
        const int64_t n = T.n;
        const unsigned gp = (unsigned)((n + 255) / 256);
        GEMB_TRY(launch(ctx, tsne_bbox_kernel, bbox_grid, 256, 0, n, dY, bpart.get()));
        GEMB_TRY(launch(ctx, tsne_root_kernel, 1, 32, 0, bbox_grid, bpart.get(), root.get()));
        GEMB_TRY(launch(ctx, tsne_morton_kernel, gp, 256, 0, n, dY, root.get(), keys_in.get(), perm_in.get()));
        size_t tb = sort_bytes;
        GEMB_CUDA(cub::DeviceRadixSort::SortPairs(sort_tmp.get(), tb, keys_in.get(), keys.get(), perm_in.get(), perm.get(),
                                                  (int)n, 0, 64, ctx->stream));
        GEMB_TRY(launch(ctx, tsne_karras_kernel, (unsigned)((n - 1 + 255) / 256), 256, 0, T));
        return launch(ctx, tsne_bottom_up_kernel, gp, 256, 0, T, dY);
    }
};

// grad (device, n x 2) and KL at positions dY: the tree, the repulsive walk, sum_Q and the attractive sweep
// (grad == nullptr: one optimiser step from dY into dYnext instead)
int tsne_gradient_dev(gemb_ctx *ctx, TreeBuffers &tb, const float *dY, float *dYnext, const int64_t *indptr, const int32_t *indices,
                      const double *pval, double exaggeration, float angle, int compute_error, float *dgrad,
                      const TsneStep &step, float2 *negf, double *sq_dev, double *out2_dev, gemb::Timer *t_tree,
                      gemb::Timer *t_grad) {
    const int64_t n = tb.T.n;
    const int gp = (int)((n + 255) / 256);
    if (t_tree) GEMB_TRY(t_tree->begin(ctx->stream));
    GEMB_TRY(tb.build(ctx, dY));
    if (t_tree) GEMB_TRY(t_tree->end(ctx->stream));
    if (t_grad) GEMB_TRY(t_grad->begin(ctx->stream));
    double *part = nullptr;
    GEMB_TRY(red_scratch(ctx, 2 * (size_t)gp, &part));
    GEMB_TRY(launch(ctx, tsne_repulsive_kernel, gp, 256, 0, tb.T, dY, angle * angle, negf, part));
    GEMB_TRY(sum_partials_launch(ctx, gp, 1, part, sq_dev));
    GEMB_TRY(launch(ctx, tsne_step_kernel, gp, 256, 0, n, indptr, indices, pval, exaggeration, (const float2 *)negf,
                    (const double *)sq_dev, compute_error, dY, dYnext, dgrad, step, part));
    if (compute_error) {
        GEMB_TRY(sum_partials_launch(ctx, gp, 1, part, out2_dev));
        GEMB_TRY(sum_partials_launch(ctx, gp, 1, part + gp, out2_dev + 1));
    }
    if (t_grad) GEMB_TRY(t_grad->end(ctx->stream));
    return GEMB_OK;
}

struct TimerGuard {
    gemb::Timer t;
    ~TimerGuard() { t.destroy(); }
};

}  // namespace

extern "C" int gemb_tsne_affinities(gemb_ctx *ctx, int64_t n, int d, const float *X, double perplexity, int64_t cap,
                                    int32_t *knn_idx_out, float *knn_d2_out, double *p_cond_out, int64_t *p_indptr_out,
                                    int32_t *p_indices_out, double *p_val_out, int32_t *k_out, int64_t *nnz_out) {
    GEMB_ARG(ctx && nnz_out, "ctx, nnz_out");
    GEMB_TRY(tsne_check_x(n, d, X));
    GEMB_ARG(perplexity > 0 && perplexity < n, "0 < perplexity < n");
    GEMB_ARG(tsne_k(n, perplexity) <= TSNE_KMAX, "k = min(n - 1, 3 perplexity + 1) <= 320");
    GEMB_CUDA(cudaSetDevice(ctx->device));
    DeviceBuffer<float> dX;
    GEMB_CUDA(dX.upload(X, (size_t)n * d, ctx->stream));
    Affinities A;
    GEMB_TRY(tsne_affinities(ctx, n, d, dX.get(), perplexity, A, nullptr, nullptr, nullptr));
    *nnz_out = A.nnz;
    if (k_out) *k_out = A.k;
    if (cap == 0) return GEMB_OK;
    GEMB_ARG(cap >= A.nnz && knn_idx_out && knn_d2_out && p_cond_out && p_indptr_out && p_indices_out && p_val_out,
             "cap >= nnz and every output array");
    cudaStream_t st = ctx->stream;
    const size_t nk = (size_t)n * A.k;
    GEMB_CUDA(cudaMemcpyAsync(knn_idx_out, A.idx.get(), sizeof(int32_t) * nk, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(knn_d2_out, A.d2.get(), sizeof(float) * nk, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(p_cond_out, A.pcond.get(), sizeof(double) * nk, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(p_indptr_out, A.indptr.get(), sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(p_indices_out, A.cols.get(), sizeof(int32_t) * A.nnz, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(p_val_out, A.val.get(), sizeof(double) * A.nnz, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    return GEMB_OK;
}

extern "C" int gemb_tsne_gradient(gemb_ctx *ctx, int64_t n, const float *Y, const int64_t *p_indptr,
                                  const int32_t *p_indices, const double *p_val, double angle, float *grad_out,
                                  double *kl_out) {
    GEMB_ARG(ctx && Y && p_indptr && grad_out && n >= 2, "ctx/Y/p_indptr/grad_out, n >= 2");
    GEMB_ARG(angle >= 0 && angle <= 1, "0 <= angle <= 1");
    for (int64_t t = 0; t < 2 * n; t++) GEMB_ARG(std::isfinite(Y[t]), "Y finite");
    const int64_t nnz = p_indptr[n];
    GEMB_ARG(p_indptr[0] == 0 && nnz >= 0 && (nnz == 0 || (p_indices && p_val)), "p_indptr[0] == 0, p_indices, p_val");
    for (int64_t i = 0; i < n; i++) GEMB_ARG(p_indptr[i + 1] >= p_indptr[i], "p_indptr non-decreasing");
    for (int64_t e = 0; e < nnz; e++) GEMB_ARG(p_indices[e] >= 0 && p_indices[e] < n, "p_indices in [0, n)");
    GEMB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DeviceBuffer<float> dY, dG;
    DeviceBuffer<int64_t> dP;
    DeviceBuffer<int32_t> dI;
    DeviceBuffer<double> dV, dS;
    DeviceBuffer<float2> negf;
    GEMB_CUDA(dY.upload(Y, 2 * n, st));
    GEMB_CUDA(dP.upload(p_indptr, n + 1, st));
    GEMB_CUDA(dI.upload(p_indices, nnz, st));
    GEMB_CUDA(dV.upload(p_val, nnz, st));
    GEMB_CUDA(dG.alloc(2 * n));
    GEMB_CUDA(dS.alloc(3));
    GEMB_CUDA(negf.alloc(n));
    TreeBuffers tb;
    GEMB_TRY(tb.alloc(ctx, n));
    GEMB_TRY(tsne_gradient_dev(ctx, tb, dY.get(), nullptr, dP.get(), dI.get(), dV.get(), 1.0, (float)angle, 1, dG.get(), TsneStep{},
                               negf.get(), dS.get(), dS.get() + 1, nullptr, nullptr));
    double kl[2];
    GEMB_CUDA(cudaMemcpyAsync(grad_out, dG.get(), sizeof(float) * 2 * n, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaMemcpyAsync(kl, dS.get() + 1, sizeof(double) * 2, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    if (kl_out) *kl_out = kl[0];
    return GEMB_OK;
}

extern "C" int gemb_tsne(gemb_ctx *ctx, int64_t n, int d, const float *X, const gemb_tsne_opts *opts, float *Y_out,
                         gemb_tsne_stats *stats) {
    GEMB_ARG(ctx && opts && Y_out, "ctx/opts/Y_out");
    GEMB_ARG(opts->struct_size == sizeof(gemb_tsne_opts), "opts->struct_size");
    GEMB_ARG(!stats || stats->struct_size == sizeof(gemb_tsne_stats), "stats->struct_size");
    GEMB_TRY(tsne_check_x(n, d, X));
    const gemb_tsne_opts o = *opts;
    GEMB_ARG(o.perplexity > 0 && o.perplexity < n, "0 < perplexity < n");
    GEMB_ARG(o.early_exaggeration > 0 && o.learning_rate > 0, "early_exaggeration > 0, learning_rate > 0");
    GEMB_ARG(o.angle >= 0 && o.angle <= 1, "0 <= angle <= 1");
    GEMB_ARG(o.max_iter >= 0 && o.n_iter_without_progress >= 0 && o.min_grad_norm >= 0,
             "max_iter, n_iter_without_progress, min_grad_norm >= 0");
    if (tsne_k(n, o.perplexity) > TSNE_KMAX) {
        set_error("k = min(n - 1, 3 perplexity + 1) = %d exceeds %d", tsne_k(n, o.perplexity), TSNE_KMAX);
        return GEMB_ERR_UNSUPPORTED;
    }
    if (d > TSNE_DMAX) {
        set_error("d = %d exceeds %d, the width of the PCA start's Jacobi eigensolver", d, TSNE_DMAX);
        return GEMB_ERR_UNSUPPORTED;
    }
    GEMB_CUDA(cudaSetDevice(ctx->device));
    const auto t_all = Clock::now();
    cudaStream_t st = ctx->stream;
    gemb_tsne_stats S{};
    DeviceBuffer<float> dX, dY, dY2;
    GEMB_CUDA(dX.upload(X, (size_t)n * d, st));
    GEMB_CUDA(dY.alloc(2 * n));
    GEMB_CUDA(dY2.alloc(2 * n));
    Affinities A;
    GEMB_TRY(tsne_affinities(ctx, n, d, dX.get(), o.perplexity, A, &S.knn_ms, &S.calib_ms, &S.sym_ms));
    A.idx.reset(); A.d2.reset(); A.pcond.reset(); A.rows.reset();
    S.n_neighbors = A.k;
    S.nnz_P = A.nnz;
    auto t0 = Clock::now();
    GEMB_TRY(tsne_pca(ctx, n, d, dX.get(), dY.get()));
    GEMB_CUDA(cudaStreamSynchronize(st));
    S.pca_ms = ms_since(t0);
    dX.reset();

    t0 = Clock::now();
    int it_done = -1;
    double error = 0.0;
    if (o.max_iter > 0) {
        DeviceBuffer<double> upd, dS;
        DeviceBuffer<float> gains;
        DeviceBuffer<float2> negf;
        GEMB_CUDA(upd.alloc(2 * n)); GEMB_CUDA(gains.alloc(2 * n)); GEMB_CUDA(negf.alloc(n)); GEMB_CUDA(dS.alloc(3));
        TreeBuffers tb;
        GEMB_TRY(tb.alloc(ctx, n));
        TimerGuard t_tree, t_grad;
        std::vector<float> ones(2 * n, 1.f);
        const int explore = 250, check_every = 50;    // TSNE._EXPLORATION_MAX_ITER, _N_ITER_CHECK
        int it = 0;
        for (int phase = 0; phase < 2; phase++) {
            const int stop = phase == 0 ? std::min(explore, o.max_iter) : o.max_iter;
            if (phase == 1 && !(it_done < explore || o.max_iter - explore > 0)) break;
            const int patience = phase == 0 ? explore : o.n_iter_without_progress;
            TsneStep step{phase == 0 ? 0.5f : 0.8f, o.learning_rate, upd.get(), gains.get()};
            const double exag = phase == 0 ? o.early_exaggeration : 1.0;
            GEMB_CUDA(cudaMemsetAsync(upd.get(), 0, sizeof(double) * 2 * n, st));
            GEMB_CUDA(cudaMemcpyAsync(gains.get(), ones.data(), sizeof(float) * 2 * n, cudaMemcpyHostToDevice, st));
            double best_error = 1.79769313486231570e308;
            int best_iter = it, i = it;
            for (i = it; i < stop; i++) {
                const bool check = (i + 1) % check_every == 0;
                const bool want_error = check || i == stop - 1;
                GEMB_TRY(tsne_gradient_dev(ctx, tb, dY.get(), dY2.get(), A.indptr.get(), A.cols.get(), A.val.get(), exag,
                                           (float)o.angle, want_error, nullptr, step, negf.get(), dS.get(), dS.get() + 1,
                                           &t_tree.t, &t_grad.t));
                std::swap(dY, dY2);
                if (want_error) {
                    double h[2];
                    GEMB_TRY(copy_sync(ctx, h, dS.get() + 1, sizeof(h), cudaMemcpyDeviceToHost));
                    error = h[0];
                    if (check) {
                        if (error < best_error) { best_error = error; best_iter = i; }
                        else if (i - best_iter > patience) break;
                        if (std::sqrt(h[1]) <= o.min_grad_norm) break;
                    }
                }
            }
            it_done = std::min(i, stop - 1);
            it = it_done + 1;
        }
        S.tree_ms = t_tree.t.total_ms();
        S.grad_ms = t_grad.t.total_ms();
    }
    GEMB_TRY(copy_sync(ctx, Y_out, dY.get(), sizeof(float) * 2 * n, cudaMemcpyDeviceToHost));
    S.opt_ms = ms_since(t0);
    S.total_ms = ms_since(t_all);
    S.n_iter = it_done;
    S.kl_divergence = error;
    if (stats) {
        S.struct_size = stats->struct_size;
        *stats = S;
    }
    return GEMB_OK;
}
