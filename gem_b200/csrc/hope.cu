// gem_b200/csrc/hope.cu -- HOPE: top-k SVD of the Katz proximity S = (I - beta A)^-1 beta A without
// ever forming S (replaces hope.py:29-36 and scipy svds, _svds.py:432-535).
//
// Two solvers behind gemb_hope():
//
//  GENERAL (any A; algorithm = 1): block subspace iteration with Rayleigh-Ritz on S^T S, the block
//  form of what ARPACK does for svds (SURVEY Appendix B).  S.x and S^T.x are Katz/Horner sweeps of
//  the CSR SpMM:
//     V <- orth(randn(n, b))                                   b = k + oversample
//     repeat
//         U  = S V                       J SpMM sweeps
//         T  = U^T U ;  (theta, Z) = eigh(T)                   Ritz values theta = sigma^2
//         stop_rule 0: stop if every top-k sigma moved by <= tol relative  (or max_iters)
//         U <- U Z Theta^-1/2 (orthonormal Ritz vectors);  W = S^T U
//         stop_rule 1: stop if max_j ||S^T u_j - sigma_j v_j|| = sqrt((W^T W)_jj - theta_j) <= tol * sigma_max
//         V <- CholQR2(W)
//     sigma = sqrt(theta) ascending over the top k;  X = [ U Z_k theta^-1/4 | V Z_k theta^1/4 ]
//
//  SYMMETRIC (A = A^T, which gemb_graph_upload knows; algorithm = 2, the default for symmetric
//  shards): S = f(A) with f(l) = beta l / (1 - beta l) shares A's eigenvectors, so the singular
//  triplets of S are (|f(l_i)|, sign(f(l_i)) v_i, v_i).  The invariant subspace is found by
//  Chebyshev-filtered subspace iteration on A itself -- one SpMM per polynomial degree instead of J
//  per operator application -- with the damped interval set each round to {l : |f(l)| < tau}, tau the
//  smallest |f| among the block's Ritz values:
//     V <- CholQR2(randn)
//     repeat
//         W = A V;  T = V^T W;  (l, Z) = eigh(T)               Rayleigh-Ritz on A
//         theta_i = f(l_i)^2, ranked;  stop on the same test as above
//         F = W (first 3 rounds: power step) or p_m(A) V       scaled three-term recurrence, fused SpMM epilogue
//         V <- orth(F) by CholeskyQR2 on the Ritz-rotated block F Z (well conditioned for any filter gain)
//     X = [ V Z_k sign(f) sqrt(sigma) | V Z_k sqrt(sigma) ]
//
// Multi-GPU: rows are sharded; each SpMM is preceded by an all-gather of the block's row shards
// and each Gram matrix is all-reduced (b x b fp64).
#include "common.cuh"
#include <chrono>
#include "nccl_api.h"
#include <math.h>
#include <string.h>
#include <algorithm>
#include <numeric>

namespace gemb {

struct HopeWork {
    gemb_graph *g;
    gemb_ctx *c;
    int b;
    int64_t rows;    // n_local
    int64_t shard;   // n_shard (buffer rows)
    float *buf[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // n_shard x b each: own_buf[], or g->halo.buf[] in halo mode
    DeviceBuffer<float> own_buf[5];
    DeviceBuffer<float> full;   // n_pad x b (multi-GPU all-gather target)
    DeviceBuffer<double> G, G2, w, Z, Zs, scal;
    DeviceBuffer<float> Minv, M1, M2;
    DeviceBuffer<int> rank_dev;
    CallEvents<2> fork_join;    // c->stream -> c->side and back (ritz_eigh)
    int64_t spmm_wide = 0, spmm_all = 0;
    int mode = 0;               // opts.spectral_mode
    DeviceBuffer<float> opT;    // spectral_mode 2: T = X - A X between the two sweeps of one application (n x b)
    DeviceBuffer<float> rscale; // spectral_mode 4: D_ii = 1 / (rowsum(A) + rowsum(A^T)), 0 for isolated rows (n floats)
    bool halo = false;       // multi-GPU: needed-rows-only exchange over peer memory (halo.cu); buf[] = g->halo.buf[]
    int64_t pushes = 0;      // blocks whose rows were pushed to the peers
    double push_bytes_per_row = 0.0;   // sum over the pushed blocks of (bytes per pushed row): NVLink bytes out = this * push_rows
    int buf_index(const float *p) const { for (int i = 0; i < 5; i++) if (buf[i] == p) return i; return -1; }
    // the five work blocks of `count` floats each, zero-filled (padded rows stay 0)
    int alloc_blocks(size_t count) {
        for (int i = 0; i < 5; i++) {
            GEMB_CUDA(own_buf[i].alloc(count));
            buf[i] = own_buf[i].get();
            GEMB_CUDA(cudaMemsetAsync(buf[i], 0, sizeof(float) * count, c->stream));
        }
        return GEMB_OK;
    }
};

struct HopeResult {
    int iters = 0, converged = 0, katz_terms = 0, algorithm = 0;
    double change = 0.0;
    float resid_max = -1.f, resid_est = -1.f;
    float *Xd = nullptr;       // device n_local x d (points into a work buffer or Xalloc)
    DeviceBuffer<float> Xalloc;
    float *sig_dev = nullptr;  // k floats
    double sigma_max = 0.0;
    double norm = 0.0;         // symmetric solvers: the spectrum bound the map ended with (SpecMap::norm)
};

// host <-> device staging: the copy, then a stream synchronise (the host reads the result, or its buffer goes out of scope)
static int copy_sync(gemb_ctx *c, void *dst, const void *src, size_t bytes, cudaMemcpyKind kind) {
    GEMB_CUDA(cudaMemcpyAsync(dst, src, bytes, kind, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

// the width-4 probes (norm estimate, Katz series probe) leave their vectors in work blocks 2..4: zero them again, as
// alloc_blocks left them
static int clear_scratch(HopeWork &W) {
    for (int i = 2; i < 5; i++) GEMB_CUDA(cudaMemsetAsync(W.buf[i], 0, sizeof(float) * (size_t)W.shard * W.b, W.c->stream));
    return GEMB_OK;
}

// X goes into work block `blk` when it fits (d <= b; blk = nullptr: never), else into its own n_local x d allocation;
// sigma goes into G2, free once the solver's iterations end
static int place_output(HopeWork &W, HopeResult &R, float *blk, int d) {
    R.Xd = blk;
    if (!blk || (size_t)d > (size_t)W.b) {
        GEMB_CUDA(R.Xalloc.alloc((size_t)std::max<int64_t>(W.rows, 1) * d));
        R.Xd = R.Xalloc.get();
    }
    R.sig_dev = (float *)W.G2.get();
    return GEMB_OK;
}

static int comm_allgather(HopeWork &W, const float *shard_src, int width) {
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    GEMB_TRY(W.c->t_comm.begin(W.c->stream));
    ncclResult_t r = api->AllGather(shard_src, W.full.get(), (size_t)W.shard * width, ncclFloat,
                                    (ncclComm_t)W.c->comm, W.c->stream);
    if (r != ncclSuccess) { set_error("ncclAllGather: %s", api->GetErrorString(r)); return GEMB_ERR_NCCL; }
    GEMB_TRY(W.c->t_comm.end(W.c->stream));
    return GEMB_OK;
}

static int comm_allreduce_f64(HopeWork &W, double *buf, size_t count) {
    if (W.c->nranks == 1) return GEMB_OK;
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    GEMB_TRY(W.c->t_comm.begin(W.c->stream));
    ncclResult_t r = api->AllReduce(buf, buf, count, ncclDouble, ncclSum, (ncclComm_t)W.c->comm, W.c->stream);
    if (r != ncclSuccess) { set_error("ncclAllReduce: %s", api->GetErrorString(r)); return GEMB_ERR_NCCL; }
    GEMB_TRY(W.c->t_comm.end(W.c->stream));
    return GEMB_OK;
}

// halo mode: ends the push of a width-wide block to the peers -- launching it first as a stand-alone push of work block
// `push_bi` when >= 0 -- with the sweep barrier (timed as communication), and counts it
static int end_push(HopeWork &W, int width, int push_bi = -1) {
    GEMB_TRY(W.c->t_comm.begin(W.c->stream));
    if (push_bi >= 0) GEMB_TRY(halo_push_launch(W.g, push_bi, width));
    GEMB_TRY(halo_barrier(W.g));
    GEMB_TRY(W.c->t_comm.end(W.c->stream));
    W.pushes++;
    W.push_bytes_per_row += 4.0 * width;
    return GEMB_OK;
}

// halo mode: the local rows of block `buf` go to the peers that reference them, then the sweep barrier
static int publish(HopeWork &W, const float *buf, int width) {
    if (!W.halo) return GEMB_OK;
    const int bi = W.buf_index(buf);
    GEMB_ARG(bi >= 0, "publish: not a work block");
    return end_push(W, width, bi);
}

// Y(shard) = alpha * op(A) * X + gamma * X(shard) + delta * X0(shard).  Sharded: halo mode gathers from the block's own
// [local | halo] rows and (push_out) stores Y's rows into the peers' halo slots from the epilogue; otherwise X is
// all-gathered first.
static int dist_spmm3(HopeWork &W, bool transpose, int width, float alpha, const float *Xshard, float gamma,
                      bool use_self, float delta, const float *X0, float *Y, bool timed, bool push_out = false) {
    if (W.halo) {
        gemb_csr_dev A = W.g->A;
        A.indices = W.g->halo.indices_ext;
        HaloPushArgs P;
        const int bo = W.buf_index(Y), bin = W.buf_index(Xshard);
        GEMB_ARG(bin >= 0, "spmm input is not a work block");
        if (push_out) { GEMB_ARG(bo >= 0, "spmm output is not a work block"); halo_push_args(W.g, bo, &P); }
        if (timed) GEMB_TRY(W.c->t_spmm.begin(W.c->stream));
        GEMB_TRY(spmm3_launch(W.c, A, W.rows, width, alpha, Xshard, gamma, use_self ? Xshard : nullptr, delta, X0, Y,
                              push_out ? &P : nullptr));
        if (timed) { GEMB_TRY(W.c->t_spmm.end(W.c->stream)); W.spmm_wide++; }
        W.spmm_all++;
        if (push_out) return end_push(W, width);
        return GEMB_OK;
    }
    const float *Xfull = Xshard;
    if (W.c->nranks > 1) {
        GEMB_TRY(comm_allgather(W, Xshard, width));
        Xfull = W.full.get();
    }
    if (timed) GEMB_TRY(W.c->t_spmm.begin(W.c->stream));
    GEMB_TRY(spmm3_launch(W.c, transpose ? W.g->AT : W.g->A, W.rows, width, alpha, Xfull, gamma,
                          use_self ? Xshard : nullptr, delta, X0, Y));
    if (timed) { GEMB_TRY(W.c->t_spmm.end(W.c->stream)); W.spmm_wide++; }
    W.spmm_all++;
    return GEMB_OK;
}

static int dist_spmm(HopeWork &W, bool transpose, int width, float alpha, const float *Xshard,
                     const float *X0, float *Y, bool timed) {
    return dist_spmm3(W, transpose, width, alpha, Xshard, 0.f, false, 1.f, X0, Y, timed);
}

// One application of the symmetric solver's operator Op:  Y = alpha * Op X + gamma * X (use_self) + delta * X0.
// spectral_modes 0 and 1: Op = A, one sweep (dist_spmm3 as it stands).  spectral_mode 2 (single GPU): the composite
// Op = -M^T M with M = I - A, uploaded as A and A^T and never formed -- sweep 1 T = X - A X, sweep 2
// Y = alpha A^T T - alpha T + gamma X + delta X0, whose epilogue takes four rows (spmm4_launch).  One application
// counts as two sweeps.
static int op_apply(HopeWork &W, int width, float alpha, const float *X, float gamma, bool use_self, float delta,
                    const float *X0, float *Y, bool timed, bool push_out = false) {
    if (W.mode != 2) return dist_spmm3(W, false, width, alpha, X, gamma, use_self, delta, X0, Y, timed, push_out);
    gemb_ctx *c = W.c;
    float *T = W.opT.get();
    if (timed) GEMB_TRY(c->t_spmm.begin(c->stream));
    GEMB_TRY(spmm3_launch(c, W.g->A, W.rows, width, -1.f, X, 1.f, X, 0.f, nullptr, T));
    GEMB_TRY(spmm4_launch(c, W.g->AT, W.rows, width, alpha, T, -alpha, T, gamma, use_self ? X : nullptr, delta, X0, Y));
    if (timed) { GEMB_TRY(c->t_spmm.end(c->stream)); W.spmm_wide += 2; }
    W.spmm_all += 2;
    return GEMB_OK;
}

// out = sum_{j=1..J} (beta op(A))^j in   (Horner: W_m = in + beta op(A) W_{m-1}); t1,t2 scratch.
// spectral_mode 5 (rooted PageRank, beta = alpha, A = P): out = (1 - alpha) sum_{j=0..J} (alpha op(P))^j in -- the same
// loop, with the j = 0 term and the factor (1 - alpha) folded into the last sweep's epilogue:
// out = alpha (1 - alpha) op(P) W_{J-1} + (1 - alpha) in.
static int katz(HopeWork &W, bool transpose, float beta, int J, const float *in, float *out,
                float *t1, float *t2) {
    const float *cur = in;
    for (int m = 1; m <= J; m++) {
        if (m < J) {
            float *dst = (m & 1) ? t1 : t2;   // halo mode: `in` was published by the caller, dst feeds the next sweep
            GEMB_TRY(dist_spmm3(W, transpose, W.b, beta, cur, 0.f, false, 1.f, in, dst, true, W.halo));
            cur = dst;
        } else if (W.mode == 5) {
            const double a = beta;
            GEMB_TRY(dist_spmm3(W, transpose, W.b, (float)(a * (1.0 - a)), cur, 0.f, false, (float)(1.0 - a), in, out, true));
        } else {
            GEMB_TRY(dist_spmm(W, transpose, W.b, beta, cur, nullptr, out, true));
        }
    }
    return GEMB_OK;
}

// out = S in, or S^T in (transpose), for the proximity of the general solver (W.mode): Katz (0) and rooted PageRank (5)
// by katz(); common neighbours (3) S = A A and Adamic-Adar (4) S = A D A by two sweeps, t1 = D op(A) in (D = I for mode
// 3; the scale is applied in sweep 1's epilogue), then out = op(A) t1 -- S^T = A^T D A^T takes A^T in both.  Single GPU
// for modes 3 and 4; one application counts as two sweeps.
static int apply_S(HopeWork &W, bool transpose, float beta, int J, const float *in, float *out, float *t1, float *t2) {
    if (W.mode != 3 && W.mode != 4) return katz(W, transpose, beta, J, in, out, t1, t2);
    gemb_ctx *c = W.c;
    const gemb_csr_dev &Op = transpose ? W.g->AT : W.g->A;
    GEMB_TRY(c->t_spmm.begin(c->stream));
    if (W.mode == 4) GEMB_TRY(spmm_scaled_launch(c, Op, W.rows, W.b, 1.f, in, W.rscale.get(), t1));
    else GEMB_TRY(spmm_launch(c, Op, W.rows, W.b, 1.f, in, nullptr, t1));
    GEMB_TRY(spmm_launch(c, Op, W.rows, W.b, 1.f, t1, nullptr, out));
    GEMB_TRY(c->t_spmm.end(c->stream));
    W.spmm_wide += 2;
    W.spmm_all += 2;
    return GEMB_OK;
}

static int gram_full(HopeWork &W, const float *P, const float *Q, double *G) {
    GEMB_TRY(W.c->t_dense.begin(W.c->stream));
    GEMB_TRY(gram_launch(W.c, W.rows, P, W.b, Q, W.b, G));
    GEMB_TRY(W.c->t_dense.end(W.c->stream));
    GEMB_TRY(comm_allreduce_f64(W, G, (size_t)W.b * W.b));
    return GEMB_OK;
}

// one CholeskyQR pass: dst = src * R^-1 with R^T R = G (G destroyed). G must hold src^T src.
static int cholqr_pass(HopeWork &W, double *G, const float *src, float *dst) {
    GEMB_TRY(W.c->t_dense.begin(W.c->stream));
    GEMB_TRY(chol_inverse_launch(W.c, W.b, G, W.Minv.get(), W.rank_dev.get()));
    GEMB_TRY(apply_launch(W.c, W.rows, src, W.b, W.Minv.get(), W.b, W.b, dst, W.b));
    GEMB_TRY(W.c->t_dense.end(W.c->stream));
    return GEMB_OK;
}

// dst = orth(src) by CholeskyQR2; tmp is scratch; src, tmp, dst pairwise distinct
static int cholqr2(HopeWork &W, const float *src, float *tmp, float *dst) {
    GEMB_TRY(gram_full(W, src, src, W.G.get()));
    GEMB_TRY(cholqr_pass(W, W.G.get(), src, tmp));
    GEMB_TRY(gram_full(W, tmp, tmp, W.G.get()));
    GEMB_TRY(cholqr_pass(W, W.G.get(), tmp, dst));
    return GEMB_OK;
}

// M1[i][j] = Z[i][b-k+j] * theta_j^(p1),  M2 likewise with p2   (theta ascending, top k)
__global__ void ritz_maps_kernel(int b, int k, const double *__restrict__ w, const double *__restrict__ Z,
                                 float *__restrict__ M1, float *__restrict__ M2, double p1, double p2,
                                 double rel_floor = 1e-28) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= b * k) return;
    const int i = idx / k, j = idx - i * k;
    const double wmax = w[b - 1];
    const double th = w[b - k + j];
    const double z = Z[(size_t)i * b + (b - k + j)];
    double a = 0.0, c = 0.0;
    if (th > rel_floor * wmax && th > 0.0) { a = z * pow(th, p1); c = z * pow(th, p2); }
    M1[idx] = (float)a;
    M2[idx] = (float)c;
}

__global__ void sqrt_top_kernel(int b, int k, const double *__restrict__ w, float *__restrict__ sigma) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < k) { const double th = w[b - k + j]; sigma[j] = (float)(th > 0.0 ? sqrt(th) : 0.0); }
}

// column sums of squares of (A - B): out[j] (fp64), n x b row-major
__global__ void coldiff_sumsq_kernel(int64_t n, int b, const float *__restrict__ A, const float *__restrict__ B,
                                     double *__restrict__ out) {
    const int j = threadIdx.x % b;  // blockDim.x is a multiple of b
    const int rpb = blockDim.x / b;
    double acc = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * rpb + threadIdx.x / b; r < n; r += (int64_t)gridDim.x * rpb) {
        const double d = (double)A[r * b + j] - (double)B[r * b + j];
        acc += d * d;
    }
    atomicAdd(out + j, acc);
}

// q[col] = z^T H z for every column z of Z (b x b, row-major), H = (AV)^T (AV): the squared norm of A V z, from which
// the stop rule takes the residual of the Ritz pair.  One CTA per column; the sums run in index order with separately
// rounded products (t = sum_s H[r][s] Z[s][col], then q = sum_r Z[r][col] t), so the value does not depend on the
// launch shape.  Dynamic shared memory: b doubles.
__global__ void ritz_quadform_kernel(int b, const double *__restrict__ H, const double *__restrict__ Z,
                                     double *__restrict__ q) {
    extern __shared__ double s_term[];
    const int col = blockIdx.x;
    for (int r = threadIdx.x; r < b; r += blockDim.x) {
        double t = 0.0;
        for (int s = 0; s < b; s++) t = __dadd_rn(t, __dmul_rn(H[(size_t)r * b + s], Z[(size_t)s * b + col]));
        s_term[r] = __dmul_rn(Z[(size_t)r * b + col], t);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double acc = 0.0;
        for (int r = 0; r < b; r++) acc = __dadd_rn(acc, s_term[r]);
        q[col] = acc;
    }
}

// Y = a * P + c * Q
__global__ void axpby_kernel(int64_t count, float a, const float4 *__restrict__ P, float c,
                             const float4 *__restrict__ Q, float4 *__restrict__ Y) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const float4 p = P[i], q = Q[i];
        Y[i] = make_float4(a * p.x + c * q.x, a * p.y + c * q.y, a * p.z + c * q.z, a * p.w + c * q.w);
    }
}

// the same, one thread group per row, storing the row into the peers' halo slots as well (halo mode)
__global__ void __launch_bounds__(256)
axpby_push_kernel(int64_t n_rows, int G, int rows_per_cta, float a, const float4 *__restrict__ P, float c,
                  const float4 *__restrict__ Q, float4 *__restrict__ Y, HaloPushArgs H) {
    const int lr = threadIdx.x / G, cc = threadIdx.x - lr * G;
    if (lr >= rows_per_cta) return;
    const int64_t row = (int64_t)blockIdx.x * rows_per_cta + lr;
    if (row >= n_rows) return;
    const float4 p = P[row * G + cc], q = Q[row * G + cc];
    const float4 v = make_float4(a * p.x + c * q.x, a * p.y + c * q.y, a * p.z + c * q.z, a * p.w + c * q.w);
    Y[row * G + cc] = v;
    halo_push_row(H, row, G, cc, v);
}

static int axpby_launch(HopeWork &W, float a, const float *P, float c, const float *Q, float *Y) {
    const int64_t count = W.rows * (int64_t)W.b / 4;
    if (W.halo) {        // Y feeds the next SpMM: its rows go to the peers from here
        const int G = W.b / 4, rpc = 256 / G, bo = W.buf_index(Y);
        GEMB_ARG(bo >= 0 && G <= 256, "axpby output is not a work block");
        HaloPushArgs H;
        halo_push_args(W.g, bo, &H);
        if (W.rows > 0) {
            axpby_push_kernel<<<(unsigned)((W.rows + rpc - 1) / rpc), 256, 0, W.c->stream>>>(
                W.rows, G, rpc, a, (const float4 *)P, c, (const float4 *)Q, (float4 *)Y, H);
            GEMB_CUDA(cudaGetLastError());
            count_launch();
        }
        return end_push(W, W.b);
    }
    if (count == 0) return GEMB_OK;
    int grid = W.c->sm_count * 8;
    if ((int64_t)grid * 256 > count) grid = (int)((count + 255) / 256);
    axpby_kernel<<<grid, 256, 0, W.c->stream>>>(count, a, (const float4 *)P, c, (const float4 *)Q, (float4 *)Y);
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    return GEMB_OK;
}

// out[0] = max_i sum_j |a_ij| (= ||A||_inf), out[1] = max(0, -min_ij a_ij)  (0 <=> all weights >= 0)
__global__ void csr_rowsum_kernel(int64_t n, const int32_t *__restrict__ indptr, const float *__restrict__ vals,
                                  double *__restrict__ out) {
    double mx = 0.0, neg = 0.0;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        const int s = indptr[r], e = indptr[r + 1];
        double acc = 0.0;
        if (vals) {
            for (int i = s; i < e; i++) { const double v = vals[i]; acc += fabs(v); if (-v > neg) neg = -v; }
        } else acc = (double)(e - s);
        if (acc > mx) mx = acc;
    }
    for (int o = 16; o > 0; o >>= 1) {
        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        neg = fmax(neg, __shfl_xor_sync(0xffffffffu, neg, o));
    }
    if ((threadIdx.x & 31) == 0) {   // non-negative doubles order like their bit patterns
        atomicMax((unsigned long long *)out, (unsigned long long)__double_as_longlong(mx));
        atomicMax((unsigned long long *)(out + 1), (unsigned long long)__double_as_longlong(neg));
    }
}

// s_i = 1 / (sum_j A_ij + sum_j AT_ij) accumulated in fp64, stored fp32; 0 where the sum is 0 (an isolated row).  AT is
// the transpose's CSR, or A itself for a symmetric upload (then s_i = 1 / (2 rowsum_i(A))).
__global__ void inv_degree_kernel(int64_t n, const int32_t *__restrict__ ip, const float *__restrict__ v,
                                  const int32_t *__restrict__ ipt, const float *__restrict__ vt, float *__restrict__ s) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        double acc = 0.0;
        if (v) { for (int i = ip[r]; i < ip[r + 1]; i++) acc += (double)v[i]; } else acc += (double)(ip[r + 1] - ip[r]);
        if (vt) { for (int i = ipt[r]; i < ipt[r + 1]; i++) acc += (double)vt[i]; } else acc += (double)(ipt[r + 1] - ipt[r]);
        s[r] = acc > 0.0 ? (float)(1.0 / acc) : 0.f;
    }
}

static int inv_degree(HopeWork &W) {
    gemb_ctx *c = W.c;
    GEMB_CUDA(W.rscale.alloc((size_t)std::max<int64_t>(W.rows, 1)));
    if (W.rows == 0) return GEMB_OK;
    const int grid = (int)std::min<int64_t>((W.rows + 255) / 256, (int64_t)c->sm_count * 8);
    inv_degree_kernel<<<grid, 256, 0, c->stream>>>(W.rows, W.g->A.indptr, W.g->A.data, W.g->AT.indptr, W.g->AT.data,
                                                   W.rscale.get());
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    return GEMB_OK;
}

static int comm_allreduce_max_f64(HopeWork &W, double *buf, size_t count) {
    if (W.c->nranks == 1) return GEMB_OK;
    NcclApi *api = nccl_api();
    if (!api) return GEMB_ERR_NCCL;
    ncclResult_t r = api->AllReduce(buf, buf, count, ncclDouble, ncclMax, (ncclComm_t)W.c->comm, W.c->stream);
    if (r != ncclSuccess) { set_error("ncclAllReduce(max): %s", api->GetErrorString(r)); return GEMB_ERR_NCCL; }
    return GEMB_OK;
}

// ||A||_inf and the sign of the weights in one pass over the CSR shard
static int rowsum_bound(HopeWork &W, double *norm_inf, bool *nonneg) {
    gemb_ctx *c = W.c;
    GEMB_CUDA(cudaMemsetAsync(W.scal.get(), 0, 2 * sizeof(double), c->stream));
    if (W.rows > 0) {
        csr_rowsum_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(W.rows, W.g->A.indptr, W.g->A.data, W.scal.get());
        GEMB_CUDA(cudaGetLastError());
        count_launch();
    }
    GEMB_TRY(comm_allreduce_max_f64(W, W.scal.get(), 2));
    double h[2];
    GEMB_TRY(copy_sync(c, h, W.scal.get(), sizeof h, cudaMemcpyDeviceToHost));
    *norm_inf = h[0];
    *nonneg = (h[1] == 0.0);
    return GEMB_OK;
}

// ||A||_2 by power iteration on A^T A with a 4-column block
static int estimate_norm2(HopeWork &W, uint64_t seed, float *x, float *y, float *z, double *out) {
    gemb_ctx *c = W.c;
    gemb_graph *g = W.g;
    const int pw = 4;
    GEMB_TRY(randn_launch(c, W.rows, pw, seed ^ 0x5bd1e995u, (uint64_t)g->row0, x));
    double est = 0.0, prev = -1.0;
    for (int it = 0; it < 16; it++) {
        double h[2];
        GEMB_TRY(sumsq_launch(c, W.rows * pw, x, W.scal.get()));
        GEMB_TRY(publish(W, x, pw));
        GEMB_TRY(dist_spmm3(W, false, pw, 1.f, x, 0.f, false, 1.f, nullptr, y, false, true));
        GEMB_TRY(dist_spmm(W, true, pw, 1.f, y, nullptr, z, false));
        GEMB_TRY(sumsq_launch(c, W.rows * pw, z, W.scal.get() + 1));
        GEMB_TRY(comm_allreduce_f64(W, W.scal.get(), 2));
        GEMB_TRY(copy_sync(c, h, W.scal.get(), sizeof h, cudaMemcpyDeviceToHost));
        if (!(h[0] > 0.0) || !(h[1] > 0.0)) { est = 0.0; break; }  // A^T A x = 0 (empty graph)
        est = sqrt(sqrt(h[1] / h[0]));   // ||A^T A x|| / ||x|| -> sigma_max^2
        GEMB_TRY(scale_launch(c, W.rows * pw, (float)(1.0 / sqrt(h[1])), z));
        std::swap(x, z);
        if (prev > 0 && fabs(est - prev) <= 1e-3 * est && it >= 3) break;
        prev = est;
    }
    *out = est;
    return GEMB_OK;
}

// spectral_mode 2: ||M||_2^2 = ||M^T M||_2 by power iteration on the composite operator with a 4-column block.  From
// below, like estimate_norm2: hope_symmetric raises it to the largest |Ritz value| (SpecMap::observe).
static int estimate_composite_norm(HopeWork &W, uint64_t seed, float *x, float *y, double *out) {
    gemb_ctx *c = W.c;
    const int pw = 4;
    GEMB_TRY(randn_launch(c, W.rows, pw, seed ^ 0x5bd1e995u, (uint64_t)W.g->row0, x));
    double est = 0.0, prev = -1.0;
    for (int it = 0; it < 32; it++) {
        double h[2];
        GEMB_TRY(sumsq_launch(c, W.rows * pw, x, W.scal.get()));
        GEMB_TRY(op_apply(W, pw, 1.f, x, 0.f, false, 1.f, nullptr, y, false));
        GEMB_TRY(sumsq_launch(c, W.rows * pw, y, W.scal.get() + 1));
        GEMB_TRY(copy_sync(c, h, W.scal.get(), sizeof h, cudaMemcpyDeviceToHost));
        if (!(h[0] > 0.0) || !(h[1] > 0.0)) { est = 0.0; break; }   // M^T M x = 0 (M = 0: P = I)
        est = sqrt(h[1] / h[0]);                                      // ||M^T M x|| / ||x|| -> ||M||_2^2
        GEMB_TRY(scale_launch(c, W.rows * pw, (float)(1.0 / sqrt(h[1])), y));
        std::swap(x, y);
        if (prev > 0 && fabs(est - prev) <= 1e-3 * est && it >= 3) break;
        prev = est;
    }
    *out = est;
    return GEMB_OK;
}

// beta * ||A||_2 >= 1 does not mean the Katz series diverges: it converges iff beta * rho(A) < 1, and a directed graph
// (a hub, a DAG: rho = 0) can have ||A||_2 far above rho(A).  Measure the series itself on a width-4 random probe:
// t_j = (beta op(A))^j t_0; J = first j with ||t_j|| <= katz_tol * max_i ||t_i|| (for A and A^T), plus a margin.
// Returns GEMB_ERR_DIVERGE when the terms do not decay (rho_est = last growth ratio / beta).
static int probe_katz_terms(HopeWork &W, float beta, double katz_tol, uint64_t seed, float *x, float *y, int *J_out,
                            double *rho_est) {
    gemb_ctx *c = W.c;
    const int pw = 4, Jmax = 2048;
    int Jbest = 1;
    *rho_est = 0.0;
    for (int tr = 0; tr < 2; tr++) {
        GEMB_TRY(randn_launch(c, W.rows, pw, seed ^ (0x7f4a7c15u + tr), (uint64_t)W.g->row0, x));
        double peak = 0.0, prev = 0.0;
        int j = 0;
        bool done = false;
        for (j = 1; j <= Jmax; j++) {
            double h = 0.0;
            GEMB_TRY(dist_spmm(W, tr == 1, pw, beta, x, nullptr, y, false));
            GEMB_TRY(sumsq_launch(c, W.rows * pw, y, W.scal.get()));
            GEMB_TRY(comm_allreduce_f64(W, W.scal.get(), 1));
            GEMB_TRY(copy_sync(c, &h, W.scal.get(), sizeof h, cudaMemcpyDeviceToHost));
            const double nt = sqrt(h);
            if (prev > 0.0) *rho_est = std::max(*rho_est * (j > 8 ? 0.0 : 1.0), nt / prev / (double)beta);
            if (!(nt < 1e30)) break;
            peak = std::max(peak, nt);
            if (nt <= katz_tol * peak) { done = true; break; }
            prev = nt;
            std::swap(x, y);
        }
        if (!done) return GEMB_ERR_DIVERGE;
        Jbest = std::max(Jbest, j);
    }
    *J_out = std::min(4096, Jbest + Jbest / 8 + 2);
    return GEMB_OK;
}

struct Opts {
    int oversample = 16, max_iters = 30, min_iters = 2, katz_terms = 0, compute_residual = 0, verbose = 0;
    int algorithm = 0, cheb_degree = 8, stop_rule = 0, lanczos_basis = 0;
    int spectral_mode = 0;   // 0: top-k singular triplets of the Katz operator (HOPE); 1: the d largest ALGEBRAIC eigenpairs of the
                             // uploaded symmetric matrix itself (Laplacian Eigenmaps: D^-1/2 A D^-1/2, lap.py:26-32);
                             // 2: those of the composite -M^T M, M = I - A (LLE: A = D^-1 W, uploaded with A^T);
                             // 3, 4, 5: HOPE on the common-neighbour, Adamic-Adar and rooted-PageRank proximities (apply_S)
    float tol = 1e-6f, katz_tol = 1e-7f, range_log2 = 8.f;
    uint64_t seed = 1234;
};

static int katz_terms_for(double beta, double nrm, double katz_tol) {
    const double x1 = beta * nrm * 1.02;
    if (x1 <= 1e-30) return 1;
    int J = (int)ceil(log(katz_tol) / log(x1));
    return std::max(1, std::min(J, 4096));
}

// The Katz terms J of S = sum_{j=1..J} (beta A)^j for the general solver and the 'SVD error' diagnostic: ||A||_2 by
// power iteration; beta ||A||_2 * 1.02 < 1 bounds the terms a priori (katz_terms_for).  Above that bound the series
// still converges when beta rho(A) < 1, and rho(A) of a directed graph can lie far below ||A||_2 (a DAG: rho = 0), so
// probe_katz_terms measures the decay of the terms; GEMB_ERR_DIVERGE only when they do not decay.  probe = false
// (symmetric A, where ||A||_2 = rho(A); the halo exchange) refuses at the bound.  Leaves work blocks 2..4 dirty.
static int general_katz_terms(HopeWork &W, float beta, double katz_tol, uint64_t seed, bool probe, double *nrm_out,
                              int *J_out) {
    double nrm = 0.0;
    GEMB_TRY(estimate_norm2(W, seed, W.buf[3], W.buf[4], W.buf[2], &nrm));
    *nrm_out = nrm;
    if ((double)beta * nrm * 1.02 < 1.0) {
        *J_out = katz_terms_for(beta, nrm, katz_tol);
        return GEMB_OK;
    }
    double rho = nrm;
    int s = GEMB_ERR_DIVERGE;
    if (probe) {
        s = probe_katz_terms(W, beta, katz_tol, seed, W.buf[3], W.buf[4], J_out, &rho);
        if (s != GEMB_OK && s != GEMB_ERR_DIVERGE) return s;
    }
    if (s != GEMB_OK)
        set_error("beta * rho(A) ~ %.4g >= 1 (||A||_2 = %.4g): the Katz series (I - beta A)^-1 beta A does not "
                  "converge; choose beta < %.4g", (double)beta * rho, nrm, 1.0 / std::max(rho, 1e-300));
    return s;
}

// max over `cols` of || S^T P_j - Qs_j || / smax ;  scr0..2 are scratch blocks
static int residual_check(HopeWork &W, float beta, int J, const float *P, const float *Qs, float *scr0, float *scr1,
                          float *scr2, const std::vector<int> &cols, double smax, float *out) {
    gemb_ctx *c = W.c;
    const int b = W.b;
    GEMB_TRY(apply_S(W, true, beta, J, P, scr0, scr1, scr2));    // scr0 = S^T P
    GEMB_CUDA(cudaMemsetAsync(W.scal.get(), 0, sizeof(double) * b, c->stream));
    const int threads = (256 / b) * b > 0 ? (256 / b) * b : b;
    coldiff_sumsq_kernel<<<c->sm_count * 4, threads, 0, c->stream>>>(W.rows, b, scr0, Qs, W.scal.get());
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    GEMB_TRY(comm_allreduce_f64(W, W.scal.get(), b));
    std::vector<double> rs(b);
    GEMB_TRY(copy_sync(c, rs.data(), W.scal.get(), sizeof(double) * b, cudaMemcpyDeviceToHost));
    double rm = 0.0;
    for (int j : cols) rm = std::max(rm, sqrt(rs[j]) / std::max(smax, 1e-300));
    *out = (float)rm;
    return GEMB_OK;
}

// Rayleigh-Ritz eigen step: (W.w, W.Z) = eigh(W.G2) (G2 destroyed; `symmetrize`: eigh of (G2 + G2^T) / 2), the
// eigenvalues (ascending) read back into lam[0..b).  Given AV (the residual stop rule), lam[b..2b) receives z^T H z of
// every Ritz vector z, H = (AV)^T (AV), in the same copy: one host round trip per step.  H does not depend on the
// eigen-decomposition, and the Jacobi is one CTA: the Gram launch runs on c->side while the Jacobi has the other SMs to
// spare (the Jacobi is launched first so that it is not queued behind the Gram's one-CTA-per-SM grid).  The Gram's
// partial sums are added in a fixed order, so H is the same whenever it runs; the all-reduce stays on c->stream.
// Jacobi accuracy follows the requested tolerance (Z only pre-rotates the CholeskyQR and forms the Ritz vectors:
// an off-diagonal remainder of 1e-2 tol is invisible at tol; one sweep less per round at the bench setting)
static int ritz_eigh(HopeWork &W, float tol, bool symmetrize, std::vector<double> &lam, const float *AV = nullptr) {
    gemb_ctx *c = W.c;
    const int b = W.b;
    GEMB_TRY(c->t_dense.begin(c->stream));
    if (AV) GEMB_CUDA(cudaEventRecord(W.fork_join[0], c->stream));   // AV and the reduction scratch are free from here
    GEMB_TRY(eigh_launch(c, b, W.G2.get(), W.w.get(), W.Z.get(), W.Zs.get(), std::min(1e-5, std::max(1e-13, 1e-2 * (double)tol)),
                         symmetrize));
    if (AV) {
        GEMB_CUDA(cudaStreamWaitEvent(c->side, W.fork_join[0], 0));
        std::swap(c->stream, c->side);                               // the launchers take their stream from the context
        const int s = gram_launch(c, W.rows, AV, b, AV, b, W.G.get());
        std::swap(c->stream, c->side);
        GEMB_TRY(s);
        GEMB_CUDA(cudaEventRecord(W.fork_join[1], c->side));
        GEMB_CUDA(cudaStreamWaitEvent(c->stream, W.fork_join[1], 0));
        GEMB_TRY(comm_allreduce_f64(W, W.G.get(), (size_t)b * b));
        ritz_quadform_kernel<<<b, 128, sizeof(double) * b, c->stream>>>(b, W.G.get(), W.Z.get(), W.w.get() + b);
        GEMB_CUDA(cudaGetLastError());
        count_launch();
    }
    GEMB_TRY(c->t_dense.end(c->stream));
    return copy_sync(c, lam.data(), W.w.get(), sizeof(double) * (AV ? 2 * b : b), cudaMemcpyDeviceToHost);
}

// stop measure: per-value relative change of the k SINGULAR values (theta = sigma^2) since the last round, floored at
// 1e-3 sigma_max (tmax = sigma_max^2): a change measured against sigma_max alone never resolves the small end of a skewed
// spectrum (R-MAT: sigma_k ~ 1e-2 sigma_max)
static double sigma_change(const double *theta, const double *theta_prev, int k, double tmax) {
    double change = 0.0;
    for (int j = 0; j < k; j++) {
        const double sj = sqrt(std::max(theta[j], 0.0)), sp = sqrt(std::max(theta_prev[j], 0.0));
        change = std::max(change, fabs(sj - sp) / std::max(sj, 1e-3 * sqrt(tmax)));
    }
    return change;
}

// the same measure on signed values s (spectral_mode 1: the eigenvalues themselves), floored at 1e-3 smax, smax = max |s_j|
static double value_change(const double *s, const double *s_prev, int k, double smax) {
    double change = 0.0;
    for (int j = 0; j < k; j++) change = std::max(change, fabs(s[j] - s_prev[j]) / std::max(fabs(s[j]), 1e-3 * smax));
    return change;
}

// ------------------------------------------------------------------------------------ general solver
static int hope_general(HopeWork &W, const Opts &o, int d, float beta, int J, HopeResult &R) {
    gemb_ctx *c = W.c;
    const int b = W.b, k = d / 2;
    float *V = W.buf[0], *U = W.buf[1], *Wk = W.buf[2], *T1 = W.buf[3], *T2 = W.buf[4];
    R.algorithm = 1;
    R.katz_terms = J;
    GEMB_TRY(randn_launch(c, W.rows, b, o.seed, (uint64_t)W.g->row0, T1));
    GEMB_TRY(cholqr2(W, T1, T2, V));

    // stop_rule 1 tests the round's residual after the S^T sweep, and extraction then needs this round's U: the sweep
    // takes its Horner scratch from a block of its own instead of U
    DeviceBuffer<float> Hs;
    float *Hscr = U;
    if (o.stop_rule == 1) {
        GEMB_CUDA(Hs.alloc((size_t)W.shard * b));
        GEMB_CUDA(cudaMemsetAsync(Hs.get(), 0, sizeof(float) * (size_t)W.shard * b, c->stream));
        Hscr = Hs.get();
    }
    std::vector<double> theta(b), theta_prev(b, 0.0), wdiag(b);
    for (int it = 1; it <= o.max_iters; it++) {
        R.iters = it;
        GEMB_TRY(apply_S(W, false, beta, J, V, U, T1, T2));           // U = S V
        GEMB_TRY(gram_full(W, U, U, W.G.get()));                            // T = U^T U
        GEMB_CUDA(cudaMemcpyAsync(W.G2.get(), W.G.get(), sizeof(double) * b * b, cudaMemcpyDeviceToDevice, c->stream));
        GEMB_TRY(ritz_eigh(W, o.tol, false, theta));
        const double tmax = std::max(theta[b - 1], 1e-300);
        const double change = sigma_change(&theta[b - k], &theta_prev[b - k], k, tmax);
        R.change = change;
        theta_prev = theta;
        if (o.verbose)
            fprintf(stderr, "[gemb_hope/general] it %d  sigma_max %.6g sigma_k %.6g  ritz change %.3g\n", it,
                    sqrt(tmax), sqrt(std::max(theta[b - k], 0.0)), change);
        if (o.stop_rule == 0) {
            if (it >= o.min_iters && change <= (double)o.tol) { R.converged = 1; break; }
            if (it == o.max_iters) break;
        }
        // T1 = U Z Theta^-1/2: exactly orthonormal columns (Z diagonalises U^T U), ordered by sigma, so the
        // next block S^T T1 ~ V Z Sigma has nearly orthogonal columns whatever the spread of sigma is
        GEMB_TRY(c->t_dense.begin(c->stream));
        ritz_maps_kernel<<<(b * b + 255) / 256, 256, 0, c->stream>>>(b, b, W.w.get(), W.Z.get(), W.M1.get(), W.M2.get(), -0.5, 0.5, 1e-10);
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        GEMB_TRY(apply_launch(c, W.rows, U, b, W.M1.get(), b, b, T1, b));
        GEMB_TRY(c->t_dense.end(c->stream));
        GEMB_TRY(apply_S(W, true, beta, J, T1, Wk, Hscr, T2));        // Wk = S^T T1   (stop_rule 0: U is scratch now)
        if (o.stop_rule == 0) { GEMB_TRY(cholqr2(W, Wk, T1, V)); continue; }   // V = orth(S^T orth(S V))
        // residual of the Ritz triplets (sigma_j, u_j = T1_j, v_j = V Z_j): S^T u_j = S^T S V Z_j theta_j^-1/2, so
        // v_j^T S^T u_j = theta_j^1/2 = sigma_j and ||S^T u_j - sigma_j v_j||^2 = (Wk^T Wk)_jj - theta_j.  That Gram is
        // the first one CholeskyQR2 forms; its diagonal is read before the Cholesky overwrites it.  S v_j - sigma_j u_j
        // is 0 by construction (U = S V).
        GEMB_TRY(gram_full(W, Wk, Wk, W.G.get()));
        GEMB_CUDA(cudaMemcpy2DAsync(wdiag.data(), sizeof(double), W.G.get(), sizeof(double) * (b + 1), sizeof(double), b,
                                    cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaStreamSynchronize(c->stream));
        double worst = 0.0;
        for (int j = b - k; j < b; j++) worst = std::max(worst, sqrt(std::max(wdiag[j] - theta[j], 0.0)) / sqrt(tmax));
        R.resid_est = (float)worst;
        if (o.verbose) fprintf(stderr, "[gemb_hope/general] it %d  residual %.3g\n", it, worst);
        if (it >= o.min_iters && worst <= (double)o.tol) { R.converged = 1; break; }
        if (it == o.max_iters) break;
        GEMB_TRY(cholqr_pass(W, W.G.get(), Wk, T1));                 // the rest of V = CholeskyQR2(Wk)
        GEMB_TRY(gram_full(W, T1, T1, W.G.get()));
        GEMB_TRY(cholqr_pass(W, W.G.get(), T1, V));
    }
    R.sigma_max = sqrt(std::max(theta[b - 1], 0.0));

    // extraction: X = [U Z_k theta^-1/4 | V Z_k theta^1/4]; U = S V (un-normalised), V orthonormal
    GEMB_TRY(place_output(W, R, T1, d));
    GEMB_TRY(c->t_dense.begin(c->stream));
    ritz_maps_kernel<<<(b * k + 255) / 256, 256, 0, c->stream>>>(b, k, W.w.get(), W.Z.get(), W.M1.get(), W.M2.get(), -0.25, 0.25);
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    GEMB_TRY(apply_launch(c, W.rows, U, b, W.M1.get(), k, k, R.Xd, d));
    GEMB_TRY(apply_launch(c, W.rows, V, b, W.M2.get(), k, k, R.Xd + k, d));
    sqrt_top_kernel<<<(k + 127) / 128, 128, 0, c->stream>>>(b, k, W.w.get(), R.sig_dev);
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    GEMB_TRY(c->t_dense.end(c->stream));

    if (o.compute_residual) {
        // left vectors P = U Z theta^-1/2 (all b Ritz pairs), right Q sigma = V Z theta^1/2
        ritz_maps_kernel<<<(b * b + 255) / 256, 256, 0, c->stream>>>(b, b, W.w.get(), W.Z.get(), W.M1.get(), W.M2.get(), -0.5, 0.5);
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        float *Pm = Wk, *Qs = T1;
        const size_t blk = (size_t)W.shard * b;
        DeviceBuffer<float> Qalloc, STP;
        if (!R.Xalloc.get()) {
            GEMB_CUDA(Qalloc.alloc(blk));
            GEMB_CUDA(cudaMemsetAsync(Qalloc.get(), 0, sizeof(float) * blk, c->stream));
            Qs = Qalloc.get();
        }
        GEMB_CUDA(STP.alloc(blk));
        GEMB_CUDA(cudaMemsetAsync(STP.get(), 0, sizeof(float) * blk, c->stream));
        GEMB_TRY(apply_launch(c, W.rows, U, b, W.M1.get(), b, b, Pm, b));
        GEMB_TRY(apply_launch(c, W.rows, V, b, W.M2.get(), b, b, Qs, b));
        std::vector<int> cols;
        for (int j = b - k; j < b; j++) cols.push_back(j);
        GEMB_TRY(residual_check(W, beta, J, Pm, Qs, STP.get(), U, T2, cols, R.sigma_max, &R.resid_max));
    }
    return GEMB_OK;
}

// dst = orth(F) where Z (= W.Z, eigenvectors of the last Rayleigh-Ritz matrix) pre-rotates the columns:
// F Z has nearly orthogonal columns (exactly, on an invariant subspace), so after the diagonal scaling
// inside chol_inverse the Cholesky factorisation is well conditioned whatever the dynamic range of the
// filter.  G' = Z^T (F^T F) Z,  G' = R^T R,  pass 1: tmp = F (Z R^-1);  pass 2: plain CholeskyQR.
static int orth_rotated(HopeWork &W, const float *F, float *tmp, float *dst) {
    gemb_ctx *c = W.c;
    const int b = W.b;
    GEMB_TRY(gram_full(W, F, F, W.G.get()));
    GEMB_TRY(c->t_dense.begin(c->stream));
    GEMB_TRY(small_gemm_launch(c, b, W.G.get(), 0, W.Z.get(), W.Zs.get(), nullptr));        // Zs = G Z
    GEMB_TRY(small_gemm_launch(c, b, W.Z.get(), 1, W.Zs.get(), W.G.get(), nullptr));        // G  = Z^T G Z
    GEMB_TRY(chol_inverse_launch(c, b, W.G.get(), W.Minv.get(), W.rank_dev.get(), W.G2.get()));   // G2 = R^-1 (fp64)
    GEMB_TRY(small_gemm_launch(c, b, W.Z.get(), 0, W.G2.get(), nullptr, W.M1.get()));       // M1 = Z R^-1
    GEMB_TRY(apply_launch(c, W.rows, F, b, W.M1.get(), b, b, tmp, b));
    GEMB_TRY(c->t_dense.end(c->stream));
    GEMB_TRY(gram_full(W, tmp, tmp, W.G.get()));
    GEMB_TRY(cholqr_pass(W, W.G.get(), tmp, dst));
    return GEMB_OK;
}

// V[:, j] <- Rn[:, j] for the columns j whose squared norm G[j][j] is below 1/2 (V orthonormal: the zeroed ones)
__global__ void refill_cols_kernel(int64_t count, int b, const double *__restrict__ G, const float *__restrict__ Rn,
                                   float *__restrict__ V) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        const int j = (int)(i % b);
        if (G[(size_t)j * b + j] < 0.5) V[i] = Rn[i];
    }
}

// Columns that the rank test of the CholeskyQR zeroed stay zero under every later filter, and their Ritz value 0 becomes
// the smallest |f| of the block, which collapses the damped interval onto 0 and makes further columns dependent.  When the
// last orthonormalisation of V dropped columns, they are replaced by Gaussian columns (seed per round) and V is
// orthonormalised again (two CholeskyQR passes); a full-rank V is left untouched.  s1, s2: scratch blocks.
static int refill_dropped(HopeWork &W, float *V, float *s1, float *s2, uint64_t seed) {
    gemb_ctx *c = W.c;
    const int b = W.b;
    int rank = b;
    GEMB_TRY(copy_sync(c, &rank, W.rank_dev.get(), sizeof(int), cudaMemcpyDeviceToHost));
    if (rank >= b) return GEMB_OK;      // the Gram is all-reduced: every rank takes the same branch
    GEMB_TRY(randn_launch(c, W.rows, b, seed, (uint64_t)W.g->row0, s1));
    GEMB_TRY(gram_full(W, V, V, W.G.get()));
    const int64_t count = W.rows * (int64_t)b;
    if (count > 0) {
        const int grid = (int)std::min<int64_t>((count + 255) / 256, (int64_t)c->sm_count * 8);
        refill_cols_kernel<<<grid, 256, 0, c->stream>>>(count, b, W.G.get(), s1, V);
        GEMB_CUDA(cudaGetLastError());
        count_launch();
    }
    GEMB_TRY(gram_full(W, V, V, W.G.get()));
    GEMB_TRY(cholqr_pass(W, W.G.get(), V, s2));
    GEMB_TRY(gram_full(W, s2, s2, W.G.get()));
    GEMB_TRY(cholqr_pass(W, W.G.get(), s2, V));
    return GEMB_OK;
}

// ------------------------------------------------------------------------------------ symmetric solvers
// The spectral map of the symmetric solvers.  Katz (spectral_mode 0): S = f(A), f(l) = beta l / (1 - beta l), so the
// wanted values are the largest |f(l)| over A's eigenvalues l; spectral_mode 1: the largest algebraic l themselves.
// spectral_mode 2 (negdef): the same on the composite -M^T M, whose spectrum is [-||M||_2^2, 0].
// Every Ritz value is clamped to [-bound, bound] ([-bound, 0] when negdef: Ritz values lie inside the spectrum) before
// it is mapped.
struct SpecMap {
    double beta;
    bool katz;
    double norm;    // a priori bound on |l|: ||A||_inf, or the power-iteration ||A||_2
    double bound;   // current bound on |l|
    bool estimated = false;   // norm is the power-iteration estimate, which can lie below ||A||_2 (a cluster of top values)
    bool negdef = false;      // spectral_mode 2: the operator is negative semi-definite; the wanted end is 0
    SpecMap(double beta, bool katz, double norm) : beta(beta), katz(katz), norm(norm), bound(norm * 1.02 + 1e-30) {}
    // an estimated norm is raised to max |l| over the Ritz values l[0..n) (all inside the spectrum), so that the clamp
    // never moves a Ritz value; false when then beta * norm >= 1 (the Katz series diverges)
    bool observe(const double *l, int n) {
        if (!estimated) return true;
        for (int i = 0; i < n; i++) norm = std::max(norm, fabs(l[i]));
        bound = std::max(bound, norm * 1.02 + 1e-30);
        return !katz || beta * norm < 1.0;
    }
    // bound from the Ritz values l[0..n): growth * max |l|, never above the a priori one
    void tighten(const double *l, int n, double growth) {
        double amax = 0.0;
        for (int i = 0; i < n; i++) amax = std::max(amax, fabs(l[i]));
        bound = std::min(norm * 1.02, growth * amax) + 1e-30;
    }
    double clamp(double l) const { return std::max(-bound, std::min(negdef ? 0.0 : bound, l)); }
    double f(double l) const { return beta * l / (1.0 - beta * l); }
    // rank key, largest wanted first: |f(l)| (= sigma), or l + bound
    double key(double l) const { l = clamp(l); return katz ? fabs(f(l)) : l + bound; }
    // the value the stop measures are taken on and relative to: the key sigma (Katz), the eigenvalue l (mode 1; its
    // key carries the shift `bound`, which would make both measures ~2x looser on D^-1/2 A D^-1/2)
    double value(double l) const { return katz ? key(l) : clamp(l); }
    // |d key / dl|: maps an eigen-residual of A to the residual of the key's triplet (|f'(l)| = beta / (1 - beta l)^2)
    double slope(double l) const { l = clamp(l); return katz ? beta / ((1.0 - beta * l) * (1.0 - beta * l)) : 1.0; }
    // Chebyshev filter interval [c0 - e, c0 + e] over the damped set {l : key(l) < key(l_min)}, l_min the block's Ritz
    // value of smallest key, and the end aL (+-bound; negdef: 0) the filter is normalised at: the dominant end, the
    // side of l_top
    struct Interval { double e, c0, aL; };
    Interval damped(double l_top, double l_min) const {
        const double tau = key(l_min);
        double hi = katz ? tau / (beta * (1.0 + tau)) : clamp(l_min);
        double lo = katz && tau < 1.0 ? -tau / (beta * (1.0 - tau)) : -bound;
        lo = std::max(lo, -bound);
        hi = std::min(hi, bound);
        if (hi - lo < 2e-3 * bound) { const double mid = 0.5 * (hi + lo); lo = mid - 1e-3 * bound; hi = mid + 1e-3 * bound; }
        const double e = 0.5 * (hi - lo), c0 = 0.5 * (hi + lo);
        return {e, c0, negdef ? 0.0 : ((!katz || l_top >= c0) ? bound : -bound)};
    }
    // the output of Ritz value l: sigma (|f(l)|, or l), the scale of its vector in X (sqrt(sigma), or 1), and whether
    // the left half of X takes the vector negated (f(l) < 0)
    struct Column { double sigma, scale; bool neg; };
    Column column(double l) const {
        l = clamp(l);
        if (!katz) return {l, 1.0, false};
        const double fl = f(l);
        return {fabs(fl), sqrt(fabs(fl)), fl < 0};
    }
    // X column of the j-th best of k: HOPE lists sigma ascending (as svds does), LE / LLE eigenvalues descending
    int out_col(int j, int k) const { return katz ? k - 1 - j : j; }
};

constexpr int GEMB_SWITCH_TO_LANCZOS = 1000;   // internal status of hope_symmetric (algorithm = 0 on a skewed spectrum)

static int diverge_error(const SpecMap &map) {
    set_error("beta * ||A||_2 >= %.4g (a Ritz value of magnitude %.4g): the Katz series (I - beta A)^-1 beta A does not "
              "converge; choose beta < %.4g", map.beta * map.norm, map.norm, 1.0 / map.norm);
    return GEMB_ERR_DIVERGE;
}

// ritz_bound: A is symmetric with non-negative weights and map.norm = ||A||_inf; then lambda_max = rho(A) >= |lambda_min|
// (Perron-Frobenius), so 1.05 * (largest Ritz value) bounds the spectrum on both sides and the 2 x 16 narrow SpMM sweeps
// of the power iteration are not needed.  Otherwise map.norm is a tight estimate of ||A||_2 (power iteration).
static int hope_symmetric(HopeWork &W, const Opts &o, int d, SpecMap map, bool ritz_bound, HopeResult &R) {
    gemb_ctx *c = W.c;
    const int mode = o.spectral_mode;
    const int b = W.b, k = mode ? d : d / 2;
    R.algorithm = 2;
    R.katz_terms = 0;
    float *V = W.buf[0], *AV = W.buf[1];
    float *pool[3] = {W.buf[2], W.buf[3], W.buf[4]};

    // warm-up: V = orth(A^3 R), R Gaussian.  The three power steps run on the raw block and ONE CholeskyQR2 closes them
    // (round 1 orthonormalised after every step: 4 x CholeskyQR2 = 3.5 ms of the 58 ms solve at S, for nothing -- the
    // block's condition number after three steps is (lambda_1 / lambda_b)^3, a few units on a community graph).  Should
    // the first Cholesky drop columns (skewed spectrum, rank-deficient A), the careful form below takes over.
    // spectral_mode 2: the wanted end of -M^T M is 0, its smallest |l|, which a power step would damp: the warm-up
    // steps run on the shifted -M^T M + bound I instead, whose wanted end is its largest value.
    const bool shift = mode == 2;
    const float nu = shift ? (float)map.bound : 0.f;
    GEMB_TRY(randn_launch(c, W.rows, b, o.seed, (uint64_t)W.g->row0, pool[0]));
    GEMB_TRY(publish(W, pool[0], b));
    GEMB_TRY(op_apply(W, b, 1.f, pool[0], nu, shift, 1.f, nullptr, pool[1], true, W.halo));
    GEMB_TRY(op_apply(W, b, 1.f, pool[1], nu, shift, 1.f, nullptr, pool[2], true, W.halo));
    GEMB_TRY(op_apply(W, b, 1.f, pool[2], nu, shift, 1.f, nullptr, AV, true));
    GEMB_TRY(gram_full(W, AV, AV, W.G.get()));
    GEMB_TRY(cholqr_pass(W, W.G.get(), AV, pool[0]));
    int rank1 = b;
    GEMB_TRY(copy_sync(c, &rank1, W.rank_dev.get(), sizeof(int), cudaMemcpyDeviceToHost));
    if (rank1 >= b) {
        GEMB_TRY(gram_full(W, pool[0], pool[0], W.G.get()));
        GEMB_TRY(cholqr_pass(W, W.G.get(), pool[0], V));
        GEMB_TRY(publish(W, V, b));
    } else {
        GEMB_TRY(randn_launch(c, W.rows, b, o.seed, (uint64_t)W.g->row0, pool[0]));
        GEMB_TRY(cholqr2(W, pool[0], pool[1], V));
        GEMB_TRY(publish(W, V, b));
        for (int s = 0; s < 3; s++) {   // plain power steps V <- orth(A V)
            GEMB_TRY(op_apply(W, b, 1.f, V, nu, shift, 1.f, nullptr, AV, true));
            GEMB_TRY(cholqr2(W, AV, pool[0], V));
            GEMB_TRY(publish(W, V, b));
        }
    }

    std::vector<double> lam(2 * b), gval(b), th_sorted(b), th_prev(b, 0.0);   // lam[b..2b): z^T (AV)^T (AV) z (stop rule 1)
    std::vector<double> vals(b), vals_prev(b, 0.0);                            // mode 1: the eigenvalues in rank order
    std::vector<int> order(b);

    // scaled three-term Chebyshev recurrence of degree deg on [c0 - e, c0 + e], normalised at the dominant end by
    // sigma1 = e / (aL - c0); returns the filtered block (one of the pool buffers); A V must be current
    auto run_filter = [&](int deg, double e, double c0, double sigma1, float **out) -> int {
        double sigma = sigma1;
        const double tau2 = 2.0 / sigma1;
        float *prev = V, *cur = pool[0];
        float *free_a = pool[1], *free_b = pool[2];
        // Y1 = (sigma/e) (A V - c0 V)  -- A V is the Rayleigh-Ritz product, no extra SpMM
        GEMB_TRY(axpby_launch(W, (float)(sigma / e), AV, (float)(-sigma * c0 / e), V, cur));
        for (int i = 2; i <= deg; i++) {
            const double sn = 1.0 / (tau2 - sigma);
            float *nxt = free_a;
            GEMB_TRY(op_apply(W, b, (float)(2.0 * sn / e), cur, (float)(-2.0 * sn * c0 / e), true, (float)(-sigma * sn),
                              prev, nxt, true, /*push_out=*/i < deg));
            sigma = sn;
            // rotate: the old `prev` becomes free unless it is V (V must survive until the new basis exists)
            float *old_prev = prev;
            prev = cur;
            cur = nxt;
            if (old_prev == V) { free_a = free_b; free_b = nullptr; }
            else { free_a = old_prev; }
        }
        *out = cur;
        return GEMB_OK;
    };

    for (int it = 1; it <= o.max_iters; it++) {
        R.iters = it;
        // Rayleigh-Ritz on A: T = V^T A V, (l, Z) = eigh(T)
        GEMB_TRY(op_apply(W, b, 1.f, V, 0.f, false, 1.f, nullptr, AV, true));
        GEMB_TRY(gram_full(W, V, AV, W.G2.get()));
        // (Measured: running the single-CTA Jacobi on a side stream while the filter starts with the PREVIOUS
        // round's interval costs two extra rounds -- 75 instead of 56 SpMM sweeps -- and is slower overall;
        // the eigen-decomposition therefore stays on the critical path.)
        GEMB_TRY(ritz_eigh(W, o.tol, true, lam, o.stop_rule == 1 ? AV : nullptr));
        if (ritz_bound) map.tighten(lam.data(), b, 1.05);
        else if (!map.observe(lam.data(), b)) return diverge_error(map);
        R.norm = map.norm;
        for (int i = 0; i < b; i++) gval[i] = map.key(lam[i]);
        std::iota(order.begin(), order.end(), 0);
        std::sort(order.begin(), order.end(), [&](int a, int c2) { return gval[a] > gval[c2]; });   // descending key
        for (int i = 0; i < b; i++) th_sorted[i] = gval[order[i]] * gval[order[i]];
        const double tmax = std::max(th_sorted[0], 1e-300);
        // vmax: max |value| over the wanted pairs (Katz: sigma_max = gval[order[0]]).  spectral_mode 2: the operator
        // bound ||M||_2^2 -- the wanted eigenvalues -sigma^2 lie near 0, and both stop measures are taken relative to
        // the operator, as the explicit form's are relative to its shift c >= ||M||_2^2
        double vmax = 0.0;
        if (mode == 2) vmax = map.norm;
        else for (int j = 0; j < k; j++) vmax = std::max(vmax, fabs(map.value(lam[order[j]])));
        double change;
        if (mode) {
            for (int i = 0; i < b; i++) vals[i] = map.value(lam[order[i]]);
            if (mode == 2) {        // round 1 has nothing to compare with (vals_prev = 0 would read as a tiny change)
                change = it == 1 ? HUGE_VAL : 0.0;
                for (int j = 0; j < k && it > 1; j++) change = std::max(change, fabs(vals[j] - vals_prev[j]) / std::max(vmax, 1e-300));
            } else change = value_change(vals.data(), vals_prev.data(), k, vmax);
            vals_prev = vals;
        } else change = sigma_change(th_sorted.data(), th_prev.data(), k, tmax);
        R.change = change;
        th_prev = th_sorted;
        // algorithm = 0 (auto): a first Rayleigh-Ritz round whose wanted values already span more than 3x -- a
        // power-law spectrum -- is a case for restarted Lanczos: a filter that damps everything below the k-th value
        // spreads the wanted columns over g^m and degenerates to power steps (DESIGN section 5)
        if (it == 1 && !mode && o.algorithm == 0 && W.g->n >= 2048 && gval[order[k - 1]] < 0.33 * gval[order[0]] &&
            gval[order[std::min(b - 1, 3)]] < 0.7 * gval[order[0]])
            return GEMB_SWITCH_TO_LANCZOS;
        double stop_measure = change;
        if (o.stop_rule == 1) {
            // residual of the Ritz pairs from the Rayleigh-Ritz products alone: with V orthonormal and (l, z) an
            // eigenpair of V^T A V,  ||A V z - l V z||^2 = z^T (AV)^T (AV) z - l^2.  Mapped to the Katz operator
            // through |f'(l)| = beta / (1 - beta l)^2 and measured against sigma_max, like compute_residual does;
            // mode 1: ||A v - l v|| against max |l| over the wanted pairs.
            double worst = 0.0;
            for (int j = 0; j < k; j++) {
                const int col = order[j];
                const double r2 = std::max(lam[b + col] - lam[col] * lam[col], 0.0);
                worst = std::max(worst, map.slope(lam[col]) * sqrt(r2) / std::max(vmax, 1e-300));
            }
            stop_measure = worst;
            R.resid_est = (float)worst;
        }
        if (o.verbose)
            fprintf(stderr, "[gemb_hope/symmetric] it %d  sigma_max %.6g sigma_k %.6g  ritz change %.3g%s%.3g\n", it,
                    gval[order[0]], gval[order[k - 1]], change, o.stop_rule == 1 ? "  residual " : " ", o.stop_rule == 1 ? stop_measure : 0.0);
        if (it >= o.min_iters && stop_measure <= (double)o.tol) { R.converged = 1; break; }
        if (it == o.max_iters) break;

        // filter interval over the damped set: every key below the smallest one in the block
        const SpecMap::Interval iv = map.damped(lam[order[0]], lam[order[b - 1]]);
        const double sigma1 = iv.e / (iv.aL - iv.c0);
        // fp32 guard: the filter spreads the block's columns over a dynamic range T_m(x_L) ~ g^m / 2; the
        // Gram-based orthonormalisation squares it, so keep it below ~2^8 (degree m), else take a power step
        const double xL = fabs(iv.aL - iv.c0) / iv.e;
        const double growth = xL + sqrt(std::max(xL * xL - 1.0, 0.0));
        int deg = o.cheb_degree;
        // opts.cheb_range_log2 (default 8): the column scaling inside the
        // Ritz-rotated CholeskyQR tolerates far more than 2^8 on the SBM spectrum (scripts/exp_solver.py sweeps the settings):
        // 2^14 with degree 16 reaches a residual of 3.0e-3 in 4 rounds / 42 sweeps (the bench setting) where 2^8 with degree 8
        // needed 8 rounds / 56 sweeps for 4.0e-3.  The library default stays conservative (tight-tolerance solves).
        if (growth > 1.0 + 1e-9) deg = std::min(deg, (int)floor(log(2.0 * exp2((double)o.range_log2)) / log(growth)));

        if (deg < 2) {                                          // A V is already there: one power step
            if (shift) {                                        // on -M^T M + bound I, as in the warm-up
                GEMB_TRY(axpby_launch(W, 1.f, AV, nu, V, pool[1]));
                GEMB_TRY(orth_rotated(W, pool[1], pool[0], V));
            } else GEMB_TRY(orth_rotated(W, AV, pool[0], V));
            GEMB_TRY(refill_dropped(W, V, pool[0], pool[1], o.seed + 7919ull * (uint64_t)it));
            GEMB_TRY(publish(W, V, b));
            continue;
        }
        float *filtered = nullptr;
        GEMB_TRY(run_filter(deg, iv.e, iv.c0, sigma1, &filtered));
        // orthonormalise the filtered block into V; scratch = any block that is neither `filtered` nor V
        float *tmp = nullptr;
        for (float *cand : {pool[0], pool[1], pool[2], AV})
            if (cand != filtered) { tmp = cand; break; }
        GEMB_TRY(orth_rotated(W, filtered, tmp, V));
        GEMB_TRY(refill_dropped(W, V, tmp, filtered, o.seed + 7919ull * (uint64_t)it));
        GEMB_TRY(publish(W, V, b));
    }

    // ---- extraction: the k wanted columns, in output order (map.out_col).  Katz: X = [ V Z_k sign(f) sqrt(sigma) |
    // V Z_k sqrt(sigma) ]; LE / LLE: X = V Z_k, the largest algebraic eigenpairs DESCENDING (= ascending eigenvalues of
    // I - A_hat, the order lap.py:28-31 sorts into)
    std::vector<double> Zh((size_t)b * b);
    GEMB_TRY(copy_sync(c, Zh.data(), W.Z.get(), sizeof(double) * b * b, cudaMemcpyDeviceToHost));
    // M = [M1 | M2] (b x d; LE / LLE: M1 alone, b x k): one apply writes whole rows of X
    const int xw = mode ? k : 2 * k;
    std::vector<float> M((size_t)b * xw), sig(k);
    std::vector<int> sel(k);
    for (int j = 0; j < k; j++) {
        const int col = order[j], q = map.out_col(j, k);
        const SpecMap::Column t = map.column(lam[col]);
        sel[q] = col;
        sig[q] = (float)t.sigma;
        for (int i = 0; i < b; i++) {
            const double z = Zh[(size_t)i * b + col];
            M[(size_t)i * xw + q] = (float)((t.neg ? -z : z) * t.scale);
            if (!mode) M[(size_t)i * xw + k + q] = (float)(z * t.scale);
        }
    }
    R.sigma_max = gval[order[0]];
    GEMB_TRY(place_output(W, R, pool[0], d));
    GEMB_CUDA(cudaMemcpyAsync(W.M1.get(), M.data(), sizeof(float) * b * xw, cudaMemcpyHostToDevice, c->stream));
    GEMB_TRY(copy_sync(c, R.sig_dev, sig.data(), sizeof(float) * k, cudaMemcpyHostToDevice));   // host staging goes out of scope
    GEMB_TRY(c->t_dense.begin(c->stream));
    GEMB_TRY(apply_launch(c, W.rows, V, b, W.M1.get(), xw, xw, R.Xd, d));
    GEMB_TRY(c->t_dense.end(c->stream));
    if (mode || !o.compute_residual) return GEMB_OK;

    // check the triplets against the Katz operator itself: || S^T u - sigma v || / sigma_max
    const int J = katz_terms_for(map.beta, ritz_bound ? map.bound / 1.02 : map.norm, o.katz_tol);
    std::vector<float> MP((size_t)b * b, 0.f), MQ((size_t)b * b, 0.f);
    for (int col = 0; col < b; col++) {
        const SpecMap::Column t = map.column(lam[col]);
        for (int i = 0; i < b; i++) {
            const double z = Zh[(size_t)i * b + col];
            MP[(size_t)i * b + col] = (float)(t.neg ? -z : z);    // u = sign(f) v
            MQ[(size_t)i * b + col] = (float)(z * t.sigma);       // v sigma
        }
    }
    DeviceBuffer<float> dMP, dMQ, Palloc, Q, STP;
    const size_t blk = (size_t)W.shard * b;
    GEMB_CUDA(dMP.alloc(b * b));
    GEMB_CUDA(dMQ.alloc(b * b));
    // every SpMM INPUT must be a work block in halo mode (its rows travel to the peers): P lives in AV, the Horner
    // scratch in pool[1] / pool[2]; pool[0] may hold the result X and stays untouched
    float *P = AV;
    if (!W.halo) {
        GEMB_CUDA(Palloc.alloc(blk));
        GEMB_CUDA(cudaMemsetAsync(Palloc.get(), 0, sizeof(float) * blk, c->stream));
        P = Palloc.get();
    }
    GEMB_CUDA(Q.alloc(blk));
    GEMB_CUDA(STP.alloc(blk));
    GEMB_CUDA(cudaMemsetAsync(Q.get(), 0, sizeof(float) * blk, c->stream));
    GEMB_CUDA(cudaMemsetAsync(STP.get(), 0, sizeof(float) * blk, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(dMP.get(), MP.data(), sizeof(float) * b * b, cudaMemcpyHostToDevice, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(dMQ.get(), MQ.data(), sizeof(float) * b * b, cudaMemcpyHostToDevice, c->stream));
    GEMB_TRY(apply_launch(c, W.rows, V, b, dMP.get(), b, b, P, b));
    GEMB_TRY(apply_launch(c, W.rows, V, b, dMQ.get(), b, b, Q.get(), b));
    GEMB_TRY(publish(W, P, b));
    return residual_check(W, (float)map.beta, J, P, Q.get(), STP.get(), W.halo ? pool[1] : AV, W.halo ? pool[2] : pool[1], sel,
                          R.sigma_max, &R.resid_max);
}

// ------------------------------------------------------------------------------------ Lanczos solver
// dst[:, col0 .. col0+w) (leading dimension ldd) = src (n x w, contiguous)
__global__ void put_cols_kernel(int64_t n, int w, const float *__restrict__ src, float *__restrict__ dst, int ldd, int col0) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * w; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / w;
        const int cc = (int)(i - r * w);
        dst[r * ldd + col0 + cc] = src[i];
    }
}
// dst[:, col_last - q] = src[:, q], q < w   (ascending-sigma column order of the result)
__global__ void reverse_put_kernel(int64_t n, int w, const float *__restrict__ src, int lds, float *__restrict__ dst, int ldd, int col_last) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * w; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / w;
        const int q = (int)(i - r * w);
        dst[r * ldd + col_last - q] = src[r * lds + q];
    }
}
__global__ void f64_to_f32_kernel(int count, const double *__restrict__ a, float *__restrict__ o) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < count) o[i] = (float)a[i];
}

// Thick-restart block Lanczos (block Krylov-Schur) on the symmetric A; S = f(A) shares its eigenvectors, so the
// singular triplets of S are (|f(l)|, sign(f(l)) v, v) for the k eigenpairs with the largest |f(l)|.  This is the
// block form of what ARPACK does behind scipy's svds (hope.py:33, SURVEY Appendix B: restarted Lanczos, ncv = 2k+1),
// and it is the solver for power-law spectra (R-MAT, BASELINE configs[3]) on which Chebyshev-filtered subspace
// iteration degenerates to power steps.
//   basis Q (n x m, m <= m_max) in chunks of 64 columns; block width p = 16
//   step:   W = A q_j (SpMM, width 16: the 64-byte rows of the input block stay L2-resident)
//           H = Q^T W, W -= Q H, twice (classical Gram-Schmidt x 2; Gram and update on the tensor cores, b x b
//           all-reduce on N GPUs); T[:, j] = H (T = Q^T A Q is kept explicitly, so the arrowhead left by a restart needs
//           no special case); q_{j+1} R = W by CholeskyQR2
//   full:   (theta, Y) = eigh(T); residual of Ritz pair i = || R Y[last block, i] || (no extra sweep);
//           stop when |f'(theta_i)| res_i <= tol * sigma_max for the k wanted pairs;
//           else keep the k + 16 best by |f|: Q <- Q Y_keep, T <- diag(theta_keep), continue with q_{j+1}
static int hope_lanczos(HopeWork &W, const Opts &o, int d, SpecMap map, HopeResult &R) {
    gemb_ctx *c = W.c;
    const int k = d / 2, p = 16, cw = 64;
    const int64_t rows = W.rows, shard = W.shard;
    R.algorithm = 3;
    R.katz_terms = 0;
    const int k_keep = (k + p + p - 1) / p * p;
    int m_max = o.lanczos_basis > 0 ? o.lanczos_basis : std::max(2 * k_keep, 160);
    m_max = (m_max + p - 1) / p * p;
    GEMB_ARG(m_max >= k_keep + 2 * p && m_max <= 1024, "algorithm3_basis");
    const int nchunk = (m_max + cw - 1) / cw;
    const int mt = m_max + p;                                    // T carries the coupling block of the next q too
    const size_t chunk_bytes = sizeof(float) * (size_t)shard * cw;
    std::vector<DeviceBuffer<float>> Q(nchunk), Qn((k_keep + cw - 1) / cw);
    for (auto &q : Q) { GEMB_CUDA(q.alloc((size_t)shard * cw)); GEMB_CUDA(cudaMemsetAsync(q.get(), 0, chunk_bytes, c->stream)); }
    for (auto &q : Qn) GEMB_CUDA(q.alloc((size_t)shard * cw));
    // narrow blocks: Vcur (SpMM input: a halo block on N GPUs), Wb, Tb
    float *Vcur = W.buf[0], *Wb = W.buf[1], *Tb = W.buf[2];
    DeviceBuffer<float> Tmp64, M32;
    DeviceBuffer<double> Gd, Td, Yd, wd, Zs;                     // device: small Gram (cw x p), T (m x m), Y, eigh's w and scratch
    GEMB_CUDA(Tmp64.alloc((size_t)shard * cw));
    GEMB_CUDA(Gd.alloc((size_t)cw * cw));
    GEMB_CUDA(Td.alloc((size_t)mt * mt));
    GEMB_CUDA(Yd.alloc((size_t)mt * mt));
    GEMB_CUDA(M32.alloc((size_t)cw * cw));
    GEMB_CUDA(wd.alloc(mt));
    GEMB_CUDA(Zs.alloc((size_t)mt * mt));

    const int grid_el = c->sm_count * 8;
    auto gram_ar = [&](const float *P, int b1, const float *Qp, int b2, double *G) -> int {
        GEMB_TRY(c->t_dense.begin(c->stream));
        GEMB_TRY(gram_launch(c, rows, P, b1, Qp, b2, G));
        GEMB_TRY(c->t_dense.end(c->stream));
        return comm_allreduce_f64(W, G, (size_t)b1 * b2);
    };
    // CholeskyQR2 of the n x p block `src` in place (scratch Tb); Rout (p x p, host, row-major upper) = R2 * R1
    std::vector<double> Rh((size_t)p * p), R1((size_t)p * p), R2((size_t)p * p), Ginv((size_t)p * p);
    auto cholqr_p = [&](float *src, float *scratch, double *Rout) -> int {
        for (int pass = 0; pass < 2; pass++) {
            GEMB_TRY(gram_ar(src, p, src, p, W.G.get()));
            GEMB_TRY(c->t_dense.begin(c->stream));
            GEMB_TRY(chol_inverse_launch(c, p, W.G.get(), W.Minv.get(), W.rank_dev.get(), W.G2.get()));     // G2 = R^-1 (fp64)
            GEMB_TRY(apply_launch(c, rows, src, p, W.Minv.get(), p, p, scratch, p));
            GEMB_TRY(c->t_dense.end(c->stream));
            GEMB_CUDA(cudaMemcpyAsync(src, scratch, sizeof(float) * (size_t)rows * p, cudaMemcpyDeviceToDevice, c->stream));
            GEMB_TRY(copy_sync(c, Ginv.data(), W.G2.get(), sizeof(double) * p * p, cudaMemcpyDeviceToHost));
            // invert the upper-triangular R^-1 on the host (p = 16): R = (R^-1)^-1; dropped columns (zero pivot) stay zero
            std::vector<double> &Rt = pass == 0 ? R1 : R2;
            std::fill(Rt.begin(), Rt.end(), 0.0);
            for (int j = 0; j < p; j++) {
                if (Ginv[(size_t)j * p + j] == 0.0) continue;
                Rt[(size_t)j * p + j] = 1.0 / Ginv[(size_t)j * p + j];
                for (int i = j - 1; i >= 0; i--) {
                    if (Ginv[(size_t)i * p + i] == 0.0) continue;
                    double sacc = 0.0;
                    for (int l = i + 1; l <= j; l++) sacc += Ginv[(size_t)i * p + l] * Rt[(size_t)l * p + j];
                    Rt[(size_t)i * p + j] = -sacc / Ginv[(size_t)i * p + i];
                }
            }
        }
        for (int i = 0; i < p; i++)
            for (int j = 0; j < p; j++) {
                double a = 0.0;
                for (int l = 0; l < p; l++) a += R2[(size_t)i * p + l] * R1[(size_t)l * p + j];
                Rout[(size_t)i * p + j] = a;
            }
        return GEMB_OK;
    };

    std::vector<double> T((size_t)mt * mt, 0.0), Hcol((size_t)m_max * p), Hc((size_t)cw * p), theta(m_max), Y((size_t)m_max * m_max);
    std::vector<double> fabsv(m_max);
    std::vector<int> order(m_max);
    GEMB_TRY(randn_launch(c, rows, p, o.seed, (uint64_t)W.g->row0, Vcur));
    GEMB_TRY(cholqr_p(Vcur, Tb, Rh.data()));
    int m = 0, restarts = 0, steps = 0;
    const int max_steps = std::max(o.max_iters, 1) * (m_max / p);
    bool done = false;
    while (!done) {
        // ---- append q_j, expand
        put_cols_kernel<<<grid_el, 256, 0, c->stream>>>(rows, p, Vcur, Q[m / cw].get(), cw, m % cw);
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        const int j0 = m;
        m += p;
        steps++;
        GEMB_TRY(publish(W, Vcur, p));
        GEMB_TRY(dist_spmm3(W, false, p, 1.f, Vcur, 0.f, false, 1.f, nullptr, Wb, true, false));
        std::fill(Hcol.begin(), Hcol.end(), 0.0);
        const int nc_live = (m + cw - 1) / cw;
        for (int pass = 0; pass < 2; pass++) {
            for (int cc = 0; cc < nc_live; cc++) {
                GEMB_TRY(gram_ar(Q[cc].get(), cw, Wb, p, Gd.get()));                               // H_c = Q_c^T W   (cw x p)
                GEMB_TRY(c->t_dense.begin(c->stream));
                f64_to_f32_kernel<<<(cw * p + 255) / 256, 256, 0, c->stream>>>(cw * p, Gd.get(), M32.get());
                GEMB_CUDA(cudaGetLastError());
                count_launch();
                GEMB_TRY(apply_launch(c, rows, Q[cc].get(), cw, M32.get(), p, p, Tb, p));           // Q_c H_c
                GEMB_TRY(axpy_launch(c, rows * (int64_t)p, -1.f, Tb, Wb));
                GEMB_TRY(c->t_dense.end(c->stream));
                GEMB_TRY(copy_sync(c, Hc.data(), Gd.get(), sizeof(double) * cw * p, cudaMemcpyDeviceToHost));
                for (int r = 0; r < cw && cc * cw + r < m; r++)
                    for (int q = 0; q < p; q++) Hcol[(size_t)(cc * cw + r) * p + q] += Hc[(size_t)r * p + q];
            }
        }
        for (int r = 0; r < m; r++)
            for (int q = 0; q < p; q++) {
                const double v = Hcol[(size_t)r * p + q];
                T[(size_t)r * mt + j0 + q] = v;
                T[(size_t)(j0 + q) * mt + r] = v;
            }
        for (int a2 = 0; a2 < p; a2++)                                                   // symmetrise the diagonal block
            for (int b2 = a2 + 1; b2 < p; b2++) {
                const double v = 0.5 * (T[(size_t)(j0 + a2) * mt + j0 + b2] + T[(size_t)(j0 + b2) * mt + j0 + a2]);
                T[(size_t)(j0 + a2) * mt + j0 + b2] = v;
                T[(size_t)(j0 + b2) * mt + j0 + a2] = v;
            }
        GEMB_TRY(cholqr_p(Wb, Tb, Rh.data()));                                           // q_{j+1} R = W
        // Vcur = q_{j+1}: always work block 0 (on N GPUs its halo is the one the peers fill), a 64-byte-per-row copy
        GEMB_CUDA(cudaMemcpyAsync(Vcur, Wb, sizeof(float) * (size_t)rows * p, cudaMemcpyDeviceToDevice, c->stream));
        const bool full = m + p > m_max;
        if (!full && steps < max_steps) continue;

        // ---- Rayleigh-Ritz on T[0:m, 0:m]
        std::vector<double> Tm((size_t)m * m);
        for (int r = 0; r < m; r++) for (int q = 0; q < m; q++) Tm[(size_t)r * m + q] = T[(size_t)r * mt + q];
        GEMB_CUDA(cudaMemcpyAsync(Td.get(), Tm.data(), sizeof(double) * m * m, cudaMemcpyHostToDevice, c->stream));
        GEMB_TRY(c->t_dense.begin(c->stream));
        GEMB_TRY(eigh_launch(c, m, Td.get(), wd.get(), Yd.get(), Zs.get(), 1e-9));      // Ritz values are needed to ~1e-6, the vectors feed fp32 GEMMs
        GEMB_TRY(c->t_dense.end(c->stream));
        GEMB_CUDA(cudaMemcpyAsync(theta.data(), wd.get(), sizeof(double) * m, cudaMemcpyDeviceToHost, c->stream));
        GEMB_TRY(copy_sync(c, Y.data(), Yd.get(), sizeof(double) * m * m, cudaMemcpyDeviceToHost));
        map.tighten(theta.data(), m, 1.02);
        for (int i = 0; i < m; i++) fabsv[i] = map.key(theta[i]);
        std::iota(order.begin(), order.begin() + m, 0);
        std::sort(order.begin(), order.begin() + m, [&](int a2, int b2) { return fabsv[a2] > fabsv[b2]; });
        const double smax = std::max(fabsv[order[0]], 1e-300);
        double worst = 0.0;
        for (int jj = 0; jj < std::min(k, m); jj++) {
            const int col = order[jj];
            double r2 = 0.0;
            for (int a2 = 0; a2 < p; a2++) {
                double t = 0.0;
                for (int b2 = 0; b2 < p; b2++) t += Rh[(size_t)a2 * p + b2] * Y[(size_t)(m - p + b2) * m + col];
                r2 += t * t;
            }
            worst = std::max(worst, map.slope(theta[col]) * sqrt(r2) / smax);
        }
        R.change = worst;
        R.resid_est = (float)worst;
        restarts++;
        R.iters = restarts;
        if (o.verbose)
            fprintf(stderr, "[gemb_hope/lanczos] restart %d  basis %d  steps %d  sigma_max %.6g sigma_k %.6g  residual %.3g\n", restarts, m,
                    steps, smax, fabsv[order[std::min(k, m) - 1]], worst);
        const bool conv = m >= k && worst <= (double)o.tol;
        if (conv) R.converged = 1;
        done = conv || steps >= max_steps;
        // ---- compress: Q <- Q Y[:, keep]   (keep = the k_keep best by |f|; on exit: the k wanted, scaled for X)
        const int nk = done ? k : std::min(k_keep, m);
        const int ncn = (nk + cw - 1) / cw;
        for (int oc = 0; oc < ncn; oc++) {
            const int ow = std::min(cw, nk - oc * cw);
            for (int cc = 0; cc < nc_live; cc++) {
                std::vector<float> Mh((size_t)cw * cw, 0.f);
                for (int r = 0; r < cw && cc * cw + r < m; r++)
                    for (int q = 0; q < ow; q++) Mh[(size_t)r * cw + q] = (float)Y[(size_t)(cc * cw + r) * m + order[oc * cw + q]];
                GEMB_TRY(copy_sync(c, M32.get(), Mh.data(), sizeof(float) * cw * cw, cudaMemcpyHostToDevice));
                GEMB_TRY(c->t_dense.begin(c->stream));
                GEMB_TRY(apply_launch(c, rows, Q[cc].get(), cw, M32.get(), cw, cw, cc == 0 ? Qn[oc].get() : Tmp64.get(), cw));
                if (cc > 0) GEMB_TRY(axpy_launch(c, rows * (int64_t)cw, 1.f, Tmp64.get(), Qn[oc].get()));
                GEMB_TRY(c->t_dense.end(c->stream));
            }
        }
        if (done) {
            // X = [ v sign(f) sqrt(sigma) | v sqrt(sigma) ], sigma ascending
            std::vector<float> sig(k);
            R.sigma_max = smax;
            GEMB_TRY(place_output(W, R, nullptr, d));
            GEMB_ARG(k <= cw * (int)Qn.size(), "k");
            // per-column scaling on the host: column jj of Qn <-> order[jj] (descending |f|); output column k-1-jj
            std::vector<float> Ms((size_t)cw * cw), Mt((size_t)cw * cw);
            for (int oc = 0; oc < ncn; oc++) {
                const int ow = std::min(cw, k - oc * cw);
                std::fill(Ms.begin(), Ms.end(), 0.f); std::fill(Mt.begin(), Mt.end(), 0.f);
                for (int q = 0; q < ow; q++) {
                    const int jj = oc * cw + q, col = order[jj];
                    const SpecMap::Column t = map.column(theta[col]);
                    sig[k - 1 - jj] = (float)t.sigma;
                    Ms[(size_t)q * cw + q] = (float)(t.neg ? -t.scale : t.scale);
                    Mt[(size_t)q * cw + q] = (float)t.scale;
                }
                for (int half = 0; half < 2; half++) {
                    GEMB_TRY(copy_sync(c, M32.get(), (half == 0 ? Ms : Mt).data(), sizeof(float) * cw * cw, cudaMemcpyHostToDevice));
                    GEMB_TRY(apply_launch(c, rows, Qn[oc].get(), cw, M32.get(), cw, cw, Tmp64.get(), cw));
                    // reversed column order into X: source column q -> X column (half*k) + k-1-(oc*cw+q)
                    reverse_put_kernel<<<grid_el, 256, 0, c->stream>>>(rows, ow, Tmp64.get(), cw, R.Xd, d, half * k + k - 1 - oc * cw);
                    GEMB_CUDA(cudaGetLastError());
                    count_launch();
                }
            }
            GEMB_TRY(copy_sync(c, R.sig_dev, sig.data(), sizeof(float) * k, cudaMemcpyHostToDevice));
            break;
        }
        // ---- restart: new basis = Qn (nk columns), T = diag(theta_keep); q_{j+1} (= Vcur) is appended next
        for (int oc = 0; oc < nchunk; oc++) {
            if (oc < ncn) GEMB_CUDA(cudaMemcpyAsync(Q[oc].get(), Qn[oc].get(), chunk_bytes, cudaMemcpyDeviceToDevice, c->stream));
            else GEMB_CUDA(cudaMemsetAsync(Q[oc].get(), 0, chunk_bytes, c->stream));
        }
        std::fill(T.begin(), T.end(), 0.0);
        for (int q = 0; q < nk; q++) T[(size_t)q * mt + q] = theta[order[q]];
        m = nk;
    }
    return GEMB_OK;
}

// ---- 'SVD error (low rank)' of hope.py:38-40
__global__ void split_halves_kernel(int64_t n, int d, const float *__restrict__ X, float *__restrict__ L, float *__restrict__ Rr) {
    const int k = d / 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * d; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / d;
        const int cc = (int)(i - r * d);
        if (cc < k) L[r * k + cc] = X[i]; else Rr[r * k + (cc - k)] = X[i];
    }
}
// Z (n x w): identity columns p0 .. p0+w-1 (exact mode) or Rademacher +-1 (probe mode)
__global__ void probe_block_kernel(int64_t n, int w, int64_t p0, int probe, uint64_t seed, float *__restrict__ Z) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * w; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / w;
        const int cc = (int)(i - r * w);
        float v;
        if (probe) {
            uint64_t h = seed ^ ((uint64_t)r * 0x9E3779B97F4A7C15ull) ^ ((uint64_t)(p0 + cc) * 0xBF58476D1CE4E5B9ull);
            h ^= h >> 31; h *= 0x94D049BB133111EBull; h ^= h >> 29;
            v = (h & 1) ? 1.f : -1.f;
        } else v = (r == p0 + cc) ? 1.f : 0.f;
        Z[i] = v;
    }
}

}  // namespace gemb

using namespace gemb;

extern "C" int gemb_hope_svd_error(gemb_graph *g, int d, float beta, const float *X, int n_probe, uint64_t seed,
                                   double *err_out) {
    GEMB_ARG(g && X && err_out, "graph/X/err_out");
    GEMB_ARG(d >= 2 && d % 2 == 0, "d must be even");
    gemb_ctx *c = g->ctx;
    GEMB_ARG(c->nranks == 1 && g->n_local == g->n, "gemb_hope_svd_error is single-GPU");
    GEMB_CUDA(cudaSetDevice(c->device));
    const int64_t n = g->n;
    const int k = d / 2;
    const bool probe = n_probe > 0;
    const int w = (int)std::min<int64_t>(64, probe ? ((n_probe + 3) / 4 * 4) : ((n + 3) / 4 * 4));   // panel width
    HopeWork W;
    W.g = g; W.c = c; W.b = w; W.rows = n; W.shard = n;
    GEMB_TRY(W.alloc_blocks((size_t)n * w));
    GEMB_CUDA(W.scal.alloc(w + 8));
    GEMB_CUDA(W.G.alloc((size_t)k * w));
    GEMB_CUDA(W.M1.alloc((size_t)k * w));
    DeviceBuffer<float> Xd, L, Rr;
    GEMB_CUDA(Xd.alloc((size_t)n * d));
    GEMB_CUDA(L.alloc((size_t)n * k));
    GEMB_CUDA(Rr.alloc((size_t)n * k));
    GEMB_CUDA(cudaMemcpyAsync(Xd.get(), X, sizeof(float) * (size_t)n * d, cudaMemcpyHostToDevice, c->stream));
    split_halves_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(n, d, Xd.get(), L.get(), Rr.get());
    GEMB_CUDA(cudaGetLastError());
    count_launch();
    c->t_spmm.reset(); c->t_dense.reset(); c->t_comm.reset();
    double nrm = 0.0;
    int J = 0;
    GEMB_TRY(general_katz_terms(W, beta, 1e-9, seed ? seed : 1, !g->symmetric, &nrm, &J));
    GEMB_TRY(clear_scratch(W));
    float *Z = W.buf[0], *SZ = W.buf[1], *LZ = W.buf[2];
    const int64_t total_cols = probe ? n_probe : n;
    double acc = 0.0;
    std::vector<double> rs(w);
    const int threads = (256 / w) * w > 0 ? (256 / w) * w : w;
    for (int64_t p0 = 0; p0 < total_cols; p0 += w) {
        const int live = (int)std::min<int64_t>(w, total_cols - p0);
        probe_block_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(n, w, p0, probe ? 1 : 0, seed, Z);
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        GEMB_TRY(katz(W, false, beta, J, Z, SZ, W.buf[3], W.buf[4]));             // S Z
        GEMB_TRY(gram_launch(c, n, Rr.get(), k, Z, w, W.G.get()));                            // X2^T Z   (k x w, fp64)
        f64_to_f32_kernel<<<(k * w + 255) / 256, 256, 0, c->stream>>>(k * w, W.G.get(), W.M1.get());
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        GEMB_TRY(apply_launch(c, n, L.get(), k, W.M1.get(), w, w, LZ, w));                    // X1 (X2^T Z)
        GEMB_CUDA(cudaMemsetAsync(W.scal.get(), 0, sizeof(double) * w, c->stream));
        coldiff_sumsq_kernel<<<c->sm_count * 4, threads, 0, c->stream>>>(n, w, LZ, SZ, W.scal.get());
        GEMB_CUDA(cudaGetLastError());
        count_launch();
        GEMB_TRY(copy_sync(c, rs.data(), W.scal.get(), sizeof(double) * w, cudaMemcpyDeviceToHost));
        for (int j = 0; j < live; j++) acc += rs[j];
    }
    *err_out = sqrt(probe ? acc / (double)n_probe : acc);
    return GEMB_OK;
}

extern "C" int gemb_hope(gemb_graph *g, int d, float beta, const gemb_hope_opts *uo, float *X_out,
                         float *sigma_out, gemb_hope_stats *stats) {
    GEMB_ARG(g != nullptr, "graph");
    GEMB_ARG(d >= 1, "d must be >= 1");
    GEMB_ARG((uo && uo->struct_size == sizeof(gemb_hope_opts) && (uo->spectral_mode == 1 || uo->spectral_mode == 2)) || d % 2 == 0,
             "d must be even (k = d/2 singular triplets)");
    GEMB_ARG(!stats || stats->struct_size == sizeof(gemb_hope_stats), "stats.struct_size");
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    GEMB_ARG(!(uo && uo->struct_size == sizeof(gemb_hope_opts) && uo->spectral_mode == 2) || c->nranks == 1,
             "spectral_mode 2 (the composite operator -M^T M) is single-GPU: use a context without a multi-GPU communicator");
    GEMB_ARG(!(uo && uo->struct_size == sizeof(gemb_hope_opts) && uo->spectral_mode >= 3 && uo->spectral_mode <= 5) ||
                 c->nranks == 1,
             "spectral_modes 3-5 (common neighbours, Adamic-Adar, rooted PageRank) are single-GPU: use a context without a "
             "multi-GPU communicator");
    GEMB_ARG(!(c->nranks > 1 && g->replicated), "multi-GPU HOPE needs row shards (upload rows [rank*ceil(n/P), ...))");
    Opts o;
    if (uo) {
        GEMB_ARG(uo->struct_size == sizeof(gemb_hope_opts), "opts.struct_size");
        if (uo->oversample >= 0) o.oversample = uo->oversample;
        if (uo->max_iters > 0) o.max_iters = uo->max_iters;
        if (uo->min_iters > 0) o.min_iters = uo->min_iters;
        if (uo->tol > 0) o.tol = uo->tol;
        if (uo->katz_terms > 0) o.katz_terms = uo->katz_terms;
        if (uo->katz_tol > 0) o.katz_tol = uo->katz_tol;
        if (uo->seed) o.seed = uo->seed;
        o.compute_residual = uo->compute_residual;
        o.verbose = uo->verbose;
        GEMB_ARG(uo->algorithm >= 0 && uo->algorithm <= 3, "opts.algorithm");
        o.algorithm = uo->algorithm;
        if (uo->cheb_degree >= 2) o.cheb_degree = uo->cheb_degree;
        if (uo->cheb_range_log2 > 0.f) o.range_log2 = uo->cheb_range_log2;
        GEMB_ARG(uo->stop_rule == 0 || uo->stop_rule == 1, "opts.stop_rule");
        o.stop_rule = uo->stop_rule;
        if (uo->algorithm3_basis > 0) o.lanczos_basis = uo->algorithm3_basis;
        GEMB_ARG(uo->spectral_mode >= 0 && uo->spectral_mode <= 5, "opts.spectral_mode");
        o.spectral_mode = uo->spectral_mode;
    }
    if (o.spectral_mode == 1) {
        GEMB_ARG(g->symmetric, "spectral_mode 1 (largest algebraic eigenpairs) needs a symmetric upload");
        GEMB_ARG(o.algorithm == 0 || o.algorithm == 2, "spectral_mode 1 runs on the Chebyshev-filtered subspace iteration (algorithm 0 or 2)");
        o.algorithm = 2;
        beta = 0.f;                 // unused: the ranking is by the eigenvalue itself
    }
    if (o.spectral_mode == 2) {
        // The wanted end of -M^T M (sigma^2 ~ 1e-2) is a sliver of a spectrum ||M||_2^2 wide (1246 on R-MAT 20's largest
        // component): per degree the filter gains ~1 + (m a)^2 / 2 at low degree m, exponentially only at high degree.
        // Degree 8 there stopped on the change rule with sigma^2 20x too large; degree 64 reaches an fp64 residual of
        // 2e-5 (DESIGN 5f).  The dynamic-range cap below still bounds it.
        if (!(uo->cheb_degree >= 2)) o.cheb_degree = 64;
        GEMB_ARG(!g->symmetric, "spectral_mode 2 needs A = D^-1 W uploaded together with its transpose (indptr_t, "
                                "indices_t, data_t): M^T M is applied as a sweep of A and a sweep of A^T");
        GEMB_ARG(o.algorithm == 0 || o.algorithm == 2, "spectral_mode 2 runs on the Chebyshev-filtered subspace iteration (algorithm 0 or 2)");
        o.algorithm = 2;
        beta = 0.f;
    }
    if (o.spectral_mode >= 3) {
        GEMB_ARG(o.algorithm <= 1, "spectral_modes 3-5 run on the general solver (algorithm 0 or 1): S is not a function "
                                   "of a symmetric A");
        o.algorithm = 1;
        if (o.spectral_mode == 5) GEMB_ARG(beta > 0.f && beta < 1.f, "spectral_mode 5 takes alpha in beta: 0 < alpha < 1");
        else beta = 0.f;            // unused: S = A A or A D A has no coefficient
    }
    if (o.algorithm >= 2 && !g->symmetric && o.spectral_mode != 2) {
        set_error("algorithm=%d (works on A itself, S = f(A)) needs a symmetric shard (upload with indptr_t = NULL)", o.algorithm);
        return GEMB_ERR_ARG;
    }
    const int algo = o.algorithm ? o.algorithm : (g->symmetric ? 2 : 1);
    const int k = (o.spectral_mode == 1 || o.spectral_mode == 2) ? d : d / 2;
    GEMB_ARG((int64_t)k <= g->n, "d/2 must not exceed the number of nodes");
    int64_t bb = std::min<int64_t>(g->n, (int64_t)k + o.oversample);
    int b = (int)((bb + 3) / 4 * 4);
    GEMB_ARG(b <= 1024, "block width d/2 + oversample must be <= 1024");

    static const bool trace = getenv("GEMB_TRACE") != nullptr;   // host wall clock of the call's stages, to stderr
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_enter = now();
    HopeWork W;
    W.g = g; W.c = c; W.b = b; W.rows = g->n_local; W.shard = g->n_shard;
    W.mode = o.spectral_mode;
    // multi-GPU, symmetric shard: needed-rows-only exchange over peer memory (halo.cu) unless GEMB_MG=allgather or
    // CUDA IPC is not available on this box (then every rank falls back to the all-gather form together)
    static const bool mg_allgather = getenv("GEMB_MG") && !strcmp(getenv("GEMB_MG"), "allgather");
    if (c->nranks > 1 && algo >= 2 && !mg_allgather) {
        int hs = halo_build(g);
        if (hs == GEMB_OK) hs = halo_buffers(g, 5, b);
        NcclApi *api = nccl_api();
        if (!api) return GEMB_ERR_NCCL;
        int hflag = (hs == GEMB_OK) ? 1 : 0;
        DeviceBuffer<int> flag;
        GEMB_CUDA(flag.alloc(1));
        GEMB_CUDA(cudaMemcpyAsync(flag.get(), &hflag, sizeof(int), cudaMemcpyHostToDevice, c->stream));
        ncclResult_t r = api->AllReduce(flag.get(), flag.get(), 1, ncclInt, ncclMin, (ncclComm_t)c->comm, c->stream);
        GEMB_TRY(copy_sync(c, &hflag, flag.get(), sizeof(int), cudaMemcpyDeviceToHost));
        if (r != ncclSuccess) { set_error("ncclAllReduce(halo agreement): %s", api->GetErrorString(r)); return GEMB_ERR_NCCL; }
        W.halo = hflag == 1;
        if (!W.halo && o.verbose) fprintf(stderr, "[gemb_hope] halo exchange unavailable (%s); all-gather per sweep\n", gemb_last_error());
    }
    if (W.halo) {
        for (int i = 0; i < 5; i++) W.buf[i] = g->halo.buf[i];
        GEMB_TRY(halo_barrier(g));    // every rank's blocks are in place before the first push can arrive
    } else {
        GEMB_TRY(W.alloc_blocks((size_t)W.shard * b));
        if (c->nranks > 1) GEMB_CUDA(W.full.alloc((size_t)g->n_pad * b));
    }
    GEMB_CUDA(W.G.alloc(b * b));
    GEMB_CUDA(W.G2.alloc(b * b));
    GEMB_CUDA(W.Z.alloc(b * b));
    GEMB_CUDA(W.Zs.alloc(b * b));
    GEMB_CUDA(W.w.alloc(2 * b));                           // eigenvalues, then the stop rule's quadratic forms
    GEMB_CUDA(W.scal.alloc(b + 8));
    GEMB_CUDA(W.Minv.alloc(b * b));
    GEMB_CUDA(W.M1.alloc((size_t)b * std::max(b, d)));     // b x b maps; the symmetric solver's b x d extraction map
    GEMB_CUDA(W.M2.alloc(b * b));
    GEMB_CUDA(W.rank_dev.alloc(1));
    GEMB_CUDA(W.fork_join.create());
    if (W.mode == 2) {                                     // the sixth n x b block: T between the two sweeps
        GEMB_CUDA(W.opT.alloc((size_t)W.shard * b));
        GEMB_CUDA(cudaMemsetAsync(W.opT.get(), 0, sizeof(float) * (size_t)W.shard * b, c->stream));
    }

    c->t_spmm.reset(); c->t_dense.reset(); c->t_comm.reset(); c->t_misc.reset();
    const double t_alloc = now();
    CallEvents<2> ev;
    GEMB_CUDA(ev.create());
    GEMB_CUDA(cudaEventRecord(ev[0], c->stream));

    double nrm = 0.0, hard_bound = 0.0;
    int J = o.katz_terms;
    bool have_nrm = false, ritz_bound = false;
    if (beta < 0.f) {
        // beta given relative to the spectral radius: beta = |beta| / ||A||_2 (= rho(A) for the symmetric graphs of
        // BASELINE.json configs[3]: "beta = 0.5 / rho_hat"), ||A||_2 by power iteration on a width-4 block
        GEMB_TRY(estimate_norm2(W, o.seed, W.buf[3], W.buf[4], W.buf[2], &nrm));
        if (!(nrm > 0.0)) { set_error("beta < 0 asks for beta = |beta| / ||A||_2, but ||A||_2 = 0 (empty graph)"); return GEMB_ERR_ARG; }
        beta = (float)(-(double)beta / nrm);
        have_nrm = true;
        GEMB_TRY(clear_scratch(W));
    }
    bool need_power = (J <= 0 && algo == 1) && !have_nrm && W.mode < 3;
    if (W.mode >= 3) {
        // no norm estimate: modes 3 and 4 are two sweeps per application, and ||alpha P||_inf <= alpha bounds the rooted
        // PageRank series a priori
        bool nonneg = true;
        double pinf = 0.0;
        if (W.mode >= 4) {
            GEMB_TRY(rowsum_bound(W, &pinf, &nonneg));
            GEMB_ARG(nonneg, "spectral_modes 4 and 5 (Adamic-Adar, rooted PageRank) need non-negative weights");
        }
        if (W.mode == 4) GEMB_TRY(inv_degree(W));
        if (W.mode != 5) J = 0;     // no series: katz_terms is ignored and reported as 0
        if (W.mode == 5) {
            GEMB_ARG(pinf <= 1.0 + 1e-5, "spectral_mode 5 needs P = D_out^-1 A (every row sum <= 1)");
            if (J <= 0) J = std::max(1, std::min(4096, (int)ceil(log((double)o.katz_tol) / log((double)beta))));
        }
    } else if (W.mode == 2) {
        // the Perron-Frobenius shortcut (ritz_bound) does not apply to -M^T M: ||M||_2^2 by power iteration
        GEMB_TRY(estimate_composite_norm(W, o.seed, W.buf[3], W.buf[4], &nrm));
        if (!(nrm > 0.0)) nrm = 1.0;                       // M = 0: the spectrum is {0}, any positive bound holds it
        GEMB_TRY(clear_scratch(W));
    } else if (algo >= 2) {
        bool nonneg = false;
        GEMB_TRY(rowsum_bound(W, &hard_bound, &nonneg));
        if (nonneg && (double)beta * hard_bound * 1.02 < 1.0) ritz_bound = true;   // spectrum bounds from Ritz values
        else need_power = !have_nrm;
    }
    if (have_nrm && !ritz_bound) {
        if ((double)beta * nrm * 1.02 >= 1.0) { set_error("|beta| / ||A||_2 with |beta| >= 0.98: outside the Katz convergence radius"); return GEMB_ERR_DIVERGE; }
        if (J <= 0) J = katz_terms_for(beta, nrm, o.katz_tol);
        if (hard_bound <= 0.0) hard_bound = nrm;
    }
    if (need_power) {
        int Jg = 0;
        GEMB_TRY(general_katz_terms(W, beta, o.katz_tol, o.seed, algo == 1 && !W.halo, &nrm, &Jg));
        if (J <= 0) J = Jg;
        if (hard_bound <= 0.0) hard_bound = nrm;
        GEMB_TRY(clear_scratch(W));
    }

    HopeResult R;
    int s;
    // thick-restart Lanczos needs room for its basis (k + 16 kept + expansions); tiny graphs take the subspace solver
    const bool lanczos_fits = g->n >= 2048;
    // a priori spectrum bound: ||A||_inf for Lanczos; for Chebyshev see hope_symmetric
    const SpecMap lanczos_map(beta, true, hard_bound);
    SpecMap sym_map(beta, o.spectral_mode == 0, ritz_bound ? hard_bound : nrm);
    sym_map.estimated = !ritz_bound;                              // else ||A||_inf: a true bound
    sym_map.negdef = o.spectral_mode == 2;
    if (algo == 3 && lanczos_fits) s = hope_lanczos(W, o, d, lanczos_map, R);
    else if (algo >= 2) {
        s = hope_symmetric(W, o, d, sym_map, ritz_bound, R);
        if (s == GEMB_SWITCH_TO_LANCZOS) { R = HopeResult(); s = hope_lanczos(W, o, d, lanczos_map, R); }
    } else s = hope_general(W, o, d, beta, J, R);
    if (s != GEMB_OK) return s;

    GEMB_CUDA(cudaEventRecord(ev[1], c->stream));
    GEMB_CUDA(cudaEventSynchronize(ev[1]));
    if (W.halo) GEMB_TRY(halo_check_timeout(g));
    float total_ms = 0.f;
    GEMB_CUDA(cudaEventElapsedTime(&total_ms, ev[0], ev[1]));

    const double t_solve = now();
    double d2h_ms = 0.0;
    if (X_out || sigma_out) {
        CallEvents<2> d2h;
        GEMB_CUDA(d2h.create());
        GEMB_CUDA(cudaEventRecord(d2h[0], c->stream));
        if (X_out) GEMB_CUDA(cudaMemcpyAsync(X_out, R.Xd, sizeof(float) * (size_t)W.rows * d, cudaMemcpyDeviceToHost, c->stream));
        if (sigma_out) GEMB_CUDA(cudaMemcpyAsync(sigma_out, R.sig_dev, sizeof(float) * k, cudaMemcpyDeviceToHost, c->stream));
        GEMB_CUDA(cudaEventRecord(d2h[1], c->stream));
        GEMB_CUDA(cudaEventSynchronize(d2h[1]));
        d2h_ms = d2h.ms(0, 1);
    }
    if (trace)
        fprintf(stderr, "[gemb_hope] host ms: alloc %.2f  solve %.2f (device %.2f)  d2h %.2f (device %.2f)\n",
                t_alloc - t_enter, t_solve - t_alloc, total_ms, now() - t_solve, d2h_ms);

    if (stats) {
        stats->iters = R.iters;
        stats->katz_terms = R.katz_terms;
        stats->block = b;
        stats->converged = R.converged;
        stats->algorithm = R.algorithm;
        stats->spmm_count = W.spmm_wide;   /* block-width sweeps (norm estimation excluded) */
        stats->spmm_ms = c->t_spmm.total_ms();
        const double nnz = (double)g->A.nnz;
        // compulsory bytes of one sweep on THIS rank: CSR + every referenced X row once + Y rows once.  Single GPU:
        // all n rows; halo mode: the shard's own rows + the distinct remote rows it references (+ the rows it stores
        // into the peers); all-gather mode: the shard's rows + the halo it would have needed (the gathered rest is not
        // compulsory and is not counted -- round 1 counted the whole gathered block here).
        double x_rows = (double)g->n;
        if (c->nranks > 1) x_rows = (double)W.rows + (W.halo ? (double)g->halo.halo_rows : 0.0);
        stats->spmm_bytes = (g->A.data ? 8.0 : 4.0) * nnz + 4.0 * (double)(W.rows + 1) +
                            4.0 * (double)b * (x_rows + (double)W.rows);
        stats->halo_rows = W.halo ? g->halo.halo_rows : 0;
        stats->push_rows = W.halo ? g->halo.push_total : 0;
        stats->pushes = W.pushes;
        stats->mg_mode = c->nranks == 1 ? 0 : (W.halo ? 2 : 1);
        stats->push_bytes = W.halo ? W.push_bytes_per_row * (double)g->halo.push_total : 0.0;
        stats->resid_est = R.resid_est;
        stats->dense_ms = c->t_dense.total_ms();
        stats->comm_ms = c->t_comm.total_ms();
        stats->total_ms = total_ms;
        stats->h2d_ms = 0.0;
        stats->d2h_ms = d2h_ms;
        /* ||A||_inf when no power iteration ran; else the power-iteration estimate, raised to the largest |Ritz value| */
        stats->norm2_A = (float)(ritz_bound ? hard_bound : std::max(nrm, R.norm));
        stats->beta_used = beta;
        stats->ritz_change = (float)R.change;
        stats->resid_max = R.resid_max;
    }
    return GEMB_OK;
}
