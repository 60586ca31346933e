// gem_b200/csrc/nc.cu -- node classification: one-vs-rest logistic regression on an embedding, and the top-k label
// prediction of upstream GEM's evaluateNodeClassification (its TopKRanker over sklearn's
// OneVsRestClassifier(LogisticRegression())).
//
// Fit.  For every label c, with s_i = +1 when row i carries c and -1 otherwise, the unique minimiser of
//     f_c(w, b) = 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w . x_i + b)))          (the intercept is not penalised)
// The labels are solved in panels of P <= 128 (the accumulator width of apply_tc / gram_tc), each panel a batch of
// independent binary problems.  One function / gradient evaluation of a panel is four launches:
//     Z = X W                 apply_launch  (n x d times d x P, fp32 out; 3xTF32 wgmma when the shape fits)
//     nc_residual_kernel      z = Z + b (fp64); R = sigma(z) - y written over Z; per-class loss and sum R, per-block
//                             partials added in a fixed order (sum_partials_launch)
//     G = X^T R               gram_launch   (d x P, fp64 out)
//     nc_step_kernel          one CTA per class: f, grad = (w + C G, C sum R), then one step of the class's L-BFGS
//                             state machine (memory NC_M, per-class line search, converged mask), and the next trial
//                             point written into the fp32 W panel and the fp64 bias
// The host reads back the P status flags after each evaluation (the loop's only round trip) and stops the panel when
// no class is running.  Memory: n x P floats for Z / R, plus the per-class L-BFGS history, for any number of labels.
// No floating-point atomics anywhere: two runs give the same bits.
//
// Line search.  The loss comes from fp32 products, so near the optimum f differences drown in rounding while the
// gradient (and with it phi'(a) = grad(x + a p) . p) stays accurate.  A trial step is accepted when Armijo holds on f
// OR phi'(a) <= 0 (f is convex along p, so it decreased up to that point).  Otherwise the step is shrunk to the secant
// root of phi' (a phi'(0) / (phi'(0) - phi'(a))), kept inside [0.1 a, 0.9 a].
//
// Predict.  nc_topk_kernel: one warp per test row picks its k labels with the largest p = 1 / (1 + exp(-z)) (fp64 from
// the decision value), exact ties to the larger label index, in k arg-max passes over the row's L decision values.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace gemb {

constexpr int NC_PANEL = 128;   // labels per panel: the widest accumulator of apply_tc / gram_tc
constexpr int NC_M = 10;        // L-BFGS memory (sklearn's lbfgs: scipy L-BFGS-B with m = 10)
constexpr int NC_MAX_BACKTRACK = 40;
enum NcStatus { NC_RUNNING = 0, NC_CONVERGED = 1, NC_CONSTANT = 2, NC_MAXITER = 3, NC_STALLED = 4 };

// ------------------------------------------------------------------------------------------------ residual
// One warp per row (grid-stride), lane l owns columns 4l .. 4l+3 of the panel.  part[blk * 2P + c] = loss of class c over
// the block's rows, part[blk * 2P + P + c] = sum of R; the eight warps' sums are added in warp order.
__global__ void __launch_bounds__(256) nc_residual_kernel(int64_t n, int P, int c0, const int64_t *__restrict__ indptr,
                                                          const int32_t *__restrict__ labels, const double *__restrict__ bias,
                                                          float *__restrict__ Z, double *__restrict__ part) {
    __shared__ double s_red[8][2 * NC_PANEL];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col = 4 * lane;
    const bool own = col < P;
    double b[4], loss[4] = {0, 0, 0, 0}, rsum[4] = {0, 0, 0, 0};
#pragma unroll
    for (int q = 0; q < 4; q++) b[q] = own ? bias[col + q] : 0.0;
    const int64_t nw = (int64_t)gridDim.x * 8;
    for (int64_t i = (int64_t)blockIdx.x * 8 + warp; i < n; i += nw) {
        int y = 0;                                        // bit q: row i carries label c0 + col + q
        for (int64_t e = indptr[i]; e < indptr[i + 1]; e++) {
            const int rel = labels[e] - c0 - col;
            if (rel >= 0 && rel < 4) y |= 1 << rel;
        }
        if (!own) continue;
        float4 *zp = (float4 *)(Z + i * P + col);
        const float4 zv = *zp;
        const float zf[4] = {zv.x, zv.y, zv.z, zv.w};
        float r[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const double z = (double)zf[q] + b[q];
            const bool pos = (y >> q) & 1;
            const double t = pos ? z : -z;               // s z
            // log(1 + exp(-t)) and sigma(z), overflow-free
            const double e = exp(-fabs(t));
            loss[q] += (t > 0 ? 0.0 : -t) + log1p(e);
            const double sig = z >= 0 ? 1.0 / (1.0 + exp(-z)) : exp(z) / (1.0 + exp(z));
            const double rr = sig - (pos ? 1.0 : 0.0);
            rsum[q] += rr;
            r[q] = (float)rr;
        }
        *zp = make_float4(r[0], r[1], r[2], r[3]);
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        if (own && col + q < P) { s_red[warp][col + q] = loss[q]; s_red[warp][P + col + q] = rsum[q]; }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < 2 * P; t += blockDim.x) {
        double s = 0.0;
        for (int w = 0; w < 8; w++) s += s_red[w][t];
        part[(size_t)blockIdx.x * 2 * P + t] = s;
    }
}

// ------------------------------------------------------------------------------------------------ L-BFGS step
struct NcState {
    int D1, P;               // d + 1, panel width
    double *x, *g, *gt, *xt, *p;          // P x D1 each: iterate, its gradient, trial gradient, trial point, direction
    double *S, *Y;                        // NC_M x P x D1: the stored pairs (ring, newest at head - 1)
    double *rho;                          // NC_M x P
    double *f, *alpha, *dphi0, *g0n, *gamma;   // P each
    int *iters, *status, *phase, *nhist, *head, *nback;
};

// sum over the block (256 threads) in a fixed order; every thread gets the same bits
__device__ __forceinline__ double nc_block_sum(double v, double *red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < 8; w++) t += red[w];
    return t;
}
__device__ __forceinline__ double nc_block_max(double v, double *red) {
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < 8; w++) t = fmax(t, red[w]);
    return t;
}

// One CTA per class c of the panel.  G: d x P (fp64, row-major) = X^T R at the trial point; sums: loss[P] | sum R[P].
// Writes the next trial point into Wf (d x P fp32, column c) and bias[c].
// The class's scalar state is read into registers once, before any thread can store, and kept in step by every thread
// (each decision rests on block sums that give every thread the same bits), so all threads take the same branches
// through the barriers of nc_block_sum.  Thread 0 stores the scalars back after the last barrier.
__global__ void __launch_bounds__(256) nc_step_kernel(NcState st, int d, double C, double tol, int max_iter,
                                                      const double *__restrict__ G, const double *__restrict__ sums,
                                                      float *__restrict__ Wf, double *__restrict__ bias) {
    __shared__ double red[8];
    __shared__ double s_a[NC_M];
    const int c = blockIdx.x, tid = threadIdx.x;
    if (st.status[c] != NC_RUNNING) return;
    const int D1 = st.D1, P = st.P;
    const size_t o = (size_t)c * D1;
    double *x = st.x + o, *g = st.g + o, *gt = st.gt + o, *xt = st.xt + o, *p = st.p + o;
    const int phase = st.phase[c];
    double f = st.f[c], alpha = st.alpha[c], dphi0 = st.dphi0[c], g0n = st.g0n[c], gamma = st.gamma[c];
    int iters = st.iters[c], nback = st.nback[c], head = st.head[c], nhist = st.nhist[c];
    double rho_new = 0.0;                        // 1 / s.y of a pair stored in this step (0: none)
    // f and the gradient at the trial point
    double ww = 0.0;
    for (int k = tid; k < D1; k += 256) {
        if (k < d) { gt[k] = xt[k] + C * G[(size_t)k * P + c]; ww += xt[k] * xt[k]; }
        else gt[k] = C * sums[P + c];
    }
    const double ft = 0.5 * nc_block_sum(ww, red) + C * sums[c];
    bool new_dir = false;
    int status = NC_RUNNING;
    if (phase == 0) {                            // the start point w = 0, b = 0
        double gm = 0.0;
        for (int k = tid; k < D1; k += 256) { x[k] = xt[k]; g[k] = gt[k]; gm = fmax(gm, fabs(gt[k])); }
        gm = nc_block_max(gm, red);
        f = ft; g0n = gm;
        if (gm == 0.0) status = NC_CONVERGED;
        else if (max_iter <= 0) status = NC_MAXITER;
        else new_dir = true;
    } else {
        double dp = 0.0;
        for (int k = tid; k < D1; k += 256) dp += gt[k] * p[k];
        const double dphit = nc_block_sum(dp, red);
        if (ft <= f + 1e-4 * alpha * dphi0 || dphit <= 0.0) {
            // accept: store the pair (s, y) = (xt - x, gt - g), move to the trial point
            double *S = st.S + ((size_t)head * P + c) * D1, *Y = st.Y + ((size_t)head * P + c) * D1;
            double sy = 0.0, yy = 0.0, gm = 0.0;
            for (int k = tid; k < D1; k += 256) {
                const double s = xt[k] - x[k], y = gt[k] - g[k];
                S[k] = s; Y[k] = y;
                sy += s * y; yy += y * y;
                x[k] = xt[k]; g[k] = gt[k];
                gm = fmax(gm, fabs(gt[k]));
            }
            sy = nc_block_sum(sy, red);
            yy = nc_block_sum(yy, red);
            gm = nc_block_max(gm, red);
            f = ft; iters++; nback = 0;
            if (sy > 0.0 && yy > 0.0) {              // strictly convex f: always, unless the step underflowed
                rho_new = 1.0 / sy;
                gamma = sy / yy;
                head = (head + 1) % NC_M;
                nhist = min(nhist + 1, NC_M);
            }
            if (gm <= tol * g0n) status = NC_CONVERGED;
            else if (iters >= max_iter) status = NC_MAXITER;
            else new_dir = true;
        } else if (++nback > NC_MAX_BACKTRACK) {
            double gm = 0.0;
            for (int k = tid; k < D1; k += 256) gm = fmax(gm, fabs(g[k]));
            gm = nc_block_max(gm, red);
            status = gm <= tol * g0n ? NC_CONVERGED : NC_STALLED;
        } else {
            alpha *= fmin(fmax(dphi0 / (dphi0 - dphit), 0.1), 0.9);
        }
    }
    __syncthreads();
    if (rho_new != 0.0 && tid == 0) st.rho[(size_t)((head - 1 + NC_M) % NC_M) * P + c] = rho_new;
    __syncthreads();
    if (new_dir) {
        // two-loop recursion: p = -H g with H0 = gamma I (first step: p = -g, alpha = 1 / |g|_2)
        const int nh = nhist, h0 = head;
        for (int k = tid; k < D1; k += 256) p[k] = g[k];
        for (int j = 0; j < nh; j++) {
            const int h = (h0 - 1 - j + NC_M) % NC_M;
            const double *S = st.S + ((size_t)h * P + c) * D1, *Y = st.Y + ((size_t)h * P + c) * D1;
            double v = 0.0;
            for (int k = tid; k < D1; k += 256) v += S[k] * p[k];
            const double a = st.rho[(size_t)h * P + c] * nc_block_sum(v, red);
            if (tid == 0) s_a[j] = a;
            for (int k = tid; k < D1; k += 256) p[k] -= a * Y[k];
        }
        const double gam = nh > 0 ? gamma : 1.0;
        for (int k = tid; k < D1; k += 256) p[k] *= gam;
        __syncthreads();
        for (int j = nh - 1; j >= 0; j--) {
            const int h = (h0 - 1 - j + NC_M) % NC_M;
            const double *S = st.S + ((size_t)h * P + c) * D1, *Y = st.Y + ((size_t)h * P + c) * D1;
            double v = 0.0;
            for (int k = tid; k < D1; k += 256) v += Y[k] * p[k];
            const double bb = st.rho[(size_t)h * P + c] * nc_block_sum(v, red);
            for (int k = tid; k < D1; k += 256) p[k] += (s_a[j] - bb) * S[k];
        }
        double gp = 0.0, gg = 0.0;
        for (int k = tid; k < D1; k += 256) { p[k] = -p[k]; gp += g[k] * p[k]; gg += g[k] * g[k]; }
        gp = nc_block_sum(gp, red);
        gg = nc_block_sum(gg, red);
        if (!(gp < 0.0)) {                       // not a descent direction (rounding): drop the history, steepest descent
            for (int k = tid; k < D1; k += 256) p[k] = -g[k];
            gp = -gg;
            nhist = 0; head = 0;
        }
        alpha = nh > 0 ? 1.0 : 1.0 / sqrt(gg);
        dphi0 = gp;
    }
    __syncthreads();
    if (tid == 0) {
        st.phase[c] = 1; st.f[c] = f; st.alpha[c] = alpha; st.dphi0[c] = dphi0; st.g0n[c] = g0n; st.gamma[c] = gamma;
        st.iters[c] = iters; st.nback[c] = nback; st.head[c] = head; st.nhist[c] = nhist; st.status[c] = status;
    }
    if (status != NC_RUNNING) return;
    for (int k = tid; k < D1; k += 256) {
        const double v = x[k] + alpha * p[k];
        xt[k] = v;
        if (k < d) Wf[(size_t)k * P + c] = (float)v;
        else bias[c] = v;
    }
}

// status: NC_CONSTANT for padded columns and labels that are constant on the training rows, NC_RUNNING otherwise;
// x = xt = 0, W panel and bias 0
__global__ void nc_init_kernel(NcState st, int d, const int *__restrict__ init_status, float *__restrict__ Wf,
                               double *__restrict__ bias) {
    const int P = st.P, D1 = st.D1;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t)P * D1; t += (int64_t)gridDim.x * blockDim.x) {
        st.x[t] = 0.0; st.xt[t] = 0.0;
        const int c = (int)(t / D1), k = (int)(t % D1);
        if (k < d) Wf[(size_t)k * P + c] = 0.f;
        if (k == 0) {
            bias[c] = 0.0;
            st.status[c] = init_status[c];
            st.iters[c] = 0; st.phase[c] = 0; st.nhist[c] = 0; st.head[c] = 0; st.nback[c] = 0;
            st.f[c] = 0.0; st.alpha[c] = 0.0; st.dphi0[c] = 0.0; st.g0n[c] = 0.0; st.gamma[c] = 1.0;
        }
    }
}

// ------------------------------------------------------------------------------------------------ top-k
// (p, c) ranks above (q, e) when p > q, or p == q and c > e  (argsort(kind='stable')[-k:]: ties to the larger index)
__device__ __forceinline__ bool nc_above(double p, int c, double q, int e) { return p > q || (p == q && c > e); }

// One warp per row of the chunk: k = koff[i + 1] - koff[i] passes, each taking the highest-ranked label below the
// previous pick.  Z: rows x ldz decision values without the intercept.
__global__ void __launch_bounds__(256) nc_topk_kernel(int64_t rows, int64_t row0, int L, int ldz, const float *__restrict__ Z,
                                                      const double *__restrict__ bias, const int64_t *__restrict__ koff,
                                                      int32_t *__restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t nw = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < rows; i += nw) {
        const int64_t o0 = koff[row0 + i], k = koff[row0 + i + 1] - o0;
        double prev_p = 2.0;          // above every probability
        int prev_c = 0;
        const float *z = Z + i * ldz;
        for (int64_t t = 0; t < k; t++) {
            double bp = -1.0;
            int bc = -1;
            for (int c = lane; c < L; c += 32) {
                const double pc = 1.0 / (1.0 + exp(-((double)z[c] + bias[c])));
                if (nc_above(prev_p, prev_c, pc, c) && nc_above(pc, c, bp, bc)) { bp = pc; bc = c; }
            }
            for (int s = 16; s > 0; s >>= 1) {
                const double op = __shfl_xor_sync(0xffffffffu, bp, s);
                const int oc = __shfl_xor_sync(0xffffffffu, bc, s);
                if (nc_above(op, oc, bp, bc)) { bp = op; bc = oc; }
            }
            if (lane == 0) out[o0 + t] = bc;
            prev_p = bp; prev_c = bc;
        }
    }
}

}  // namespace gemb

using namespace gemb;

extern "C" int gemb_nc_fit(gemb_ctx *ctx, int64_t n, int d, const float *X, const int64_t *indptr, const int32_t *labels,
                           int L, double C, double tol, int max_iter, double *W_out, int32_t *iters_out,
                           int32_t *status_out, gemb_nc_stats *stats) {
    GEMB_ARG(ctx && X && indptr && W_out && n > 0 && d > 0 && L > 0, "ctx/X/indptr/W_out/n/d/L");
    GEMB_ARG(C > 0 && tol >= 0 && max_iter >= 0, "C > 0, tol >= 0, max_iter >= 0");
    GEMB_ARG(!stats || stats->struct_size == sizeof(gemb_nc_stats), "stats->struct_size");
    const int64_t nnz = indptr[n];
    GEMB_ARG(indptr[0] == 0 && nnz >= 0 && (nnz == 0 || labels), "indptr[0] == 0, labels");
    // positives per label; the rows' label ids must be strictly ascending and in [0, L)
    std::vector<int64_t> npos(L, 0);
    for (int64_t i = 0; i < n; i++) {
        GEMB_ARG(indptr[i + 1] >= indptr[i], "indptr non-decreasing");
        for (int64_t e = indptr[i]; e < indptr[i + 1]; e++) {
            GEMB_ARG(labels[e] >= 0 && labels[e] < L, "label id in [0, L)");
            GEMB_ARG(e == indptr[i] || labels[e] > labels[e - 1], "label ids strictly ascending per row");
            npos[labels[e]]++;
        }
    }
    GEMB_CUDA(cudaSetDevice(ctx->device));
    const int D1 = d + 1;
    CallEvents<2> ev;
    GEMB_CUDA(ev.create());
    GEMB_CUDA(cudaEventRecord(ev[0], ctx->stream));
    DeviceBuffer<float> dX, dZ, dWf;
    DeviceBuffer<int64_t> dIndptr;
    DeviceBuffer<int32_t> dLab;
    DeviceBuffer<double> dG, dSums, dBias, dVec, dHist, dScal;
    DeviceBuffer<int> dInts;
    const int PM = NC_PANEL;
    GEMB_CUDA(dX.upload(X, (size_t)n * d, ctx->stream));
    GEMB_CUDA(dIndptr.upload(indptr, n + 1, ctx->stream));
    GEMB_CUDA(dLab.upload(labels, nnz, ctx->stream));
    GEMB_CUDA(dZ.alloc((size_t)n * PM));
    GEMB_CUDA(dWf.alloc((size_t)d * PM));
    GEMB_CUDA(dG.alloc((size_t)d * PM));
    GEMB_CUDA(dSums.alloc(2 * PM));
    GEMB_CUDA(dBias.alloc(PM));
    GEMB_CUDA(dVec.alloc((size_t)5 * PM * D1));
    GEMB_CUDA(dHist.alloc((size_t)2 * NC_M * PM * D1 + (size_t)NC_M * PM));
    GEMB_CUDA(dScal.alloc((size_t)5 * PM));
    GEMB_CUDA(dInts.alloc((size_t)7 * PM));
    const int grid_res = grid_stride(ctx, n, 8, 8);
    std::vector<int> init(PM), status(PM), iters(PM);
    std::vector<double> xh((size_t)PM * D1);
    int64_t evals = 0, unconverged = 0, constant = 0;
    int max_it = 0;
    double bytes = 0.0;
    for (int c0 = 0; c0 < L; c0 += PM) {
        const int nc = std::min(PM, L - c0), P = (nc + 3) / 4 * 4;   // padded columns: constant, never written out
        NcState st;
        st.D1 = D1; st.P = P;
        double *v = dVec.get();
        st.x = v; st.g = v + (size_t)P * D1; st.gt = v + (size_t)2 * P * D1; st.xt = v + (size_t)3 * P * D1; st.p = v + (size_t)4 * P * D1;
        st.S = dHist.get(); st.Y = st.S + (size_t)NC_M * P * D1; st.rho = st.Y + (size_t)NC_M * P * D1;
        double *s = dScal.get();
        st.f = s; st.alpha = s + P; st.dphi0 = s + 2 * P; st.g0n = s + 3 * P; st.gamma = s + 4 * P;
        int *ii = dInts.get();
        st.iters = ii; st.status = ii + P; st.phase = ii + 2 * P; st.nhist = ii + 3 * P; st.head = ii + 4 * P; st.nback = ii + 5 * P;
        int *d_init = ii + 6 * P;
        for (int c = 0; c < P; c++)
            init[c] = (c >= nc || npos[c0 + c] == 0 || npos[c0 + c] == n) ? NC_CONSTANT : NC_RUNNING;
        GEMB_CUDA(cudaMemcpyAsync(d_init, init.data(), sizeof(int) * P, cudaMemcpyHostToDevice, ctx->stream));
        GEMB_TRY(launch(ctx, nc_init_kernel, grid_stride(ctx, (int64_t)P * D1, 256, 8), 256, 0, st, d, d_init, dWf.get(),
                        dBias.get()));
        bool running = std::count(init.begin(), init.begin() + P, (int)NC_RUNNING) > 0;
        while (running) {
            GEMB_TRY(apply_launch(ctx, n, dX.get(), d, dWf.get(), P, P, dZ.get(), P));
            double *part = nullptr;
            GEMB_TRY(red_scratch(ctx, (size_t)grid_res * 2 * P, &part));
            GEMB_TRY(launch(ctx, nc_residual_kernel, grid_res, 256, 0, n, P, c0, dIndptr.get(), dLab.get(), dBias.get(), dZ.get(),
                            part));
            GEMB_TRY(sum_partials_launch(ctx, grid_res, 2 * P, part, dSums.get()));
            GEMB_TRY(gram_launch(ctx, n, dX.get(), d, dZ.get(), P, dG.get()));
            GEMB_TRY(launch(ctx, nc_step_kernel, P, 256, 0, st, d, C, tol, max_iter, dG.get(), dSums.get(), dWf.get(), dBias.get()));
            evals++;
            // compulsory bytes: apply (X in, Z out), residual (Z in, R out, labels), Gram (X and R in)
            bytes += (double)n * (8.0 * d + 16.0 * P + 8.0) + 4.0 * (double)nnz;
            GEMB_TRY(copy_sync(ctx, status.data(), st.status, sizeof(int) * P, cudaMemcpyDeviceToHost));
            running = std::count(status.begin(), status.begin() + P, (int)NC_RUNNING) > 0;
        }
        GEMB_CUDA(cudaMemcpyAsync(status.data(), st.status, sizeof(int) * P, cudaMemcpyDeviceToHost, ctx->stream));
        GEMB_CUDA(cudaMemcpyAsync(iters.data(), st.iters, sizeof(int) * P, cudaMemcpyDeviceToHost, ctx->stream));
        GEMB_CUDA(cudaMemcpyAsync(xh.data(), st.x, sizeof(double) * (size_t)P * D1, cudaMemcpyDeviceToHost, ctx->stream));
        GEMB_CUDA(cudaStreamSynchronize(ctx->stream));
        for (int c = 0; c < nc; c++) {
            double *w = W_out + (size_t)(c0 + c) * D1;
            if (status[c] == NC_CONSTANT) {       // sklearn's _ConstantPredictor: p = 0 or 1 for every row
                std::fill(w, w + d, 0.0);
                w[d] = npos[c0 + c] ? INFINITY : -INFINITY;
                constant++;
            } else {
                std::copy(xh.begin() + (size_t)c * D1, xh.begin() + (size_t)(c + 1) * D1, w);
                if (status[c] != NC_CONVERGED) unconverged++;
            }
            if (iters_out) iters_out[c0 + c] = iters[c];
            if (status_out) status_out[c0 + c] = status[c];
            max_it = std::max(max_it, iters[c]);
        }
    }
    GEMB_CUDA(cudaEventRecord(ev[1], ctx->stream));
    GEMB_CUDA(cudaEventSynchronize(ev[1]));
    if (stats) {
        stats->panels = (L + PM - 1) / PM;
        stats->evaluations = evals;
        stats->max_iters = max_it;
        stats->unconverged = unconverged;
        stats->constant = constant;
        stats->eval_bytes = bytes;
        stats->total_ms = ev.ms(0, 1);
    }
    return GEMB_OK;
}

extern "C" int gemb_nc_topk(gemb_ctx *ctx, int64_t m, int d, const float *X, int L, const double *W, const int64_t *koff,
                            int32_t *pred_out) {
    GEMB_ARG(ctx && X && W && koff && m > 0 && d > 0 && L > 0, "ctx/X/W/koff/m/d/L");
    GEMB_ARG(koff[0] == 0, "koff[0] == 0");
    for (int64_t i = 0; i < m; i++) GEMB_ARG(koff[i + 1] >= koff[i] && koff[i + 1] - koff[i] <= L, "0 <= k_i <= L");
    const int64_t total = koff[m];
    GEMB_ARG(total == 0 || pred_out, "pred_out");
    if (total == 0) return GEMB_OK;
    GEMB_CUDA(cudaSetDevice(ctx->device));
    const int D1 = d + 1, Lp = (L + 3) / 4 * 4;
    std::vector<float> wf((size_t)d * Lp, 0.f);
    std::vector<double> bias(Lp, 0.0);
    for (int c = 0; c < L; c++) {
        for (int k = 0; k < d; k++) wf[(size_t)k * Lp + c] = (float)W[(size_t)c * D1 + k];
        bias[c] = W[(size_t)c * D1 + d];
    }
    // test rows in chunks of at most 2^28 decision values (1 GiB)
    const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(m, ((int64_t)1 << 28) / Lp));
    DeviceBuffer<float> dX, dW, dZ;
    DeviceBuffer<double> dB;
    DeviceBuffer<int64_t> dK;
    DeviceBuffer<int32_t> dOut;
    GEMB_CUDA(dX.upload(X, (size_t)m * d, ctx->stream));
    GEMB_CUDA(dW.upload(wf.data(), wf.size(), ctx->stream));
    GEMB_CUDA(dB.upload(bias.data(), Lp, ctx->stream));
    GEMB_CUDA(dK.upload(koff, m + 1, ctx->stream));
    GEMB_CUDA(dOut.alloc(total));
    GEMB_CUDA(dZ.alloc((size_t)chunk * Lp));
    for (int64_t r0 = 0; r0 < m; r0 += chunk) {
        const int64_t rows = std::min(chunk, m - r0);
        GEMB_TRY(apply_launch(ctx, rows, dX.get() + (size_t)r0 * d, d, dW.get(), Lp, Lp, dZ.get(), Lp));
        GEMB_TRY(launch(ctx, nc_topk_kernel, grid_stride(ctx, rows, 8, 8), 256, 0, rows, r0, L, Lp, dZ.get(), dB.get(), dK.get(),
                        dOut.get()));
    }
    return copy_sync(ctx, pred_out, dOut.get(), sizeof(int32_t) * total, cudaMemcpyDeviceToHost);
}
