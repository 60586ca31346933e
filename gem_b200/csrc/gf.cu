// gem_b200/csrc/gf.cu -- Graph Factorization (SURVEY 8(f) rank 4): the edge SGD of gem/embedding/gf.py:94-104 (and of its C++ twin
// gem/c_src/gf.cpp:143-164):  for every epoch, for every edge (i, j, w) with j > i:
//        X[i] <- X[i] - eta * ( regu * X[i] - (w - <X[i], X[j]>) * X[j] )
// mode 0 (reference order): ONE warp walks the edge list in the order given, epoch after epoch -- exactly the reference's
//        sequential Gauss-Seidel sweep (fp32 where the Python loop is fp64); for the sizes the reference is used at.
// mode 1 (rows in parallel): one warp per source row; a row's own edges are applied in order with its running x_i (Gauss-Seidel
//        inside the row), the partner rows X[j] are read from the PREVIOUS epoch's table (Jacobi across rows, two tables): deterministic
//        and bit-reproducible whatever the launch shape, which is what lets tests/ compare it with the oracle's restatement.
// A lane owns the dimensions lane, lane + 32, ...; the dot product is a warp shuffle reduction; d <= 1024.
#include "common.cuh"
#include <chrono>

namespace gemb {

constexpr int GF_MAXV = 32;   // dimensions per lane kept in registers (d <= 1024)

template <int NV>
__device__ __forceinline__ void gf_edge(float (&xi)[NV], const float *__restrict__ xj_row, int d, int lane, float w, float eta, float regu) {
    float xj[NV];
    float dot = 0.f;
#pragma unroll
    for (int v = 0; v < NV; v++) {
        const int c = lane + 32 * v;
        xj[v] = c < d ? xj_row[c] : 0.f;
        dot = fmaf(xi[v], xj[v], dot);
    }
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float g = w - dot;
#pragma unroll
    for (int v = 0; v < NV; v++) xi[v] -= eta * (regu * xi[v] - g * xj[v]);
}

// mode 0: one warp, the reference's order
template <int NV>
__global__ void gf_sequential_kernel(int64_t m, const int32_t *__restrict__ src, const int32_t *__restrict__ dst,
                                     const float *__restrict__ w, int d, float eta, float regu, int epochs, float *X) {
    const int lane = threadIdx.x;
    for (int ep = 0; ep < epochs; ep++) {
        for (int64_t e = 0; e < m; e++) {
            const int i = src[e], j = dst[e];
            if (j <= i) continue;
            float xi[NV];
            float *xr = X + (int64_t)i * d;
#pragma unroll
            for (int v = 0; v < NV; v++) { const int c = lane + 32 * v; xi[v] = c < d ? xr[c] : 0.f; }
            gf_edge<NV>(xi, X + (int64_t)j * d, d, lane, w ? w[e] : 1.f, eta, regu);
#pragma unroll
            for (int v = 0; v < NV; v++) { const int c = lane + 32 * v; if (c < d) xr[c] = xi[v]; }
            __syncwarp();
        }
    }
}

// mode 1: warp per row; Xold read-only this epoch, Xnew written
template <int NV>
__global__ void __launch_bounds__(256)
gf_rows_kernel(int64_t n, const int64_t *__restrict__ rowptr, const int32_t *__restrict__ dst, const float *__restrict__ w, int d,
               float eta, float regu, const float *__restrict__ Xold, float *__restrict__ Xnew) {
    const int lane = threadIdx.x & 31;
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = warp; i < n; i += nwarps) {
        float xi[NV];
#pragma unroll
        for (int v = 0; v < NV; v++) { const int c = lane + 32 * v; xi[v] = c < d ? Xold[i * d + c] : 0.f; }
        for (int64_t e = rowptr[i]; e < rowptr[i + 1]; e++) {
            const int j = dst[e];
            if (j <= i) continue;
            gf_edge<NV>(xi, Xold + (int64_t)j * d, d, lane, w ? w[e] : 1.f, eta, regu);
        }
#pragma unroll
        for (int v = 0; v < NV; v++) { const int c = lane + 32 * v; if (c < d) Xnew[i * d + c] = xi[v]; }
    }
}

}  // namespace gemb

using namespace gemb;

extern "C" int gemb_gf(gemb_ctx *ctx, int64_t n, int64_t m, const int32_t *src, const int32_t *dst, const float *w, int d, float eta,
                       float regu, int max_iter, int mode, const float *X0, float *X_out, double *device_ms_out) {
    GEMB_ARG(ctx && n > 0 && m >= 0 && X0 && X_out, "ctx / n / X0 / X_out");
    GEMB_ARG(m == 0 || (src && dst), "edge arrays");
    GEMB_ARG(d >= 1 && d <= 32 * GF_MAXV, "d must be in 1..1024");
    GEMB_ARG(max_iter >= 0 && (mode == 0 || mode == 1), "max_iter / mode");
    GEMB_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<int64_t> rowptr;
    for (int64_t e = 0; e < m; e++) {
        GEMB_ARG(src[e] >= 0 && src[e] < n && dst[e] >= 0 && dst[e] < n, "edge endpoint outside [0, n)");
        if (mode == 1 && e > 0) GEMB_ARG(src[e] >= src[e - 1], "mode 1 needs the edges grouped by source row (non-decreasing src)");
    }
    DeviceBuffer<int32_t> d_src, d_dst;
    DeviceBuffer<float> d_w, Xa, Xb;
    DeviceBuffer<int64_t> d_rp;
    const size_t xb = sizeof(float) * (size_t)n * d;
    GEMB_CUDA(d_dst.upload(dst, m, st));
    if (w) GEMB_CUDA(d_w.upload(w, m, st));
    GEMB_CUDA(Xa.upload(X0, (size_t)n * d, st));
    if (mode == 0) {
        GEMB_CUDA(d_src.upload(src, m, st));
    } else {
        rowptr.assign(n + 1, 0);
        for (int64_t e = 0; e < m; e++) rowptr[src[e] + 1]++;
        for (int64_t i = 0; i < n; i++) rowptr[i + 1] += rowptr[i];
        GEMB_CUDA(d_rp.upload(rowptr.data(), n + 1, st));
        GEMB_CUDA(Xb.alloc((size_t)n * d));
    }
    CallEvents<2> ev;
    GEMB_CUDA(ev.create());
    GEMB_CUDA(cudaEventRecord(ev[0], st));
    int vi = 0;                                   // the instantiation: NV = 2^vi >= ceil(d / 32)
    while ((32 << vi) < d) vi++;
    float *cur = Xa.get();
    if (mode == 0) {
        if (m > 0 && max_iter > 0) {
            decltype(&gf_sequential_kernel<1>) const seq[] = {gf_sequential_kernel<1>, gf_sequential_kernel<2>, gf_sequential_kernel<4>,
                                                              gf_sequential_kernel<8>, gf_sequential_kernel<16>, gf_sequential_kernel<32>};
            GEMB_TRY(launch(ctx, seq[vi], 1, 32, 0, m, d_src.get(), d_dst.get(), d_w.get(), d, eta, regu, max_iter, Xa.get()));
        }
    } else {
        decltype(&gf_rows_kernel<1>) const rows[] = {gf_rows_kernel<1>, gf_rows_kernel<2>, gf_rows_kernel<4>,
                                                     gf_rows_kernel<8>, gf_rows_kernel<16>, gf_rows_kernel<32>};
        const int grid = grid_stride(ctx, n * 32, 256, 16);
        float *nxt = Xb.get();
        for (int ep = 0; ep < max_iter; ep++) {
            GEMB_TRY(launch(ctx, rows[vi], grid, 256, 0, n, d_rp.get(), d_dst.get(), d_w.get(), d, eta, regu, cur, nxt));
            std::swap(cur, nxt);
        }
    }
    GEMB_CUDA(cudaEventRecord(ev[1], st));
    GEMB_CUDA(cudaMemcpyAsync(X_out, cur, xb, cudaMemcpyDeviceToHost, st));
    GEMB_CUDA(cudaStreamSynchronize(st));
    if (device_ms_out) *device_ms_out = ev.ms(0, 1);
    return GEMB_OK;
}
