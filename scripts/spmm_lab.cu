// scripts/spmm_lab.cu -- developer microbenchmark (not the product): design space of the CSR SpMM sweep
//     Y = alpha * A X + gamma * X + delta * X0        (the Chebyshev three-term step of the HOPE solver)
// on the BASELINE configs[1] graph (SBM 1M nodes / 19.86M directed edges).  Variants:
//   rm    : row-major n x b block, group of b/4 threads per row (the round-1 kernel)
//   panel : the block stored PANEL-major, [b/W][n][W]; one pass per W-column panel, so that the panel being gathered
//           (4 n W bytes) can stay L2 resident while the streaming operands pass by with evict-first hints
//   tile  : panel-major + the diagonal block of every R-row tile staged into shared memory by one TMA bulk copy;
//           neighbours inside the tile are read from shared memory (an SBM community is a diagonal block), the
//           `gamma * X[row]` term comes from the staged tile for free
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -o /tmp/spmm_lab scripts/spmm_lab.cu
// Run:   /tmp/spmm_lab indptr.bin indices.bin   (raw int32 arrays written by scripts/spmm_lab.py)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ void fma4(float4 &a, const float4 &x) { a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w; }
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- rowgroup kernel over an n x W array (row-major with ld = W): used for `rm` (W = b) and for `panel`
template <bool STREAM>
__global__ void __launch_bounds__(256)
rowgroup_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n, int G, int rpc,
                float alpha, float gamma, float delta, const float4 *__restrict__ X, const float4 *__restrict__ X0,
                float4 *__restrict__ Y) {
    const int lr = threadIdx.x / G, c = threadIdx.x - lr * G;
    if (lr >= rpc) return;
    const int64_t row = (int64_t)blockIdx.x * rpc + lr;
    if (row >= n) return;
    const int s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
    const float4 *Xc = X + c;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int i = s;
    for (; i + 4 <= e; i += 4) {
        const int c0 = __ldg(indices + i), c1 = __ldg(indices + i + 1), c2 = __ldg(indices + i + 2), c3 = __ldg(indices + i + 3);
        const float4 x0 = __ldg(Xc + (int64_t)c0 * G), x1 = __ldg(Xc + (int64_t)c1 * G);
        const float4 x2 = __ldg(Xc + (int64_t)c2 * G), x3 = __ldg(Xc + (int64_t)c3 * G);
        fma4(acc, x0); fma4(acc, x1); fma4(acc, x2); fma4(acc, x3);
    }
    for (; i < e; i++) fma4(acc, __ldg(Xc + (int64_t)__ldg(indices + i) * G));
    const float4 xs = __ldg(Xc + row * G);
    const float4 z = STREAM ? __ldcs(X0 + row * G + c) : __ldg(X0 + row * G + c);
    float4 r;
    r.x = alpha * acc.x + gamma * xs.x + delta * z.x;
    r.y = alpha * acc.y + gamma * xs.y + delta * z.y;
    r.z = alpha * acc.z + gamma * xs.z + delta * z.z;
    r.w = alpha * acc.w + gamma * xs.w + delta * z.w;
    if (STREAM) __stcs(Y + row * G + c, r); else Y[row * G + c] = r;
}

// ---- tile kernel: one CTA per R-row tile of one panel; the tile's own rows of X staged in shared memory
template <int G>   // threads per row = W / 4
__global__ void __launch_bounds__(256)
tile_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n, int R,
            float alpha, float gamma, float delta, const float4 *__restrict__ X, const float4 *__restrict__ X0,
            float4 *__restrict__ Y) {
    extern __shared__ __align__(128) float4 tile[];
    __shared__ __align__(8) uint64_t bar;
    constexpr int RPC = 256 / G;
    const int lr = threadIdx.x / G, c = threadIdx.x - lr * G;
    const int64_t r0 = (int64_t)blockIdx.x * R;
    const int64_t r1 = r0 + R < n ? r0 + R : n;
    const uint32_t b32 = smem_u32(&bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b32));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t bytes = (uint32_t)((r1 - r0) * G * 16);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b32), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(tile)), "l"(X + r0 * G), "r"(bytes), "r"(b32) : "memory");
    }
    __syncthreads();
    {
        uint32_t ok = 0;
        for (uint32_t it = 0; it < (1u << 22) && !ok; it++) {
            asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.b32 %0, 1, 0, p;\n}"
                         : "=r"(ok) : "r"(b32), "r"(0u) : "memory");
        }
        if (!ok) __trap();
    }
    if (lr >= RPC) return;
    const float4 *Xc = X + c;
    const float4 *Tc = tile + c;
    const int lo = (int)r0;
    const unsigned span = (unsigned)(r1 - r0);
    for (int64_t row = r0 + lr; row < r1; row += RPC) {
        const int s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        int i = s;
        for (; i + 4 <= e; i += 4) {
            const int c0 = __ldg(indices + i), c1 = __ldg(indices + i + 1), c2 = __ldg(indices + i + 2), c3 = __ldg(indices + i + 3);
            const unsigned d0 = (unsigned)(c0 - lo), d1 = (unsigned)(c1 - lo), d2 = (unsigned)(c2 - lo), d3 = (unsigned)(c3 - lo);
            float4 x0, x1, x2, x3;
            if (d0 < span) x0 = Tc[d0 * G]; else x0 = __ldg(Xc + (int64_t)c0 * G);
            if (d1 < span) x1 = Tc[d1 * G]; else x1 = __ldg(Xc + (int64_t)c1 * G);
            if (d2 < span) x2 = Tc[d2 * G]; else x2 = __ldg(Xc + (int64_t)c2 * G);
            if (d3 < span) x3 = Tc[d3 * G]; else x3 = __ldg(Xc + (int64_t)c3 * G);
            fma4(acc, x0); fma4(acc, x1); fma4(acc, x2); fma4(acc, x3);
        }
        for (; i < e; i++) {
            const int c0 = __ldg(indices + i);
            const unsigned d0 = (unsigned)(c0 - lo);
            float4 x0;
            if (d0 < span) x0 = Tc[d0 * G]; else x0 = __ldg(Xc + (int64_t)c0 * G);
            fma4(acc, x0);
        }
        const float4 xs = Tc[(row - r0) * G];
        const float4 z = __ldcs(X0 + row * G + c);
        float4 r;
        r.x = alpha * acc.x + gamma * xs.x + delta * z.x;
        r.y = alpha * acc.y + gamma * xs.y + delta * z.y;
        r.z = alpha * acc.z + gamma * xs.z + delta * z.z;
        r.w = alpha * acc.w + gamma * xs.w + delta * z.w;
        __stcs(Y + row * G + c, r);
    }
}

__device__ __forceinline__ float4 ldg_na(const float4 *p) {   // read-only path, no L1 allocation
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// ---- rm variants: UNROLL gathers in flight, NA = gathers bypass L1 allocation
template <int UNROLL, int HINT>
__global__ void __launch_bounds__(256)
rowgroup_u_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n, int G, int rpc,
                  float alpha, float gamma, float delta, const float4 *__restrict__ X, const float4 *__restrict__ X0,
                  float4 *__restrict__ Y) {
    const int lr = threadIdx.x / G, c = threadIdx.x - lr * G;
    if (lr >= rpc) return;
    const int64_t row = (int64_t)blockIdx.x * rpc + lr;
    if (row >= n) return;
    const int s = __ldg(indptr + row), e = __ldg(indptr + row + 1);
    const float4 *Xc = X + c;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int i = s;
    for (; i + UNROLL <= e; i += UNROLL) {
        int cc[UNROLL];
        float4 x[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; u++) cc[u] = __ldg(indices + i + u);
#pragma unroll
        for (int u = 0; u < UNROLL; u++) x[u] = (HINT & 4) ? ldg_na(Xc + (int64_t)cc[u] * G) : __ldg(Xc + (int64_t)cc[u] * G);
#pragma unroll
        for (int u = 0; u < UNROLL; u++) fma4(acc, x[u]);
    }
    for (; i < e; i++) fma4(acc, (HINT & 4) ? ldg_na(Xc + (int64_t)__ldg(indices + i) * G) : __ldg(Xc + (int64_t)__ldg(indices + i) * G));
    const float4 xs = __ldg(Xc + row * G);
    const float4 z = (HINT & 1) ? __ldcs(X0 + row * G + c) : __ldg(X0 + row * G + c);
    float4 r;
    r.x = alpha * acc.x + gamma * xs.x + delta * z.x;
    r.y = alpha * acc.y + gamma * xs.y + delta * z.y;
    r.z = alpha * acc.z + gamma * xs.z + delta * z.z;
    r.w = alpha * acc.w + gamma * xs.w + delta * z.w;
    if (HINT & 2) __stcs(Y + row * G + c, r); else Y[row * G + c] = r;
}

// ---- rm + the CTA's slice of the column ids staged into shared memory by ONE TMA bulk copy (non-persistent: one tile
// of PASSES * rpc consecutive rows per CTA; the other resident CTAs of the SM hide the copy's latency)
constexpr int TMA_CAP = 3072;
template <int UNROLL, int HINT>
__global__ void __launch_bounds__(256)
rowgroup_tma_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n, int64_t nnz_pad, int G, int rpc,
                    int passes, float alpha, float gamma, float delta, const float4 *__restrict__ X,
                    const float4 *__restrict__ X0, float4 *__restrict__ Y) {
    __shared__ __align__(16) int32_t s_idx[TMA_CAP + 8];
    __shared__ __align__(8) uint64_t bar;
    __shared__ int s_base;
    const int lr = threadIdx.x / G, c = threadIdx.x - lr * G;
    const int64_t r0 = (int64_t)blockIdx.x * rpc * passes;
    const int64_t r1 = r0 + rpc * passes < n ? r0 + rpc * passes : n;
    const uint32_t b32 = smem_u32(&bar);
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b32));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const int s = __ldg(indptr + r0), e = __ldg(indptr + r1);
        const int a0 = s & ~3;
        int cnt = (e - a0 + 3) & ~3;
        if ((int64_t)a0 + cnt > nnz_pad) cnt = (int)(nnz_pad - a0);
        if (e > s && cnt <= TMA_CAP) {
            s_base = a0;
            const uint32_t bytes = (uint32_t)cnt * 4u;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b32), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32(s_idx)), "l"(indices + a0), "r"(bytes), "r"(b32) : "memory");
        } else {
            s_base = -1;
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(b32) : "memory");
        }
    }
    __syncthreads();
    if (lr >= rpc) return;
    // the row's offsets are fetched while the bulk copy is in flight
    int64_t row = r0 + lr;
    int s = 0, e = 0;
    if (row < r1) { s = __ldg(indptr + row); e = __ldg(indptr + row + 1); }
    {
        uint32_t ok = 0;
        for (uint32_t it = 0; it < (1u << 22) && !ok; it++)
            asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.b32 %0, 1, 0, p;\n}"
                         : "=r"(ok) : "r"(b32), "r"(0u) : "memory");
        if (!ok) __trap();
    }
    const int base = s_base;
    const int32_t *li = base >= 0 ? s_idx - base : nullptr;
    const float4 *Xc = X + c;
    for (; row < r1; row += rpc) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        int i = s;
        for (; i + UNROLL <= e; i += UNROLL) {
            int cc[UNROLL];
            float4 x[UNROLL];
#pragma unroll
            for (int u = 0; u < UNROLL; u++) cc[u] = li ? li[i + u] : __ldg(indices + i + u);
#pragma unroll
            for (int u = 0; u < UNROLL; u++) x[u] = __ldg(Xc + (int64_t)cc[u] * G);
#pragma unroll
            for (int u = 0; u < UNROLL; u++) fma4(acc, x[u]);
        }
        for (; i < e; i++) fma4(acc, __ldg(Xc + (int64_t)(li ? li[i] : __ldg(indices + i)) * G));
        const float4 xs = __ldg(Xc + row * G);
        const float4 z = (HINT & 1) ? __ldcs(X0 + row * G + c) : __ldg(X0 + row * G + c);
        float4 r;
        r.x = alpha * acc.x + gamma * xs.x + delta * z.x;
        r.y = alpha * acc.y + gamma * xs.y + delta * z.y;
        r.z = alpha * acc.z + gamma * xs.z + delta * z.z;
        r.w = alpha * acc.w + gamma * xs.w + delta * z.w;
        if (HINT & 2) __stcs(Y + row * G + c, r); else Y[row * G + c] = r;
        const int64_t nrow = row + rpc;
        if (nrow < r1) { s = __ldg(indptr + nrow); e = __ldg(indptr + nrow + 1); }
    }
}

static std::vector<int32_t> read_i32(const char *path) {
    FILE *f = fopen(path, "rb");
    if (!f) { fprintf(stderr, "cannot open %s\n", path); exit(1); }
    fseek(f, 0, SEEK_END);
    long sz = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::vector<int32_t> v(sz / 4);
    if (fread(v.data(), 4, v.size(), f) != v.size()) { fprintf(stderr, "short read\n"); exit(1); }
    fclose(f);
    return v;
}

struct Run { std::string name; double ms; double maxdiff; };

int main(int argc, char **argv) {
    if (argc < 3) { fprintf(stderr, "usage: spmm_lab indptr.bin indices.bin [b]\n"); return 1; }
    std::vector<int32_t> ip = read_i32(argv[1]), ix = read_i32(argv[2]);
    const int64_t n = (int64_t)ip.size() - 1, nnz = ix.size();
    const int reps = 10;
    const bool quick = argc > 3 && !strcmp(argv[3], "quick");
    printf("{\"n\": %lld, \"nnz\": %lld}\n", (long long)n, (long long)nnz);
    int32_t *d_ip, *d_ix;
    CK(cudaMalloc(&d_ip, 4 * (n + 1)));
    CK(cudaMalloc(&d_ix, 4 * (nnz + 8)));
    CK(cudaMemcpy(d_ip, ip.data(), 4 * (n + 1), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_ix, ix.data(), 4 * nnz, cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const float alpha = 0.37f, gamma = -0.21f, delta = -0.83f;

    for (int b : {72, 80}) {
        const size_t elems = (size_t)n * b;
        std::vector<float> hX(elems), hX0(elems);
        uint32_t st = 12345u + b;
        for (size_t i = 0; i < elems; i++) { st = st * 1664525u + 1013904223u; hX[i] = (float)(int)(st >> 8) * (1.f / 8388608.f) - 1.f; }
        for (size_t i = 0; i < elems; i++) { st = st * 1664525u + 1013904223u; hX0[i] = (float)(int)(st >> 8) * (1.f / 8388608.f) - 1.f; }
        float *X, *X0, *Y, *Yref;
        CK(cudaMalloc(&X, 4 * elems)); CK(cudaMalloc(&X0, 4 * elems)); CK(cudaMalloc(&Y, 4 * elems)); CK(cudaMalloc(&Yref, 4 * elems));
        // ---- row-major reference
        CK(cudaMemcpy(X, hX.data(), 4 * elems, cudaMemcpyHostToDevice));
        CK(cudaMemcpy(X0, hX0.data(), 4 * elems, cudaMemcpyHostToDevice));
        {
            const int G = b / 4, rpc = 256 / G;
            const unsigned grid = (unsigned)((n + rpc - 1) / rpc);
            for (int w = 0; w < 2; w++)
                rowgroup_kernel<false><<<grid, 256>>>(d_ip, d_ix, n, G, rpc, alpha, gamma, delta, (const float4 *)X, (const float4 *)X0, (float4 *)Yref);
            CK(cudaEventRecord(e0));
            for (int r = 0; r < reps; r++)
                rowgroup_kernel<false><<<grid, 256>>>(d_ip, d_ix, n, G, rpc, alpha, gamma, delta, (const float4 *)X, (const float4 *)X0, (float4 *)Yref);
            CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            printf("{\"variant\": \"rm\", \"b\": %d, \"ms_per_sweep\": %.4f}\n", b, ms / reps);
            fflush(stdout);
        }
        std::vector<float> hRef(elems);
        CK(cudaMemcpy(hRef.data(), Yref, 4 * elems, cudaMemcpyDeviceToHost));
        {
            const int G = b / 4, rpc = 256 / G;
            const unsigned grid = (unsigned)((n + rpc - 1) / rpc);
            const int64_t nnz_pad = (nnz + 3) & ~(int64_t)3;
            auto timeit = [&](const char *name, int extra, auto launch) {
                CK(cudaMemset(Y, 0, 4 * elems));
                launch(); launch();
                CK(cudaGetLastError());
                CK(cudaEventRecord(e0));
                for (int r = 0; r < reps; r++) launch();
                CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
                float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
                std::vector<float> hY(elems);
                CK(cudaMemcpy(hY.data(), Y, 4 * elems, cudaMemcpyDeviceToHost));
                double md = 0;
                for (size_t i = 0; i < elems; i += 13) md = fmax(md, fabs((double)hY[i] - (double)hRef[i]));
                printf("{\"variant\": \"%s\", \"b\": %d, \"param\": %d, \"ms_per_sweep\": %.4f, \"maxdiff\": %.3g}\n", name, b, extra, ms / reps, md);
                fflush(stdout);
            };
#define RMU(U, H) timeit("rm_u" #U "_h" #H, H, [&]() { rowgroup_u_kernel<U, H><<<grid, 256>>>(d_ip, d_ix, n, G, rpc, alpha, gamma, delta, (const float4 *)X, (const float4 *)X0, (float4 *)Y); });
            RMU(4, 0) RMU(4, 1) RMU(4, 2) RMU(4, 3) RMU(8, 0) RMU(2, 0)
#undef RMU
            for (int passes : {2, 3, 4, 6}) {
                const unsigned g2 = (unsigned)((n + (int64_t)rpc * passes - 1) / ((int64_t)rpc * passes));
                timeit("rm_tma_u4_h0", passes, [&]() { rowgroup_tma_kernel<4, 0><<<g2, 256>>>(d_ip, d_ix, n, nnz_pad, G, rpc, passes, alpha, gamma, delta, (const float4 *)X, (const float4 *)X0, (float4 *)Y); });
                timeit("rm_tma_u2_h0", passes, [&]() { rowgroup_tma_kernel<2, 0><<<g2, 256>>>(d_ip, d_ix, n, nnz_pad, G, rpc, passes, alpha, gamma, delta, (const float4 *)X, (const float4 *)X0, (float4 *)Y); });
                timeit("rm_tma_u4_h1", passes, [&]() { rowgroup_tma_kernel<4, 1><<<g2, 256>>>(d_ip, d_ix, n, nnz_pad, G, rpc, passes, alpha, gamma, delta, (const float4 *)X, (const float4 *)X0, (float4 *)Y); });
            }
        }
        if (quick) { CK(cudaFree(X)); CK(cudaFree(X0)); CK(cudaFree(Y)); CK(cudaFree(Yref)); continue; }

        // ---- panel-major variants
        for (int W : {8, 12, 16, 24, 36, 40}) {
            if (b % W) continue;
            const int np = b / W, G = W / 4;
            // repack X, X0 panel-major on the host
            std::vector<float> pX(elems), pX0(elems);
            for (int p = 0; p < np; p++)
                for (int64_t r = 0; r < n; r++) {
                    memcpy(&pX[(size_t)p * n * W + (size_t)r * W], &hX[(size_t)r * b + p * W], 4 * W);
                    memcpy(&pX0[(size_t)p * n * W + (size_t)r * W], &hX0[(size_t)r * b + p * W], 4 * W);
                }
            CK(cudaMemcpy(X, pX.data(), 4 * elems, cudaMemcpyHostToDevice));
            CK(cudaMemcpy(X0, pX0.data(), 4 * elems, cudaMemcpyHostToDevice));
            auto check = [&](const char *name, double ms, int R) {
                std::vector<float> hY(elems);
                CK(cudaMemcpy(hY.data(), Y, 4 * elems, cudaMemcpyDeviceToHost));
                double md = 0;
                for (int p = 0; p < np; p++)
                    for (int64_t r = 0; r < n; r += 97)
                        for (int j = 0; j < W; j++)
                            md = fmax(md, fabs((double)hY[(size_t)p * n * W + (size_t)r * W + j] - (double)hRef[(size_t)r * b + p * W + j]));
                printf("{\"variant\": \"%s\", \"b\": %d, \"W\": %d, \"R\": %d, \"ms_per_sweep\": %.4f, \"ms_per_panel\": %.4f, \"maxdiff\": %.3g}\n",
                       name, b, W, R, ms, ms / np, md);
                fflush(stdout);
            };
            {
                const int rpc = 256 / G;
                const unsigned grid = (unsigned)((n + rpc - 1) / rpc);
                auto sweep = [&]() {
                    for (int p = 0; p < np; p++) {
                        const size_t off = (size_t)p * n * W;
                        rowgroup_kernel<true><<<grid, 256>>>(d_ip, d_ix, n, G, rpc, alpha, gamma, delta, (const float4 *)(X + off),
                                                             (const float4 *)(X0 + off), (float4 *)(Y + off));
                    }
                };
                CK(cudaMemset(Y, 0, 4 * elems));
                sweep(); sweep();
                CK(cudaEventRecord(e0));
                for (int r = 0; r < reps; r++) sweep();
                CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
                float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
                check("panel", ms / reps, 0);
            }
            for (int R : {256, 512, 1000, 1024, 2048}) {
                const size_t smem = (size_t)R * W * 4;
                if (smem > 200 * 1024) continue;
                const unsigned grid = (unsigned)((n + R - 1) / R);
                auto launch = [&](size_t off) {
#define TK(GG) case GG: { static bool set##GG = false; if (!set##GG) { CK(cudaFuncSetAttribute(tile_kernel<GG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); set##GG = true; } \
                    tile_kernel<GG><<<grid, 256, smem>>>(d_ip, d_ix, n, R, alpha, gamma, delta, (const float4 *)(X + off), (const float4 *)(X0 + off), (float4 *)(Y + off)); } break;
                    switch (G) { TK(2) TK(3) TK(4) TK(6) TK(9) TK(10) default: break; }
#undef TK
                };
                auto sweep = [&]() { for (int p = 0; p < np; p++) launch((size_t)p * n * W); };
                CK(cudaMemset(Y, 0, 4 * elems));
                sweep(); sweep();
                CK(cudaGetLastError());
                CK(cudaEventRecord(e0));
                for (int r = 0; r < reps; r++) sweep();
                CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
                float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
                check("tile", ms / reps, R);
            }
        }
        CK(cudaFree(X)); CK(cudaFree(X0)); CK(cudaFree(Y)); CK(cudaFree(Yref));
    }
    return 0;
}
