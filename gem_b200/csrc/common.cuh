// gem_b200/csrc/common.cuh -- shared declarations of libgemb200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include "../../include/gemb200.h"

namespace gemb {

void set_error(const char *fmt, ...);
void count_launch(int k = 1);   // every kernel launch of this library is counted (gemb_launch_count)

#define GEMB_CUDA(call)                                                                       \
    do {                                                                                      \
        cudaError_t _e = (call);                                                              \
        if (_e != cudaSuccess) {                                                              \
            gemb::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,              \
                            cudaGetErrorString(_e));                                          \
            (void)cudaGetLastError(); /* clear a non-sticky error for later calls */          \
            return GEMB_ERR_CUDA;                                                             \
        }                                                                                     \
    } while (0)

#define GEMB_TRY(call)                                                                        \
    do {                                                                                      \
        int _s = (call);                                                                      \
        if (_s != GEMB_OK) return _s;                                                         \
    } while (0)

#define GEMB_ARG(cond, msg)                                                                   \
    do {                                                                                      \
        if (!(cond)) {                                                                        \
            gemb::set_error("bad argument: %s (%s)", msg, #cond);                             \
            return GEMB_ERR_ARG;                                                              \
        }                                                                                     \
    } while (0)

// ---- NCCL, resolved lazily with dlopen so that the single-GPU path has no NCCL dependency
//      and so that a process that already loaded torch's libnccl.so.2 shares it.
struct NcclApi;
NcclApi *nccl_api();  // nullptr (and error set) if libnccl cannot be loaded

// ---- device memory (core.cu).  Released blocks are kept in a per-device free list and handed back on the next
//      request of the same rounded size (2 MiB granules from 1 MiB up, 512 B below), so a second learn_embedding call on the
//      same problem shape makes no driver allocation at all (cudaMalloc/cudaFree of 2.5 GB per call cost a
//      sporadic 100+ ms of page mapping).  GEMB_CACHE_MB caps the cached bytes (0 disables, default 65536);
//      gemb_mem_trim() releases everything.  dfree keeps cudaFree's implicit device synchronisation.
cudaError_t dmalloc_bytes(void **p, size_t bytes);
cudaError_t dfree(void *p);
template <class T> inline cudaError_t dmalloc(T **p, size_t bytes) { return dmalloc_bytes((void **)p, bytes); }

// Owner of one dmalloc block of `count` T for the scope it is declared in: released by dfree on every return path.
// Move-only: releasing a block twice would put it on the free list twice, and two later requests would share it.
// release() hands the block to a longer-lived object, which then frees it itself.
template <class T> class DeviceBuffer {
  public:
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer &) = delete;
    DeviceBuffer &operator=(const DeviceBuffer &) = delete;
    DeviceBuffer(DeviceBuffer &&o) noexcept : p_(o.release()) {}
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept {
        if (this != &o) { reset(); p_ = o.release(); }
        return *this;
    }
    ~DeviceBuffer() { reset(); }
    cudaError_t alloc(size_t count) { reset(); return dmalloc(&p_, sizeof(T) * count); }   // count 0: a minimal block
    T *get() const { return p_; }
    T *release() { T *p = p_; p_ = nullptr; return p; }
    void reset() { dfree(p_); p_ = nullptr; }

  private:
    T *p_ = nullptr;
};

// The N CUDA events of one call, destroyed on every return path.
template <int N> class CallEvents {
  public:
    CallEvents() = default;
    CallEvents(const CallEvents &) = delete;
    CallEvents &operator=(const CallEvents &) = delete;
    ~CallEvents() { for (cudaEvent_t e : ev_) if (e) cudaEventDestroy(e); }
    cudaError_t create() {
        for (cudaEvent_t &e : ev_) { const cudaError_t r = cudaEventCreate(&e); if (r != cudaSuccess) return r; }
        return cudaSuccess;
    }
    cudaEvent_t operator[](int i) const { return ev_[i]; }
    float ms(int from, int to) const { float t = 0.f; cudaEventElapsedTime(&t, ev_[from], ev_[to]); return t; }  // 0 on error

  private:
    cudaEvent_t ev_[N] = {};
};

struct Timer {  // pairs of events on ctx->stream, summed on demand
    std::vector<cudaEvent_t> ev;
    size_t used = 0;
    int begin(cudaStream_t s);
    int end(cudaStream_t s);
    double total_ms();  // synchronises on the recorded events
    void reset() { used = 0; }
    void destroy();
};

}  // namespace gemb

// Multi-GPU work blocks of the halo exchange (halo.cu), owned by the CONTEXT and kept across graphs and calls: the
// 5 x ~1 GB blocks, their CUDA-IPC mappings on every peer (35 cudaIpcOpenMemHandle at 8 ranks) and the barrier flags cost
// 1.4 s per learn_embedding call when they were set up per graph (r02k: e2e 1480 ms against an 86 ms solve).
struct gemb_halo_pool {
    size_t cap_floats = 0;            // capacity of every block (identical on all ranks: max over ranks of the need)
    int nbuf = 0;
    float *buf[8] = {};
    float *peer_buf[8][8] = {};       // [block][rank]
    unsigned long long *flags = nullptr;          // [nranks]; peer q writes flags[q]
    unsigned long long *peer_flags[8] = {};
    unsigned long long epoch = 0;
    int *timeout_flag = nullptr;
};

struct gemb_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaStream_t side = nullptr;     // work that runs beside a single-CTA kernel of `stream` (forked and joined by events)
    // multi-GPU
    int rank = 0, nranks = 1;
    void *comm = nullptr;  // ncclComm_t
    float *spmm_scratch = nullptr;   // chunk partial sums of the heavy rows (n_items x b), grown on demand
    size_t spmm_scratch_bytes = 0;
    double *red_scratch = nullptr;   // per-CTA partials of the fixed-order reductions (dense.cu), grown on demand
    size_t red_scratch_bytes = 0;
    gemb::Timer t_spmm, t_dense, t_comm, t_misc;
    gemb_halo_pool halo_pool;
};

struct gemb_csr_dev {
    int64_t nnz = 0;
    int32_t *indptr = nullptr;   // n_local + 1
    int32_t *indices = nullptr;  // nnz, global column ids
    float *data = nullptr;       // nnz or nullptr (unit weights)
    // rows longer than SPMM_HEAVY_DEG (power-law graphs) are cut into chunks of SPMM_HEAVY_CHUNK nonzeros that
    // whole CTAs process (spmm.cu); built at upload time from the host offsets
    int32_t n_heavy = 0, n_items = 0;
    int32_t *heavy_row = nullptr;    // n_heavy: shard-local row ids
    int32_t *heavy_first = nullptr;  // n_heavy + 1: first chunk of each heavy row
    int32_t *item_row = nullptr;     // n_items
    int32_t *item_beg = nullptr;     // n_items: offset of the chunk's first nonzero
};
constexpr int SPMM_HEAVY_DEG = 128, SPMM_HEAVY_CHUNK = 512;

// Multi-GPU HOPE on a symmetric shard: "needed rows only" exchange over NVLink peer memory (halo.cu).
// Every rank keeps its n x b work blocks as [n_shard local rows | halo_rows copies of the remote rows its CSR shard
// references]; the kernel that PRODUCES a block (SpMM epilogue, axpby, or a stand-alone push) stores each local row
// straight into the halo slots of the peers that reference it (P2P stores through CUDA-IPC mappings), so the next
// sweep gathers from local HBM only.  A flag barrier over the same mappings separates the sweeps.
constexpr int GEMB_MAX_RANKS = 8;
constexpr int GEMB_HALO_BUFS = 8;
struct gemb_halo {
    bool ready = false;
    int64_t halo_rows = 0;            // distinct remote rows this shard references
    int64_t push_total = 0;           // (local row, peer) pairs this rank pushes per exchanged block
    int32_t *indices_ext = nullptr;   // nnz: local column -> [0, n_shard), remote column -> n_shard + halo slot
    int32_t *push_ptr = nullptr;      // n_local + 1
    uint32_t *push_dst = nullptr;     // push_total: (peer << 29) | halo slot on that peer
    // peer-mapped work buffers, each (n_shard + halo_rows) x width floats
    int nbuf = 0, width = 0;
    float *buf[GEMB_HALO_BUFS] = {};
    float *peer_buf[GEMB_HALO_BUFS][GEMB_MAX_RANKS] = {};
    unsigned long long *flags = nullptr;                      // [nranks]; peer q writes flags[q]
    unsigned long long *peer_flags[GEMB_MAX_RANKS] = {};
    unsigned long long epoch = 0;
    int *timeout_flag = nullptr;                              // device: set when a barrier wait gave up
};
struct HaloPushArgs {                 // by-value kernel argument: where the rows of an output block also go
    const int32_t *push_ptr;
    const uint32_t *push_dst;
    float4 *peer[GEMB_MAX_RANKS];     // the SAME block on every rank (own rank unused)
    int64_t halo_row0;                // = n_shard: first halo row of a block
};

struct gemb_graph {
    gemb_ctx *ctx = nullptr;
    int64_t n = 0;        // global number of nodes
    int64_t row0 = 0;     // first row of this shard
    int64_t n_local = 0;  // real rows of this shard
    int64_t n_shard = 0;  // rows per rank used for collectives (= ceil(n / nranks)); n_local <= n_shard
    int64_t n_pad = 0;    // n_shard * nranks
    bool symmetric = false;
    bool replicated = false;  // multi-GPU: the whole graph on every rank (node2vec) instead of a row shard
    gemb_csr_dev A, AT;   // AT aliases A when symmetric
    gemb_halo halo;       // multi-GPU symmetric shards (built on first use)
};

namespace gemb {

// ---- spmm.cu
// Y[n_rows x b] = X0 + alpha * A * X ; X has leading dimension ldx (>= b), rows indexed by the
// global column ids in A.  X0/Y are row shards (ld = b).  All device pointers.
int spmm_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, float alpha,
                const float *X, const float *X0, float *Y);
// Y = alpha * A * X + gamma * Xself + delta * X0   (Xself / X0: row shards, may be null)
int spmm3_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, float alpha, const float *X,
                 float gamma, const float *Xself, float delta, const float *X0, float *Y,
                 const HaloPushArgs *push = nullptr);
// the same with a fourth epilogue operand: Y = alpha * A * X + gamma * Xself + delta * X0 + eps * X1 (single GPU, no
// push; X1 needs Xself and X0).  The composite operator's Chebyshev step (hope.cu, spectral_mode 2) takes four rows.
int spmm4_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, float alpha, const float *X,
                 float gamma, const float *Xself, float delta, const float *X0, float eps, const float *X1, float *Y);
// Y = alpha * diag(rscale) * A * X: every row's sum scaled by its entry of rscale (n_rows floats, device; single GPU, no
// other epilogue operand).  Sweep 1 of the Adamic-Adar operator A D A (hope.cu, spectral_mode 4).
int spmm_scaled_launch(gemb_ctx *ctx, const gemb_csr_dev &A, int64_t n_rows, int b, float alpha, const float *X,
                       const float *rscale, float *Y);

// ---- halo.cu (multi-GPU)
int halo_build(gemb_graph *g);                                   // collective; idempotent
int halo_buffers(gemb_graph *g, int nbuf, int width);            // collective; (re)allocates + IPC-maps the work blocks
int halo_push_launch(gemb_graph *g, int buf_index, int width);  // stand-alone push of a block's local rows
int halo_barrier(gemb_graph *g);                                 // all ranks' pushes issued before it have landed
void halo_push_args(const gemb_graph *g, int buf_index, HaloPushArgs *out);
int halo_free(gemb_graph *g);
void halo_pool_release(gemb_ctx *c);                              // at context destruction (not collective)
// Y = a P + c Q over the local rows of halo blocks, pushing Y's rows to the peers (Chebyshev first step)
int halo_check_timeout(gemb_graph *g);

// ---- dense.cu
// G[b1 x b2] (fp64, row-major, OVERWRITTEN) = P^T Q over n rows (P: n x b1, Q: n x b2, fp32).
int gram_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G);
// Out[n x b2] = Q[n x b1] * M[b1 x b2]  (M fp32 device, row-major, ld = ldm). Out may not alias Q.
int apply_launch(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int ldm, int b2,
                 float *Out, int ldo);
int apply_fp32_launch(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int ldm, int b2,
                      float *Out, int ldo);
// Small b x b factorizations, single CTA, fp64 (device pointers):
//  chol_inverse: G (b x b, SPD up to rank deficiency) -> Minv fp32 (b x b) with G = R^T R, Minv = R^-1
//  (columns whose pivot of the unit-diagonal scaled G falls below GEMB_PIV_EPS are zeroed: Q*Minv then has zero columns
//  there).  G is overwritten where the matrix does not fit in shared memory (b > 168 on H100).
int chol_inverse_launch(gemb_ctx *ctx, int b, double *G, float *Minv, int *rank_out_dev, double *Minv64 = nullptr);
//  C (fp64) and/or C32 (fp32) = op(A) * B for b x b fp64 matrices (one CTA)
int small_gemm_launch(gemb_ctx *ctx, int b, const double *A, int transA, const double *B, double *C, float *C32);
// CUDA-core Gram (gram_launch prefers the wgmma kernel in gram_tc.cu when the shape fits)
int gram_fp32_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G);
int gram_tc_launch(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, double *G);
// Reductions across CTAs never use floating-point atomics: every CTA writes its partial, and
// out[i] = sum_{c < parts} part[c * count + i] is added in a fixed order, so a result is the same on every run.
int red_scratch(gemb_ctx *ctx, size_t doubles, double **out);
int sum_partials_launch(gemb_ctx *ctx, int parts, int64_t count, const double *part, double *out);
//  eigh: G -> eigenvalues w ascending (b), eigenvectors Z (b x b, column j <-> w[j]); G destroyed where the matrix does
//  not fit in shared memory (b >= 168).
// rel_tol: stop the Jacobi sweeps when ||offdiag||_F <= rel_tol * ||G||_F
int eigh_launch(gemb_ctx *ctx, int b, double *G, double *w, double *Z, double *Zscratch /* b x b */, double rel_tol = 1e-11,
                bool symmetrize = false /* decompose (G + G^T) / 2 */);
int randn_launch(gemb_ctx *ctx, int64_t n, int b, uint64_t seed, uint64_t row_offset, float *X);
// sum of squares of all entries (fp64 accumulate) -> out_dev[0]
int sumsq_launch(gemb_ctx *ctx, int64_t count, const float *X, double *out_dev);
int scale_launch(gemb_ctx *ctx, int64_t count, float s, float *X);
// Y += a * X over count floats (one rounding per element: a = -1 gives exactly Y - X)
int axpy_launch(gemb_ctx *ctx, int64_t count, float a, const float *X, float *Y);


#ifdef __CUDACC__
// store the finished row chunk r (4 floats of local row `row`, chunk c of G) into every peer halo slot that references it
__device__ __forceinline__ void halo_push_row(const HaloPushArgs &P, int64_t row, int G, int c, const float4 &r) {
    const int i0 = P.push_ptr[row], i1 = P.push_ptr[row + 1];
    if (i0 == i1) return;
    for (int i = i0; i < i1; i++) {
        const uint32_t d = P.push_dst[i];
        P.peer[d >> 29][(P.halo_row0 + (int64_t)(d & 0x1fffffffu)) * G + c] = r;
    }
}
#endif

}  // namespace gemb
