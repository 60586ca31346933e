/*
 * include/gemb200.h -- C ABI of libgemb200.so, the H100 (sm_90a) core behind GEM's
 * StaticGraphEmbedding plugin API for HOPE and node2vec.
 *
 * The reference has no FFI for this path: HOPE is four NumPy/SciPy lines
 * (gem/embedding/hope.py:28-36) and node2vec is an argv + text-file hand-off to a prebuilt
 * SNAP executable (gem/embedding/node2vec.py:31-53).  Each entry point below names the reference
 * interface it replaces; INTEGRATION.md shows the ctypes stub a GEM maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; every function returns 0 (GEMB_OK) or a negative
 *     gemb_status; gemb_last_error() gives the message of the last failure on this thread.
 *   - the caller owns every host buffer; the library owns device memory behind opaque handles.
 *   - calls are blocking; one gemb_ctx is bound to one CUDA device and is not thread-safe.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     GEMB_ERR_CUDA.
 *   - matrices are row-major; node ids / column ids are int32; CSR offsets are int64 on the
 *     host ABI (node2vec) or int32 (HOPE shards, nnz < 2^31 per shard).
 */
#ifndef GEMB200_H
#define GEMB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GEMB_VERSION 100 /* 0.1.0 */

typedef enum {
    GEMB_OK = 0,
    GEMB_ERR_CUDA = -1,      /* no device / CUDA runtime or kernel failure */
    GEMB_ERR_ARG = -2,       /* bad argument */
    GEMB_ERR_NOMEM = -3,     /* host or device allocation failed */
    GEMB_ERR_DIVERGE = -4,   /* beta * rho(A) >= 1: Katz series does not converge */
    GEMB_ERR_NCCL = -5,      /* NCCL missing or collective failed */
    GEMB_ERR_UNSUPPORTED = -6
} gemb_status;

typedef struct gemb_ctx gemb_ctx;     /* one CUDA device + stream (+ optional NCCL communicator) */
typedef struct gemb_graph gemb_graph; /* a CSR row shard (and its transpose) resident in HBM   */

int gemb_version(void);
const char *gemb_last_error(void);
int gemb_device_count(void); /* number of CUDA devices, 0 if none / no driver */
int64_t gemb_launch_count(void); /* kernels this library has launched in this process so far */

int gemb_ctx_create(int device, gemb_ctx **out);
int gemb_ctx_destroy(gemb_ctx *ctx);

/* Pinned (page-locked) host buffers for the host<->device copies of the e2e path. */
int gemb_host_alloc(size_t bytes, void **out);
int gemb_host_free(void *p);

/* Device work buffers of one call (the CSR arrays, the n x (d/2+p) blocks) are kept in a per-device free
 * list when the call returns, so that the next learn_embedding on the same problem shape makes no driver
 * allocation (the reference re-allocates everything per call, hope.py:26-34; at 2.5 GB per call the
 * driver's page mapping costs more than the solve).  GEMB_CACHE_MB caps the list (0 = off).
 * gemb_mem_trim returns every cached block to the driver; gemb_mem_cached_bytes reports the list.
 * gemb_mem_live_blocks counts the blocks handed out and not yet released (graphs, reconstructions, context scratch,
 * and the work buffers of calls in flight); 0 when the cache is off.  A call that returns leaves it as it found it. */
int gemb_mem_trim(void);
size_t gemb_mem_cached_bytes(void);
size_t gemb_mem_live_blocks(void);

/* ---- Graph Factorization (SURVEY 8(f) rank 4).  Replaces the edge SGD of gem/embedding/gf.py:94-104 (its C++ twin:
 * gem/c_src/gf.cpp:143-164; the reference shells out to gem/c_exe/gf when it exists and then runs the Python loop anyway):
 *     for epoch in range(max_iter): for (i, j, w) in edges, j > i:  X[i] -= eta * (regu * X[i] - (w - <X[i], X[j]>) * X[j])
 * src / dst / w: the m directed edges (host; w NULL = 1).  X0: the n x d start (the reference draws 0.01 * randn), X_out: n x d.
 * mode 0: one warp applies the edges in the order given, epoch after epoch (the reference's sequential sweep, fp32).
 * mode 1: one warp per source row (edges grouped by src, in order), partner rows read from the previous epoch's table
 *         (Jacobi across rows, Gauss-Seidel inside a row): deterministic, for graphs beyond the reference's reach. */
int gemb_gf(gemb_ctx *ctx, int64_t n, int64_t m, const int32_t *src, const int32_t *dst, const float *w, int d, float eta,
            float regu, int max_iter, int mode, const float *X0, float *X_out, double *device_ms_out);

/* ---- bench infrastructure: Graph500 R-MAT generator on the device (BASELINE.json configs[3], configs[4]: scale 24).
 * No reference counterpart (GEM ships no generator; gem/tests load fixed fixtures); the host generator
 * gem_b200/synth.py::rmat makes the same kind of graph with NumPy for the small parity cases.
 * Rows [row0, row0 + n_rows) (n_rows < 0: all) of the symmetrised, loop-free, duplicate-free graph with sorted column
 * ids.  indices_out = NULL: only *nnz_out (shard) and *nnz_total_out (graph) are set; otherwise indptr_out (n_rows + 1
 * int64, shard-local offsets) and indices_out (cap >= nnz) are filled.  Counter-based RNG: identical on every rank. */
int gemb_synth_rmat(gemb_ctx *ctx, int scale, int edge_factor, double a, double b, double c, uint64_t seed, int permute,
                    int64_t row0, int64_t n_rows, int64_t *nnz_out, int64_t *nnz_total_out, int64_t *indptr_out,
                    int32_t *indices_out, int64_t cap);

/* ---- multi-GPU: one process per GPU; rank 0 makes the id, every rank calls init.
 * (No reference counterpart: GEM is single-process; SURVEY 2.2.) */
#define GEMB_UNIQUE_ID_BYTES 128
int gemb_comm_unique_id(void *id_out /* GEMB_UNIQUE_ID_BYTES */);
int gemb_comm_init(gemb_ctx *ctx, int rank, int nranks, const void *id);

/* ---- graph upload.
 * Replaces: nx.to_numpy_matrix(graph) (hope.py:28) and the text edge list written by
 * graph_util.saveGraphToEdgeListTxtn2v (graph_util.py:137-140) + SNAP ReadGraph (bin@0x406550).
 *
 * The shard holds rows [row0, row0+n_local) of the n x n adjacency A in CSR form with GLOBAL
 * column ids, and the same row range of A^T (pass indptr_t == NULL when A is symmetric: A^T = A).
 * data / data_t may be NULL (all weights 1.0).  Single GPU: row0 = 0, n_local = n.
 * Multi GPU (after gemb_comm_init): for HOPE every rank uploads rows [rank*ceil(n/P), ...) (the last rank
 * may own fewer real rows; the library pads); for node2vec every rank uploads the whole graph
 * (row0 = 0, n_local = n: CSR and alias tables are replicated, the walk index space is sharded).  */
int gemb_graph_upload(gemb_ctx *ctx, int64_t n, int64_t row0, int64_t n_local,
                      const int32_t *indptr, const int32_t *indices, const float *data,
                      const int32_t *indptr_t, const int32_t *indices_t, const float *data_t,
                      gemb_graph **out);
int gemb_graph_free(gemb_graph *g);

/* Test hook for the dominant kernel:  Y = alpha * op(A) * X + gamma * Xself + delta * X0
 * (Xself / X0 may be NULL: that term is left out; the Horner sweep is gamma = 0, delta = 1, the Chebyshev step
 * passes Xself = the local rows of X).  X is the full n x b block, Xself, X0 and Y are the n_local x b row shards;
 * all HOST, row-major fp32.  b must be a multiple of 4, <= 1024. */
int gemb_spmm(gemb_graph *g, int transpose, int b, float alpha, const float *X, float gamma, const float *Xself,
              float delta, const float *X0, float *Y);
/* The same with the fourth epilogue operand of spectral_mode 2's Chebyshev step (single GPU):
 * Y = alpha * op(A) * X + gamma * Xself + delta * X0 + eps * X1; X1 == NULL is gemb_spmm, else Xself and X0 are needed. */
int gemb_spmm4(gemb_graph *g, int transpose, int b, float alpha, const float *X, float gamma, const float *Xself,
               float delta, const float *X0, float eps, const float *X1, float *Y);
/* The sweep with a per-row scale, as the first sweep of spectral_mode 4 (Adamic-Adar) runs it, on light and heavy rows:
 * Y = alpha * diag(rscale) * op(A) * X.  X and Y are n x b, rscale n floats; all HOST.  Single GPU (row0 = 0,
 * n_local = n, no communicator).  b must be a multiple of 4, <= 1024. */
int gemb_spmm_scaled(gemb_graph *g, int transpose, int b, float alpha, const float *X, const float *rscale, float *Y);

/* Test hook for the tensor-core contraction: G (b1 x b2, fp64, row-major) = P^T Q over n rows; P, Q host
 * fp32 row-major (Q == NULL means Q = P).  use_tensor_cores: 1 = wgmma kernel (GEMB_ERR_UNSUPPORTED if the
 * shape does not fit it), 0 = CUDA-core fp32 kernel. */
int gemb_gram(gemb_ctx *ctx, int64_t n, const float *P, int b1, const float *Q, int b2, int use_tensor_cores,
              double *G_out);

/* Test hook for the tall-skinny product Out (n x b2) = Q (n x b1) * M (b1 x b2), host fp32 row-major buffers.
 * use_tensor_cores: 1 = wgmma kernel, 0 = CUDA-core kernel. */
int gemb_apply(gemb_ctx *ctx, int64_t n, const float *Q, int b1, const float *M, int b2, int use_tensor_cores,
               float *Out);

/* Test hooks for the single-CTA fp64 factorizations of the b x b matrices (1 <= b <= 1024; all HOST, row-major).
 * The kernel variant is chosen by b, as in the solvers.
 * chol_inverse: G symmetric -> Minv = R^-1 (upper triangular) with G = R^T R, as fp64 and as fp32 (the fp32 copy is
 *   the fp64 result rounded); a column whose pivot of the diagonally scaled matrix D^-1/2 G D^-1/2 is <= 1e-5 is
 *   dropped: its column of Minv is 0.  *rank_out = number of kept columns.
 * eigh: G symmetric -> eigenvalues w (b, ascending) and eigenvectors Z (b x b, column j <-> w[j]) by cyclic Jacobi,
 *   stopping when ||offdiag||_F <= rel_tol * ||G||_F (at most 30 sweeps). */
int gemb_chol_inverse(gemb_ctx *ctx, int b, const double *G, double *Minv64_out, float *Minv32_out, int *rank_out);
int gemb_eigh(gemb_ctx *ctx, int b, const double *G, double rel_tol, double *w_out, double *Z_out);

/* ---- HOPE.  Replaces hope.py:29-36: S = (I - beta A)^-1 beta A (or, by spectral_mode, another proximity) is never formed; its top
 * k = d/2 singular triplets come from a block subspace iteration with Rayleigh-Ritz whose
 * operator applications are CSR SpMM sweeps (Katz/Horner sweeps of S and S^T in general; a Chebyshev
 * filter in A itself when A is symmetric, since then S = f(A)).  Output convention = the reference:
 * X = [U sqrt(Sigma) | V sqrt(Sigma)], sigma ASCENDING (scipy svds order, SURVEY F3). */
typedef struct {
    uint32_t struct_size;  /* = sizeof(gemb_hope_opts) */
    int32_t oversample;    /* extra block columns, default 16 (block b = min(n, d/2 + oversample)) */
    int32_t max_iters;     /* max subspace iterations, default 30 */
    int32_t min_iters;     /* default 2 */
    float tol;             /* stop when every one of the top k singular values moved by less than tol relative to
                              itself between two Rayleigh-Ritz rounds: max_j |sigma_j - sigma_j_prev| /
                              max(sigma_j, 1e-3 sigma_max) <= tol; default 1e-6 */
    int32_t katz_terms;    /* Horner terms J; 0 = choose so that (beta*||A||_2)^J <= katz_tol */
    float katz_tol;        /* default 1e-7 */
    uint64_t seed;         /* start block, default 1234 */
    int32_t compute_residual; /* 1: one extra Katz application to report ||S^T u - sigma v|| */
    int32_t verbose;
    int32_t algorithm;     /* 0 = auto (symmetric shard: 2, or 3 when the first Rayleigh-Ritz round shows a skewed
                              spectrum; else 1); 1 = subspace iteration on S^T S through Katz sweeps (any A);
                              2 = Chebyshev-filtered subspace iteration on A itself, S = f(A) (symmetric A only);
                              3 = thick-restart block Lanczos on A (symmetric A only; power-law spectra) */
    int32_t cheb_degree;   /* filter degree per outer iteration of algorithm 2, default 8 (spectral_mode 2: 64) */
    float cheb_range_log2; /* algorithm 2: the filter degree is lowered until the filtered block's column dynamic range
                              T_m(x_L) stays below 2^cheb_range_log2 (fp32 Gram-based orthonormalisation squares it);
                              0 = default (8) */
    int32_t stop_rule;     /* algorithms 1 and 2 (algorithm 3 always stops on its residual, whatever this says):
                              0 = change: max_j |s_j - s_j'| / max(|s_j|, 1e-3 max|s|) <= tol between two rounds, s the k
                                  singular values (spectral_mode 1: the d eigenvalues) (default);
                              1 = residual <= tol over the top k, estimated from the products the round forms anyway:
                                  algorithm 1: max_j ||S^T u_j - sigma_j v_j|| / sigma_max, from the diagonal of the
                                  Gram of S^T U (S v_j - sigma_j u_j is 0 by construction); algorithm 2:
                                  max_j |f'(l_j)| ||A v_j - l_j v_j|| / sigma_max, from z^T (AV)^T (AV) z - l^2
                                  (||S v_j - sigma_j u_j|| is at most kappa_j = (1 - beta l_j) / (1 - beta l_max) >= 1
                                  times its term); spectral_mode 1: max_j ||A v_j - l_j v_j|| / max_j |l_j|.
                                  Both are differences of fp32-accurate Gram entries: they do not resolve residuals
                                  below ~6e-4 */
    int32_t algorithm3_basis; /* algorithm 3 (thick-restart block Lanczos on A, symmetric A): maximum basis width,
                              0 = default (max(2 k_keep, 160), k_keep = k + 16 rounded up to a multiple of 16);
                              rounded up to a multiple of 16 */
    int32_t spectral_mode; /* 0 = HOPE (top d/2 singular triplets of the Katz operator).
                              1 = the d largest ALGEBRAIC eigenpairs of the uploaded symmetric matrix itself, on the same
                              Chebyshev-filtered subspace iteration (beta ignored): X_out = n x d eigenvectors in DESCENDING
                              eigenvalue order, sigma_out = the d eigenvalues.  Laplacian Eigenmaps (lap.py:26-32:
                              eigs(normalized_laplacian, k = d+1, which='SM')) = this on D^-1/2 A D^-1/2 with d+1 pairs.
                              2 = the d largest algebraic eigenpairs of the composite -M^T M, M = I - A, UNSHIFTED and never
                              formed: the upload is A = P = D^-1 W (not symmetric) together with its transpose
                              (indptr_t / indices_t / data_t; W symmetric: P^T has W's pattern with values w_ij / s_j), and
                              one application of -M^T M is two SpMM sweeps, T = X - A X and A^T T - T.  X_out = n x d
                              eigenvectors, sigma_out = the d eigenvalues l_j = -sigma_j^2 DESCENDING (sigma_j ascending: the
                              smallest singular values of M and their right singular vectors; LLE, lle.py:25-32, is this with
                              d+1 pairs).  Single GPU; algorithm 0 or 2 (beta ignored).  The spectrum bound is ||M||_2^2 by
                              power iteration on -M^T M (stats->norm2_A), raised to the largest |Ritz value|.  Both stop
                              measures are taken relative to that bound, not to each small eigenvalue:
                              stop_rule 0: max_j |l_j - l_j'| / ||M||_2^2 (round 1: not converged);  stop_rule 1: max_j ||M^T M v_j - sigma_j^2 v_j||
                              / ||M||_2^2.  Device memory: one n x b block more than modes 0 and 1 (T).  spmm_count counts
                              two sweeps per application.
                              3, 4, 5 = HOPE on another proximity S (Ou et al., KDD 2016, Table 1), same output as mode 0
                              (k = d/2 triplets of S, d even; X_out = [U sqrt(Sigma) | V sqrt(Sigma)], sigma ascending):
                              3 = common neighbours S = A A;  4 = Adamic-Adar S = A D A, D_ii = 1 / (sum_j A_ij + sum_j A_ji),
                              0 where that sum is 0 (computed on the device from A and A^T: n floats);  5 = rooted PageRank
                              S = (1 - alpha) sum_{j=0..J} (alpha P)^j ~ (1 - alpha) (I - alpha P)^-1, the upload being
                              P = D_out^-1 A and its transpose, normalised by the caller (row sums <= 1, else GEMB_ERR_ARG),
                              alpha passed in `beta`, 0 < alpha < 1.  J = ceil(log(katz_tol) / log(alpha)) (||alpha P||_inf
                              <= alpha; no power iteration), or katz_terms when given.  Modes 4 and 5 refuse negative
                              weights.  S and S^T are applied matrix-free by the general solver: algorithm 0 resolves to 1;
                              algorithms 2 and 3, a multi-GPU communicator and (mode 5) alpha outside (0, 1) are
                              GEMB_ERR_ARG before any work.  compute_residual and both stop_rules work on this S.  Modes 3
                              and 4 apply S as two sweeps (T = D op(A) X, then op(A) T; S^T takes A^T), mode 5 as J sweeps.
                              Stats: katz_terms = J (mode 5) or 0; norm2_A = 0 (no norm estimate is made); beta_used =
                              alpha (mode 5) or 0; spmm_count counts every sweep. */
} gemb_hope_opts;

typedef struct {
    uint32_t struct_size;
    int32_t iters;         /* subspace iterations performed */
    int32_t katz_terms;    /* J actually used (spectral_mode 5: the rooted-PageRank series' J; 3, 4: 0) */
    int32_t block;         /* b */
    int32_t converged;
    int32_t algorithm;     /* 1 or 2: the solver that ran */
    int64_t spmm_count;    /* SpMM sweeps executed (all of width `block` except norm estimation) */
    double spmm_ms;        /* sum of CUDA-event durations of the block-width SpMM launches */
    double spmm_bytes;     /* algorithmic bytes of ONE block-width sweep: 8*nnz + 4*(n+1) + 8*n*b
                              (SURVEY 8(d); 4*nnz less when the shard is unweighted) */
    double dense_ms;       /* Gram + apply + small factorizations */
    double comm_ms;        /* NCCL time (multi-GPU) */
    double total_ms;       /* device time of the whole call (events), excluding H2D/D2H */
    double h2d_ms, d2h_ms;
    float norm2_A;         /* estimated ||A||_2 (spectral_mode 2: ||M||_2^2; spectral_modes 3-5: 0, not estimated) */
    float ritz_change;     /* algorithms 1 and 2: the last round's change measure (stop_rule 0 above), whichever rule
                              stopped; algorithm 3: the last restart's residual estimate (= resid_est) */
    float resid_max;       /* max_j ||S^T u_j - sigma_j v_j|| / sigma_max (compute_residual=1; spectral_modes 0, 3-5) */
    float resid_est;       /* the residual estimate of the last round (stop_rule 1 above; algorithm 3: max_j
                              |f'(l_j)| ||A v_j - l_j v_j|| / sigma_max from the Lanczos coupling block, computed for
                              either stop_rule), else -1 */
    int32_t mg_mode;       /* 0 = single GPU; 1 = all-gather of the block per sweep; 2 = needed-rows-only exchange over
                              NVLink peer memory (CUDA IPC): rows are stored into the peers' halo slots by the kernel
                              that produces them.  3 (fp16 halo copies) is no longer produced. */
    int64_t halo_rows;     /* mg_mode 2: distinct remote rows this shard references */
    int64_t push_rows;     /* mg_mode 2: (row, peer) pairs this rank stores per exchanged block */
    int64_t pushes;        /* mg_mode 2: blocks exchanged in this call (NVLink bytes out = pushes*push_rows*4*block) */
    float beta_used;       /* the beta the solve ran with (differs from the argument when that was negative;
                              spectral_mode 5: alpha; 1-4: 0) */
    double push_bytes;     /* mg_mode 2: bytes this rank stored into its peers over NVLink in this call */
} gemb_hope_stats;

/* X_out: n_local x d host buffer, or NULL to leave the result on the device (bench `value`).
 * sigma_out: d/2 floats (ascending) or NULL.
 * beta > 0: hope.py's beta.  beta < 0: beta = |beta| / ||A||_2, ||A||_2 (= rho(A) for symmetric A) estimated by power
 * iteration inside the call -- BASELINE.json configs[3] prescribes beta = 0.5 / rho_hat(A); stats->beta_used reports it. */
int gemb_hope(gemb_graph *g, int d, float beta, const gemb_hope_opts *opts, float *X_out,
              float *sigma_out, gemb_hope_stats *stats);

/* Test hook: one application of the operator gemb_hope solves for opts->spectral_mode, through the same option checks
 * and device set-up (negative-weight and row-sum refusals, D, the rooted-PageRank J):
 *   modes 0, 3, 4, 5: Y = S X, or S^T X (transpose), S as spectral_mode describes it -- mode 0 the Katz series
 *                     sum_{j=1..J} (beta A)^j with J = opts->katz_terms, which must be > 0 (no norm estimate is made),
 *                     and beta >= 0;
 *   modes 1, 2:       Y = Op X, the symmetric solver's operator (A, or the composite -M^T M); transpose is ignored.
 * X and Y are n x b, b a multiple of 4, <= 1024; all HOST.  *J_out (may be NULL): the series' terms used (modes 0 and 5),
 * else 0.  Single GPU (row0 = 0, n_local = n, no communicator). */
int gemb_hope_apply(gemb_graph *g, const gemb_hope_opts *opts, float beta, int transpose, int b, const float *X,
                    float *Y, int *J_out);

/* The diagnostic hope.py:38-40 prints: || U diag(s) V^T - S ||_F = || X1 X2^T - S ||_F with S = (I - beta A)^-1 beta A.
 * X: host, n x d row-major fp32 (the embedding gemb_hope returned).  S is never stored whole:
 *   n_probe <= 0 : exact -- S is applied to the identity in column panels (n sweeps' worth of work: meant for
 *                  n <= ~10^4, the sizes at which the reference can run at all);
 *   n_probe  > 0 : Hutchinson estimate sqrt(mean_j ||(X1 X2^T - S) z_j||^2) over n_probe Rademacher vectors
 *                  (SURVEY H8), relative standard error ~ sqrt(2 / n_probe).
 * S takes the Katz terms of gemb_hope's general solver (a directed graph with beta ||A||_2 >= 1 is accepted when the
 * series converges, i.e. beta rho(A) < 1); GEMB_ERR_DIVERGE when it does not.
 * Single GPU (the graph uploaded with row0 = 0, n_local = n). */
int gemb_hope_svd_error(gemb_graph *g, int d, float beta, const float *X, int n_probe, uint64_t seed,
                        double *err_out);

/* ---- node2vec.  Replaces the SNAP executable GEM shells out to (node2vec.py:31-48):
 * PreprocessTransitionProbs (bin@0x4127f0), node2vec() walks (bin@0x40c420),
 * LearnEmbeddings/TrainModel (bin@0x40ea30 / 0x40d6a0), WriteOutput + loadEmbedding
 * (graph_util.py:161-169).  p = q = 1 uses first-order tables (one per node); any other p, q > 0 builds the reference's
 * second-order tables -- one alias table per directed edge (t -> v) over v's out-neighbours, sum_(t->v) outdeg(v) entries
 * of 12 bytes -- on the device (GEMB_ERR_NOMEM with the size when they do not fit in HBM; the reference keeps the same
 * tables in host memory).
 *
 * The graph must be uploaded single-GPU style (row0 = 0, n_local = n) with every row's column
 * ids sorted ascending (SNAP adjacency order).  weights64: fp64 edge weights in CSR order or
 * NULL for 1.0 (the reference parses the "%f" text into doubles; alias tables are built in fp64
 * so that walks are bit-exact against oracle/n2v_oracle.c). */
int gemb_n2v_alias(gemb_graph *g, const double *weights64, int32_t *K_out /* nnz */,
                   double *U_out /* nnz */);

typedef struct {
    uint32_t struct_size;
    double alias_ms, shuffle_ms, walk_ms, vocab_ms, sgns_ms, total_ms, h2d_ms, d2h_ms, comm_ms;
    int64_t n_tokens;      /* vocabulary size V (includes the phantom token 0 if walks were padded) */
    int64_t n_walks;       /* walks generated by this rank */
    int64_t pairs;         /* (centre, context) pairs trained by this rank */
    double sgns_bytes;     /* algorithmic bytes: pairs * 14 rows * 4*d (SURVEY 8(d)) */
    double walk_bytes;     /* 24 B per transition */
} gemb_n2v_stats;

/* Walks only (parity hook).  nids: the N start nodes in SNAP node-table order (first appearance
 * in the edge list).  seed: the TRnd seed (the binary uses time(NULL)).  Walk w = i*N + j
 * (round i, shuffled position j) reads the Park-Miller stream at offset
 * (i+1)*(N-1) + w*(2*walk_len-3)  -- identical to the single-threaded binary whenever no walk
 * hits a dead end (oracle mode 1).  Walks [w_begin, w_end) are generated;
 * walks_out: (w_end-w_begin) x walk_len int32 host buffer (zero padded after a dead end). */
int gemb_n2v_walks(gemb_graph *g, const double *weights64, const int32_t *nids, int64_t N,
                   int walk_len, int num_walks, double p, double q, int32_t seed, int64_t w_begin,
                   int64_t w_end, int32_t *walks_out, gemb_n2v_stats *stats);

/* Full pipeline.  X_out: n_rows x d host fp32 (row = node id, like loadEmbedding; rows of ids
 * that never appear stay 0) or NULL.  sequential != 0 trains with ONE warp consuming the single
 * TRnd(seed) stream in program order (parity mode: follows oracle/n2v_oracle.c up to fp32
 * rounding); sequential == 0 is the Hogwild production mode.  d <= 512.  Every warp keeps its walk
 * in shared memory, so walk_len <= (the device's opt-in shared memory per block) / (4 * warps per
 * block): 1 warp in sequential mode, 4 in Hogwild mode (58 112 and 14 528 on an H100).  Both
 * limits are checked before any work (GEMB_ERR_UNSUPPORTED). */
int gemb_node2vec(gemb_graph *g, const double *weights64, const int32_t *nids, int64_t N, int d,
                  int walk_len, int num_walks, int con_size, int max_iter, double p, double q,
                  int32_t seed, int sequential, int64_t n_rows, float *X_out,
                  gemb_n2v_stats *stats);

/* ---- reconstruction and its evaluation (SURVEY 8(f) rank 1; the step after learn_embedding in tests/fit_model.py:10).
 * gemb_recon_create replaces the n^2 get_edge_weight calls of static_graph_embedding.py:48-65: A_hat = L R^T with a
 * zero diagonal, ON THE DEVICE, made of 64-column panels (n x 64 fp32 each, n * 256 bytes) in BLOCKS of consecutive
 * panels.  When the whole n x n matrix fits in 0.9 x (free + cached) device memory beside X and the factors, it is one
 * block, made at create and kept: every call below reads it.  Otherwise the handle keeps X and the factors plus one
 * block buffer of as many panels as fit (leaving 1 GiB + 16 bytes per node for the calls' scratch), and every call
 * regenerates the blocks in order -- a PASS, costing the product once more (4 n^2 bytes written and read):
 *   ranks: 2 passes (the true edges' scores, then the counting); top: 1 pass for the count when every candidate is
 *   returned (max_k < 0 or max_k >= the count), else 2, and 1 more for the entries; pairs: the blocks that hold a
 *   pair's column; dense: 1 pass.  The scores are the same bits in both modes.  GEMB_ERR_NOMEM only when not even one
 *   panel fits.
 *   kind = 1 (or any value other than 0 and 2): L = X[:, :d/2], R = X[:, d/2:]
 *                                                 (HOPE.get_edge_weight, hope.py:43-44)
 *   kind = 0: L = R = X                          (node2vec.get_edge_weight, node2vec.py:56-57)
 *   kind = 2: score exp(-delta_ij), delta_ij = |x_i - x_j|^2 summed as sum_k (x_ik - x_jk)^2 in fp32 (exactly 0 for
 *             equal rows)   (LaplacianEigenmaps / LocallyLinearEmbedding.get_edge_weight, lap.py:39-42, lle.py:37-40).
 *             The ranking, n_pred and top-k below order by delta ascending (= score descending) and count a pair as
 *             predicted when delta <= 745.1332f, where the fp64 score is still > 0.  dense, pairs and the w_out of
 *             top return delta, not the score: +inf on the diagonal and where delta > 745.1332f, so that
 *             score = exp(-out) holds for every entry.  A non-finite X is GEMB_ERR_ARG.
 * X: host, n x d row-major fp32. */
#define GEMB_RECON_DOT 0
#define GEMB_RECON_SPLIT 1
#define GEMB_RECON_GAUSS 2
typedef struct gemb_recon gemb_recon;
int gemb_recon_create(gemb_ctx *ctx, const float *X, int64_t n, int d, int kind, gemb_recon **out);
/* gemb_recon_create with the block size given (test hook): panels_per_block > 0 makes blocks of that many panels (one
 * block when they cover all ceil(n / 64) panels; GEMB_ERR_NOMEM when they do not fit), 0 chooses as gemb_recon_create
 * does. */
int gemb_recon_create_blocked(gemb_ctx *ctx, const float *X, int64_t n, int d, int kind, int64_t panels_per_block,
                              gemb_recon **out);
/* The block layout: panels per block and number of blocks (1: the matrix stays on the device between calls). */
int gemb_recon_info(gemb_recon *r, int64_t *panels_per_block, int64_t *blocks);
int gemb_recon_free(gemb_recon *r);

/* The dense matrix get_reconstructed_adj returns (static_graph_embedding.py:48-65): adj_out host, n x n row-major
 * (kind 2: delta, see above). */
int gemb_recon_dense(gemb_recon *r, float *adj_out);

/* A_hat[i[t]][j[t]] for m pairs (0 on the diagonal; kind 2: delta, +inf on the diagonal): the sampled-pairs branch
 * of get_edge_list_from_adj_mtrx (evaluation_util.py:25-28) and the weighted reconstruction error
 * (evaluate_graph_reconstruction.py:37-40). */
int gemb_recon_pairs(gemb_recon *r, const int32_t *i, const int32_t *j, int64_t m, float *out);

/* computeMAP (metrics.py:28-46) without sorting.  The true graph is a CSR by node id (host, int32).  For every
 * true edge e = (i -> j): rank_out[e] = 1-based position of (i, j) in node i's predicted edges sorted by weight
 * (descending, ties in ascending j -- Python's stable sort), or 0 when (i, j) is not a predicted edge (j == i,
 * A_hat[i][j] <= 0, or j < i with is_undirected -- evaluation_util.py:29-35).  n_pred_row[i] = number of
 * predicted edges with source i.  AP and MAP follow from the ranks on the host. */
int gemb_recon_ranks(gemb_recon *r, const int32_t *indptr, const int32_t *indices, int is_undirected,
                     int32_t *rank_out, int32_t *n_pred_row);

/* computePrecisionCurve (metrics.py:6-25): the predicted edges that can be among the max_k heaviest (max_k < 0: all
 * of them), i.e. every valid entry >= the max_k-th largest value; UNORDERED.  *m_out = their number.  Call with
 * cap = 0 to get the count, then with cap >= count and three arrays of that length; the caller orders them
 * (weight descending, then i, then j ascending = the reference's stable sort of the row-major list; kind 2: w_out
 * is delta, ordered ascending). */
int gemb_recon_top(gemb_recon *r, int is_undirected, int64_t max_k, int64_t cap, int32_t *i_out, int32_t *j_out,
                   float *w_out, int64_t *m_out);

/* Link prediction: rank held-out edges among the candidates that are not training edges.  Replaces, on top of the
 * two calls above, the train/test split's consequence in the evaluation -- the predicted list filtered edge by edge,
 * [e for e in pred if not train.has_edge(e[0], e[1])], after split_di_graph_to_train_test (evaluation_util.py:39-53).
 * ex_indptr (n + 1 offsets) / ex_indices (host, int32, strictly ascending column ids per row) is the exclusion, copied
 * to the device; ex_indptr == NULL clears it.  While it is set, gemb_recon_ranks and gemb_recon_top report their
 * results over the candidates NOT in it: a true edge that is itself excluded gets rank 0, n_pred_row counts only the
 * remaining candidates, and top selects among them.  Without an exclusion both are unchanged.  Setting or clearing it
 * drops the cached top selection.  Cost: ranks and top run their usual passes with the excluded entries of each block
 * set to 0 while that block is counted -- one scatter over the block's share of the exclusion before and one after,
 * which puts the values back, so gemb_recon_dense and gemb_recon_pairs never see the zeros. */
int gemb_recon_exclude(gemb_recon *r, const int32_t *ex_indptr, const int32_t *ex_indices);

/* ---- node classification (upstream GEM's evaluateNodeClassification: OneVsRestClassifier(LogisticRegression()) and
 * its TopKRanker; not in the reference checkout).  gemb_nc_fit replaces the one-vs-rest fit: for every label c, with
 * s_i = +1 when row i carries c and -1 otherwise, the minimiser of
 *     f_c(w, b) = 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w . x_i + b)))      (sklearn's objective; b not penalised)
 * by batched L-BFGS (memory 10) on the device, labels in panels of 128.  Class c stops when
 * max|grad f_c| <= tol * max|grad f_c(0, 0)|, or after max_iter accepted steps.
 * X: host, n x d row-major fp32 (the training rows).  indptr (n + 1, int64) / labels (int32, strictly ascending per
 * row, in [0, L)): the rows' labels.  W_out: L x (d + 1) fp64, row c = (w_c, b_c); a label with no positive training
 * row gets w = 0, b = -inf (p = 0), one that every training row carries w = 0, b = +inf (p = 1) -- sklearn's
 * _ConstantPredictor.  iters_out (L, or NULL): accepted L-BFGS steps per label.  status_out (L, or NULL):
 * GEMB_NC_CONVERGED, _CONSTANT, _MAXITER (max_iter reached) or _STALLED (no acceptable step in 40 line-search trials).
 * Two calls on the same device give the same bits. */
#define GEMB_NC_CONVERGED 1
#define GEMB_NC_CONSTANT 2
#define GEMB_NC_MAXITER 3
#define GEMB_NC_STALLED 4
typedef struct {
    uint32_t struct_size;  /* = sizeof(gemb_nc_stats) */
    int32_t panels;        /* label panels of <= 128 solved */
    int64_t evaluations;   /* panel function / gradient evaluations (each: apply, residual, Gram, L-BFGS step) */
    int32_t max_iters;     /* largest iters_out */
    int64_t unconverged;   /* labels stopped by max_iter or a stalled line search */
    int64_t constant;      /* labels that are constant on the training rows */
    double eval_bytes;     /* compulsory HBM bytes of the evaluations' launches: per evaluation
                              n (8 d + 16 P + 8) + 4 nnz (P = panel width) */
    double total_ms;       /* device time of the call (events), uploads included */
} gemb_nc_stats;
int gemb_nc_fit(gemb_ctx *ctx, int64_t n, int d, const float *X, const int64_t *indptr, const int32_t *labels, int L,
                double C, double tol, int max_iter, double *W_out, int32_t *iters_out, int32_t *status_out,
                gemb_nc_stats *stats);

/* The TopKRanker prediction: for test row i (X: host, m x d fp32) the k_i = koff[i + 1] - koff[i] labels with the
 * largest p = 1 / (1 + exp(-(w_c . x_i + b_c))) (fp64 from the decision value, whose product w . x is fp32), exact
 * ties to the larger label index.  W: L x (d + 1) fp64 as gemb_nc_fit returns it.  pred_out (koff[m] int32): row i's
 * labels at koff[i] .. koff[i + 1] - 1, highest p first.  A row with k_i = 0 gets nothing here (upstream predicts every
 * label for it; the caller fills that in). */
int gemb_nc_topk(gemb_ctx *ctx, int64_t m, int d, const float *X, int L, const double *W, const int64_t *koff,
                 int32_t *pred_out);

/* ---- weakly connected components and the largest one (get_lcc, graph_util.py:29-34: the largest weakly connected
 * component, relabelled 0..k-1 in node order).  One handle, so the CSR is uploaded once.
 * gemb_cc_create uploads the n x n CSR (host: indptr n + 1 int64 with indptr[0] = 0, non-decreasing; indices int32 in
 * [0, n); 0 <= n < 2^31) and labels it: every stored edge joins its two ends whatever its direction (self loops,
 * isolated vertices and one-way edges allowed).  Bad input is GEMB_ERR_ARG before any device work.  Two calls give the
 * same bits.
 * gemb_cc_info: the number of components; the LCC -- the largest, the one with the smallest vertex id on a tie
 * (= max(nx.weakly_connected_components(G), key=len) over row order) -- by its smallest vertex id, its vertex count
 * and its stored edges.  n = 0: 0 components, lcc_root -1, size 0.  Any output pointer may be NULL.
 * gemb_cc_labels: comp_out (n int32) = component number of every vertex, 0..n_comp-1 in the order of each
 * component's smallest vertex.
 * gemb_cc_lcc: the LCC as a CSR.  node_l_out (lcc_size int64): old row of every new row, ascending (new id = rank of
 * the old id among the LCC's vertices, so column ids stay sorted within each row); indptr_out (lcc_size + 1 int64);
 * indices_out (lcc_nnz int32, new ids); data (nnz fp64, or NULL = unit weights): data_out (lcc_nnz) gets the weights
 * of the kept edges (not written when data is NULL).
 * gemb_cc_times: device time of the labelling in gemb_cc_create and of the last gemb_cc_lcc's extraction (events
 * around the kernels; the host copies are outside). */
typedef struct gemb_cc gemb_cc;
int gemb_cc_create(gemb_ctx *ctx, int64_t n, const int64_t *indptr, const int32_t *indices, gemb_cc **out);
int gemb_cc_info(gemb_cc *cc, int64_t *n_comp, int64_t *lcc_root, int64_t *lcc_size, int64_t *lcc_nnz);
int gemb_cc_labels(gemb_cc *cc, int32_t *comp_out);
int gemb_cc_lcc(gemb_cc *cc, const double *data, int64_t *node_l_out, int64_t *indptr_out, int32_t *indices_out,
                double *data_out);
int gemb_cc_times(gemb_cc *cc, double *label_ms, double *extract_ms);
int gemb_cc_free(gemb_cc *cc);

/* ---- t-SNE to two dimensions: the TSNE(n_components=2).fit_transform(node_pos) of plot_embedding2D
 * (visualize_embedding.py:7-12), restated from sklearn 1.9's defaults (init='pca', method='barnes_hut', euclidean).
 * X: host, n x d row-major fp32, finite, n >= 2, d >= 1.  Y_out: host, n x 2 fp32.
 *   kNN          k = min(n - 1, floor(3 perplexity + 1)) exact nearest rows, selected by fp32 d^2 = sum_c (x_c - y_c)^2,
 *                ties to the lower index, the row itself excluded (_t_sne.py TSNE._fit; NearestNeighbors is brute force
 *                for d > 15); the k d^2 are then summed in fp64 and rounded to fp32, as sklearn rounds its fp64 distances.
 *                k <= 320 (perplexity < 106.33 for n > 320), else GEMB_ERR_UNSUPPORTED.
 *   calibration  _utils.pyx _binary_search_perplexity, in fp64.
 *   joint P      _t_sne.py _joint_probabilities_nn: (P_cond + P_cond^T) / sum, fp64, exact zeros dropped.
 *   start        PCA(n_components=2) scores with svd_flip(u_based_decision=False) signs, column 0 scaled to standard
 *                deviation 1e-4 (TSNE._fit, init='pca').  d <= 1024 (the width of the Jacobi eigensolver), else
 *                GEMB_ERR_UNSUPPORTED.
 *   gradient     _barnes_hut_tsne.pyx gradient on _quad_tree.pyx's cells, times c = 2 (dof + 1) / dof = 4.
 *   optimiser    _t_sne.py _gradient_descent as TSNE._tsne runs it: 250 iterations (or max_iter, if fewer) at momentum
 *                0.5 with P times early_exaggeration, then momentum 0.8 up to max_iter; the KL error and the
 *                n_iter_without_progress / min_grad_norm stops every 50 iterations.  max_iter = 0 returns the start.
 * Refused with GEMB_ERR_ARG before any device work: X not finite, perplexity outside (0, n), early_exaggeration or
 * learning_rate <= 0 (the caller resolves sklearn's 'auto', max(n / early_exaggeration / 4, 50)), angle outside [0, 1],
 * negative max_iter, n_iter_without_progress or min_grad_norm.  Two calls give the same bits. */
typedef struct {
    uint32_t struct_size;            /* = sizeof(gemb_tsne_opts) */
    int32_t max_iter;                /* sklearn: 1000 */
    int32_t n_iter_without_progress; /* sklearn: 300 */
    double perplexity;               /* sklearn: 30 */
    double early_exaggeration;       /* sklearn: 12 */
    double learning_rate;            /* > 0 */
    double min_grad_norm;            /* sklearn: 1e-7 */
    double angle;                    /* sklearn: 0.5 */
} gemb_tsne_opts;
typedef struct {
    uint32_t struct_size;  /* = sizeof(gemb_tsne_stats) */
    int32_t n_neighbors;   /* k */
    int32_t n_iter;        /* TSNE.n_iter_: the last iteration run (-1 when max_iter = 0) */
    int64_t nnz_P;         /* entries of the joint P */
    double kl_divergence;  /* the KL error of the last iteration (TSNE.kl_divergence_); 0 when max_iter = 0 */
    double knn_ms, calib_ms, sym_ms, pca_ms, opt_ms, total_ms;   /* host clock per stage, each ending in a synchronise */
    double tree_ms, grad_ms;   /* device time (events) summed over the iterations: quadtree build; repulsive walk,
                                  attractive sweep and update */
} gemb_tsne_stats;
int gemb_tsne(gemb_ctx *ctx, int64_t n, int d, const float *X, const gemb_tsne_opts *opts, float *Y_out,
              gemb_tsne_stats *stats);

/* Test hook: the affinities of gemb_tsne.  Call with cap = 0 to get *k_out and *nnz_out, then with cap >= nnz and
 * every array: knn_idx_out / knn_d2_out (n x k, each row ascending by (d^2, index)), p_cond_out (n x k, the conditional
 * P of _binary_search_perplexity in the same order), and the joint P as CSR (p_indptr_out n + 1, p_indices_out and
 * p_val_out nnz, column ids ascending per row). */
int gemb_tsne_affinities(gemb_ctx *ctx, int64_t n, int d, const float *X, double perplexity, int64_t cap,
                         int32_t *knn_idx_out, float *knn_d2_out, double *p_cond_out, int64_t *p_indptr_out,
                         int32_t *p_indices_out, double *p_val_out, int32_t *k_out, int64_t *nnz_out);

/* Test hook: _kl_divergence_bh at positions Y (host, n x 2 fp32) for the joint P given as CSR (host; p_indptr n + 1
 * int64, p_indices int32, p_val fp64): grad_out (n x 2, including the factor 4) and *kl_out (may be NULL).  angle 0
 * gives the exact gradient except for the pairs sklearn's tree also leaves out (points within 1e-6 of each other). */
int gemb_tsne_gradient(gemb_ctx *ctx, int64_t n, const float *Y, const int64_t *p_indptr, const int32_t *p_indices,
                       const double *p_val, double angle, float *grad_out, double *kl_out);

/* ---- wire formats (SURVEY 8(f) rank 2): the reference's text files, read and written natively and in parallel.
 * HOST code only -- these entry points need no GPU.
 * Edge list: every non-blank line "src dst [weight]" (loadGraphFromEdgeListTxt, graph_util.py:143-158: exactly three
 * tokens -> float(weight), otherwise 1.0).  `skip` leading lines are ignored (the two header lines that
 * saveGraphToEdgeListTxt writes, graph_util.py:131-132).  scan counts the edge lines; parse fills caller arrays of
 * that length (w may be NULL); *all_unit = 1 when no weight differs from 1.0. */
int gemb_edge_list_scan(const char *path, int64_t skip, int64_t *n_edges);
int gemb_edge_list_parse(const char *path, int64_t skip, int64_t n_edges, int64_t *src, int64_t *dst, double *w,
                         int32_t *all_unit);
/* One "%d %d %f\n" per edge (saveGraphToEdgeListTxtn2v, graph_util.py:137-140); header_nodes >= 0 first writes
 * "<nodes>\n<edges>\n" (saveGraphToEdgeListTxt, :129-134).  w == NULL writes 1.000000. */
int gemb_edge_list_write(const char *path, int64_t n_edges, const int64_t *src, const int64_t *dst, const double *w,
                         int64_t header_nodes);
/* ".emb": "<rows> <d>" then "<id> v1 ... vd" (loadEmbedding, graph_util.py:161-169; written by SNAP's WriteOutput,
 * bin@0x406ef0, with 6 significant digits).  read: X == NULL returns only rows and d; otherwise X is rows x d fp64,
 * zeroed by the caller, row = id.  write: ids == NULL means rows 0..n_ids-1; X is indexed by id. */
int gemb_emb_read(const char *path, int64_t *rows, int32_t *d, double *X);
int gemb_emb_write(const char *path, int64_t n_ids, const int64_t *ids, int32_t d, const double *X, int64_t header_rows);

#ifdef __cplusplus
}
#endif
#endif /* GEMB200_H */
