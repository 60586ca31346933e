/*
 * oracle/n2v_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Single-threaded, explicitly seeded CPU restatement of the SNAP `node2vec`
 * program that GEM shells out to (reference: gem/embedding/node2vec.py:27-54
 * calls the prebuilt ELF gem/c_exe/node2vec; its C++ source is NOT in the
 * reference tree).  The algorithm below was restated from the published SNAP
 * node2vec algorithm (snap-adv n2v / biasedrandomwalk / word2vec) and checked
 * against the disassembly of the unstripped binary (addresses `bin@0x...` in
 * the comments refer to gem/c_exe/node2vec) and -- bit for bit -- against the
 * binary itself run with an LD_PRELOAD `time()` shim and OMP_NUM_THREADS=1
 * (oracle/pin_n2v_oracle.py; goldens in tests/golden/n2v_bin_*.npz).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this file's shared object.  The product
 * (gem_b200/) never does.
 *
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off, no -ffast-math:
 * the fp64 operation order is part of the specification).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

/* ---------------------------------------------------------------- TRnd ---
 * Park-Miller minimal standard generator with Schrage's method
 * (bin@0x41bb0c-0x41bb40: constants 0x41a7, 0x1f31d, 0xb14, 0x7fffffff). */
typedef struct { int32_t seed; } trnd_t;

static inline int32_t trnd_next(trnd_t *r) {
    int32_t s = r->seed;
    s = 16807 * (s % 127773) - 2836 * (s / 127773);
    if (s <= 0) s += 2147483647;
    r->seed = s;
    return s;
}
/* TRnd::GetUniDevInt(Range) bin@0x41baf0 */
static inline int32_t trnd_int(trnd_t *r, int32_t range) {
    int32_t s = trnd_next(r);
    return range == 0 ? s : s % range;
}
/* TRnd::GetUniDev(): seed / double(m) */
static inline double trnd_uni(trnd_t *r) {
    return (double)trnd_next(r) / 2147483647.0;
}

/* Skip-ahead: state after k steps from seed s is 16807^k * s mod (2^31-1). */
static uint64_t mulmod31(uint64_t a, uint64_t b) { return (a * b) % 2147483647ULL; }
int32_t n2v_oracle_rng_skip(int32_t seed, uint64_t k) {
    uint64_t base = 16807, acc = 1;
    while (k) { if (k & 1) acc = mulmod31(acc, base); base = mulmod31(base, base); k >>= 1; }
    return (int32_t)mulmod31(acc, (uint64_t)seed);
}

/* ----------------------------------------------------- Vose alias table ---
 * GetNodeAlias bin@0x4115f0: P (normalised) -> K (int), U (double).
 * Under/Over are LIFO stacks; order of pushes is part of the spec. */
static void vose_alias(const double *P, int64_t N, int32_t *K, double *U,
                       int32_t *stack /* scratch, 2*N */) {
    int32_t *under = stack, *over = stack + N;
    int64_t nu = 0, no = 0;
    for (int64_t i = 0; i < N; i++) { K[i] = 0; U[i] = 0; }
    for (int64_t i = 0; i < N; i++) {
        U[i] = P[i] * (double)N;
        if (U[i] < 1) under[nu++] = (int32_t)i; else over[no++] = (int32_t)i;
    }
    while (nu > 0 && no > 0) {
        int32_t small = under[--nu];
        int32_t large = over[--no];
        K[small] = large;
        U[large] = U[large] + U[small] - 1;
        if (U[large] < 1) under[nu++] = large; else over[no++] = large;
    }
    while (nu > 0) U[under[--nu]] = 1;
    while (no > 0) U[over[--no]] = 1;
}

/* AliasDrawInt bin@0x411360: two draws. */
static inline int64_t alias_draw(const int32_t *K, const double *U, int64_t N, trnd_t *r) {
    int64_t X = (int64_t)(trnd_uni(r) * (double)N);
    double Y = trnd_uni(r);
    return Y < U[X] ? X : K[X];
}

/* Graph: CSR over node ids 0..n-1, out-neighbours of each row SORTED BY ID
 * (SNAP keeps adjacency vectors sorted), fp64 weights. */

/* First-order tables (p = q = 1): PreprocessNode bin@0x411f40 with
 * ParamP = ParamQ = 1 -> the table of edge (t,v) depends only on v:
 * P[j] = w(v,x_j) / sum_j w(v,x_j), summed in neighbour order. */
int n2v_oracle_alias_first_order(int64_t n, const int64_t *indptr, const double *w,
                                 int32_t *K, double *U) {
    int64_t maxdeg = 0;
    for (int64_t v = 0; v < n; v++) { int64_t d = indptr[v+1]-indptr[v]; if (d > maxdeg) maxdeg = d; }
    double *P = (double*)malloc(sizeof(double) * (maxdeg + 1));
    int32_t *st = (int32_t*)malloc(sizeof(int32_t) * 2 * (maxdeg + 1));
    if (!P || !st) return -1;
    for (int64_t v = 0; v < n; v++) {
        int64_t s = indptr[v], d = indptr[v+1] - s;
        double psum = 0;
        for (int64_t j = 0; j < d; j++) { P[j] = w[s+j]; psum += w[s+j]; }
        for (int64_t j = 0; j < d; j++) P[j] /= psum;
        vose_alias(P, d, K + s, U + s, st);
    }
    free(P); free(st);
    return 0;
}

static int has_edge(const int64_t *indptr, const int32_t *idx, int64_t u, int32_t x) {
    int64_t lo = indptr[u], hi = indptr[u+1];
    while (lo < hi) { int64_t m = (lo + hi) >> 1; if (idx[m] < x) lo = m + 1; else hi = m; }
    return lo < indptr[u+1] && idx[lo] == x;
}

/* Second-order table of edge (t -> v), PreprocessNode bin@0x411f40:
 * unnormalised pi(x) = w(v,x) * {1/p if x==t; 1 if x in N_out(t); 1/q else}. */
static void second_order_table(const int64_t *indptr, const int32_t *idx, const double *w,
                               int64_t t, int64_t v, double p, double q,
                               double *P, int32_t *K, double *U, int32_t *st) {
    int64_t s = indptr[v], d = indptr[v+1] - s;
    double psum = 0;
    for (int64_t j = 0; j < d; j++) {
        int32_t x = idx[s+j];
        double val;
        if (x == t) val = w[s+j] / p;
        else if (has_edge(indptr, idx, t, x)) val = w[s+j];
        else val = w[s+j] / q;
        P[j] = val; psum += val;
    }
    for (int64_t j = 0; j < d; j++) P[j] /= psum;
    vose_alias(P, d, K, U, st);
}

/* One walk, SimulateWalk bin@0x411a00.  Row `out` (walk_len int32) must be
 * zero-initialised by the caller (WalksVV is zero-initialised: early-stopped
 * walks are padded with node id 0, SURVEY F10). */
typedef struct {
    int64_t n; const int64_t *indptr; const int32_t *idx; const double *w;
    double p, q; int first_order;
    const int32_t *K1; const double *U1;      /* first-order tables (or NULL) */
    double *P; int32_t *K; double *U; int32_t *st;  /* scratch, maxdeg */
} walk_ctx_t;

static void simulate_walk(const walk_ctx_t *c, int32_t start, int walk_len, trnd_t *r, int32_t *out) {
    int len = 0;
    out[len++] = start;
    if (walk_len == 1) return;
    int64_t deg = c->indptr[start+1] - c->indptr[start];
    if (deg == 0) return;
    /* step 1: uniform over out-neighbours, ignores weights (bin@0x411b31) */
    out[len++] = c->idx[c->indptr[start] + trnd_int(r, (int32_t)deg)];
    while (len < walk_len) {
        int32_t dst = out[len-1], src = out[len-2];
        int64_t s = c->indptr[dst], d = c->indptr[dst+1] - s;
        if (d == 0) return;
        int64_t nx;
        if (c->first_order) nx = alias_draw(c->K1 + s, c->U1 + s, d, r);
        else {
            second_order_table(c->indptr, c->idx, c->w, src, dst, c->p, c->q, c->P, c->K, c->U, c->st);
            nx = alias_draw(c->K, c->U, d, r);
        }
        out[len++] = c->idx[s + nx];
    }
}

/* TVec<TInt>::Shuffle bin@0x40d1a0 (Len < TInt::Mx branch at 0x40d220):
 * for j in 0..N-2: swap(j, j + GetUniDevInt(N - j)). One draw per swap. */
static void shuffle(int32_t *a, int64_t N, trnd_t *r) {
    for (int64_t j = 0; j < N - 1; j++) {
        int64_t k = j + trnd_int(r, (int32_t)(N - j));
        int32_t t = a[j]; a[j] = a[k]; a[k] = t;
    }
}

/*
 * All walks, node2vec() bin@0x40c420.
 *   nids    : the N node ids in SNAP node-table order (first appearance in the
 *             edge list), NOT modified.
 *   mode 0  : "snap-sequential": one TRnd(seed) shared by shuffles and walks,
 *             consumed in program order (== the binary with OMP_NUM_THREADS=1).
 *   mode 1  : "strided": shuffles use the same positions of the stream as mode
 *             0 would if no walk stopped early; walk (i, j) starts at stream
 *             offset  (i+1)*(N-1) + (i*N + j)*(2*walk_len-3).  Identical to
 *             mode 0 when no walk hits a dead end; well defined (and
 *             parallelisable by LCG skip-ahead) when some do.
 *   walks   : (num_walks*N) x walk_len int32, row-major, zero-filled here.
 *   order_out (nullable): num_walks x N shuffled start orders.
 */
int n2v_oracle_walks(int64_t n, const int64_t *indptr, const int32_t *idx, const double *w,
                     const int32_t *nids, int64_t N, int walk_len, int num_walks,
                     double p, double q, int32_t seed, int mode,
                     int32_t *walks, int32_t *order_out) {
    walk_ctx_t c; memset(&c, 0, sizeof c);
    c.n = n; c.indptr = indptr; c.idx = idx; c.w = w; c.p = p; c.q = q;
    c.first_order = (p == 1.0 && q == 1.0);
    int64_t nnz = indptr[n], maxdeg = 0;
    for (int64_t v = 0; v < n; v++) { int64_t d = indptr[v+1]-indptr[v]; if (d > maxdeg) maxdeg = d; }
    int32_t *K1 = NULL; double *U1 = NULL;
    if (c.first_order) {
        K1 = (int32_t*)malloc(sizeof(int32_t) * (nnz + 1)); U1 = (double*)malloc(sizeof(double) * (nnz + 1));
        if (!K1 || !U1) return -1;
        if (n2v_oracle_alias_first_order(n, indptr, w, K1, U1)) return -1;
        c.K1 = K1; c.U1 = U1;
    }
    c.P = (double*)malloc(sizeof(double) * (maxdeg + 1));
    c.K = (int32_t*)malloc(sizeof(int32_t) * (maxdeg + 1));
    c.U = (double*)malloc(sizeof(double) * (maxdeg + 1));
    c.st = (int32_t*)malloc(sizeof(int32_t) * 2 * (maxdeg + 1));
    int32_t *order = (int32_t*)malloc(sizeof(int32_t) * (N > 0 ? N : 1));
    if (!c.P || !c.K || !c.U || !c.st || !order) return -1;
    memcpy(order, nids, sizeof(int32_t) * N);
    memset(walks, 0, sizeof(int32_t) * (size_t)num_walks * N * walk_len);

    trnd_t rnd; rnd.seed = seed;
    const uint64_t per_walk = (walk_len >= 2) ? (uint64_t)(2 * walk_len - 3) : 0;
    for (int64_t i = 0; i < num_walks; i++) {
        if (mode == 1) {
            /* position of round i's shuffle in the no-dead-end stream */
            uint64_t off = (uint64_t)i * (uint64_t)(N - 1) + (uint64_t)i * (uint64_t)N * per_walk;
            rnd.seed = n2v_oracle_rng_skip(seed, off);
        }
        shuffle(order, N, &rnd);
        if (order_out) memcpy(order_out + i * N, order, sizeof(int32_t) * N);
        for (int64_t j = 0; j < N; j++) {
            if (mode == 1) {
                uint64_t off = (uint64_t)(i + 1) * (uint64_t)(N - 1)
                             + ((uint64_t)i * (uint64_t)N + (uint64_t)j) * per_walk;
                rnd.seed = n2v_oracle_rng_skip(seed, off);
            }
            simulate_walk(&c, order[j], walk_len, &rnd, walks + ((size_t)i * N + j) * walk_len);
        }
    }
    free(K1); free(U1); free(c.P); free(c.K); free(c.U); free(c.st); free(order);
    return 0;
}

/* ------------------------------------------------------------ word2vec ---
 * LearnEmbeddings bin@0x40ea30 and TrainModel bin@0x40d6a0, sequential. */
#define N2V_NEG 5
#define N2V_MAXEXP 6.0
#define N2V_EXP_PREC 10000
#define N2V_TABLE 120000  /* MaxExp * ExpTablePrecision * 2 */
#define N2V_START_ALPHA 0.025

/* TMath::Power(Base, Exp) = exp(log(Base) * Exp)  (bin@0x40e5af-0x40e5bc) */
static double tpower(double base, double ex) { return exp(log(base) * ex); }

/*
 * walks are renumbered IN PLACE to token ids by first appearance (row-major).
 * Outputs: *V_out tokens; token_node[V] = node id of token; syn_pos V x d.
 * Caller passes token_node with capacity >= n_ids (max node id + 1) and
 * syn_pos capacity >= n_ids * d.  syn_neg_out nullable (same capacity).
 * walk_streams 0: training continues the ONE TRnd(seed) stream of InitPosEmb,
 *                 walk after walk (the single-threaded binary).
 * walk_streams 1: walk wi of epoch `it` starts at position
 *                   2^30 + (it * n_walks + wi) * walk_len * (1 + 20 * win)
 *                 of TRnd(seed): the per-walk streams of the GPU's Hogwild mode
 *                 (n2v.cu, sgns_kernel).  walk_len * (1 + 20 * win) bounds the
 *                 draws of one walk: one window draw per word, ten per pair, at
 *                 most 2 * win pairs per word.  With one walk per epoch the
 *                 Hogwild result is then a deterministic function of this stream.
 */
int n2v_oracle_learn(int32_t *walks, int64_t n_walks, int walk_len, int64_t n_ids,
                     int d, int win, int iters, int32_t seed, int walk_streams,
                     int64_t *V_out, int32_t *token_node, double *syn_pos, double *syn_neg_out) {
    int64_t tot = n_walks * walk_len;
    int32_t *rn = (int32_t*)malloc(sizeof(int32_t) * (n_ids > 0 ? n_ids : 1));
    if (!rn) return -1;
    for (int64_t i = 0; i < n_ids; i++) rn[i] = -1;
    int64_t V = 0;
    for (int64_t t = 0; t < tot; t++) {
        int32_t id = walks[t];
        if (rn[id] < 0) { rn[id] = (int32_t)V; token_node[V] = id; V++; }
        walks[t] = rn[id];
    }
    /* LearnVocab bin@0x40d560 */
    int64_t *vocab = (int64_t*)calloc(V, sizeof(int64_t));
    for (int64_t t = 0; t < tot; t++) vocab[walks[t]]++;
    trnd_t rnd; rnd.seed = seed;
    /* InitPosEmb bin@0x40e270 ; InitNegEmb bin@0x40e040 */
    double *syn_neg = (double*)calloc((size_t)V * d, sizeof(double));
    for (int64_t i = 0; i < V; i++)
        for (int j = 0; j < d; j++)
            syn_pos[i * d + j] = (trnd_uni(&rnd) - 0.5) / d;
    /* InitUnigramTable bin@0x40e520 */
    int32_t *KT = (int32_t*)malloc(sizeof(int32_t) * V);
    double *UT = (double*)malloc(sizeof(double) * V);
    double *prob = (double*)malloc(sizeof(double) * V);
    int32_t *st = (int32_t*)malloc(sizeof(int32_t) * 2 * V);
    double tw = 0;
    for (int64_t i = 0; i < V; i++) { prob[i] = tpower((double)vocab[i], 0.75); tw += prob[i]; }
    for (int64_t i = 0; i < V; i++) prob[i] /= tw;
    vose_alias(prob, V, KT, UT, st);
    double *etab = (double*)malloc(sizeof(double) * N2V_TABLE);
    for (int i = 0; i < N2V_TABLE; i++) {
        double value = -N2V_MAXEXP + (double)i / (double)N2V_EXP_PREC;
        etab[i] = tpower(2.71828182845904523536, value);
    }
    double alpha = N2V_START_ALPHA;
    int64_t word_cnt = 0;
    double *neu1e = (double*)malloc(sizeof(double) * d);
    for (int it = 0; it < iters; it++) {
        for (int64_t wi = 0; wi < n_walks; wi++) {
            const int32_t *wk = walks + wi * walk_len;
            if (walk_streams) {
                const uint64_t stride = (uint64_t)walk_len * (uint64_t)(1 + 2 * win * N2V_NEG * 2);
                rnd.seed = n2v_oracle_rng_skip(seed, 0x40000000ULL + ((uint64_t)it * (uint64_t)n_walks + (uint64_t)wi) * stride);
            }
            for (int64_t wordI = 0; wordI < walk_len; wordI++) {
                if (word_cnt % 10000 == 0) {
                    alpha = N2V_START_ALPHA * (1 - word_cnt / (double)((int64_t)iters * tot + 1));
                    if (alpha < N2V_START_ALPHA * 0.0001) alpha = N2V_START_ALPHA * 0.0001;
                }
                int64_t word = wk[wordI];
                int offset = trnd_int(&rnd, 0) % win;
                for (int a = offset; a < win * 2 + 1 - offset; a++) {
                    if (a == win) continue;
                    int64_t ci = wordI - win + a;
                    if (ci < 0 || ci >= walk_len) continue;
                    int64_t cw = wk[ci];
                    for (int i = 0; i < d; i++) neu1e[i] = 0;
                    for (int j = 0; j < N2V_NEG + 1; j++) {
                        int64_t target; int label;
                        if (j == 0) { target = word; label = 1; }
                        else {
                            /* RndUnigramInt bin@0x40d5f0: first lookup goes THROUGH KTable */
                            int32_t X = KT[(int64_t)(trnd_uni(&rnd) * (double)V)];
                            double Y = trnd_uni(&rnd);
                            target = Y < UT[X] ? X : KT[X];
                            if (target == word) continue;
                            label = 0;
                        }
                        double product = 0;
                        double *sp = syn_pos + cw * d, *sn = syn_neg + target * d;
                        for (int i = 0; i < d; i++) product += sp[i] * sn[i];
                        double grad;
                        if (product > N2V_MAXEXP) grad = (label - 1) * alpha;
                        else if (product < -N2V_MAXEXP) grad = label * alpha;
                        else {
                            double e = etab[(int)(product * N2V_EXP_PREC) + N2V_TABLE / 2];
                            grad = (label - 1 + 1 / (1 + e)) * alpha;
                        }
                        for (int i = 0; i < d; i++) {
                            neu1e[i] += grad * sn[i];
                            sn[i] += grad * sp[i];
                        }
                    }
                    double *sp = syn_pos + cw * d;
                    for (int i = 0; i < d; i++) sp[i] += neu1e[i];
                }
                word_cnt++;
            }
        }
    }
    if (syn_neg_out) memcpy(syn_neg_out, syn_neg, sizeof(double) * (size_t)V * d);
    *V_out = V;
    free(rn); free(vocab); free(syn_neg); free(KT); free(UT); free(prob); free(st); free(etab); free(neu1e);
    return 0;
}
