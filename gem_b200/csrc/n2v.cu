// gem_b200/csrc/n2v.cu -- node2vec on the GPU: alias tables, shuffled biased walks, SGNS.
//
// Replaces the prebuilt SNAP executable GEM shells out to (gem/embedding/node2vec.py:31-48;
// function addresses `bin@...` refer to gem/c_exe/node2vec, see SURVEY Appendix A):
//   PreprocessTransitionProbs/GetNodeAlias (bin@0x4127f0 / 0x4115f0) -> alias_build_kernel  (first order, thread per node)
//   PreprocessNode (bin@0x411f40)                                    -> alias2_build_kernel (p, q != 1, thread per edge)
//                                                                       both through one Vose routine, vose()
//   TVec::Shuffle (bin@0x40d1a0)                                     -> shuffle_rounds (host, LCG skip-ahead)
//   SimulateWalk / AliasDrawInt (bin@0x411a00 / 0x411360)            -> walk_kernel<SECOND> (thread per walk, both orders)
//   LearnVocab / InitUnigramTable (bin@0x40d560 / 0x40e520)          -> vocab_kernel + host Vose
//   InitPosEmb / TrainModel (bin@0x40e270 / 0x40d6a0)                -> init_pos_kernel, sgns_kernel (warp per walk)
//
// Bit-exactness contract (tests/test_gpu_n2v.py): alias tables (K int32, U fp64) and the walk matrix
// are identical to oracle/n2v_oracle.c (mode 1), which itself reproduces the reference binary.
// The RNG is SNAP's TRnd (Park-Miller, a = 16807, m = 2^31-1); because it is a multiplicative LCG,
// position t of the stream is seed * 16807^t mod m, so every walk can start at its own offset of the
// ONE stream the single-threaded binary consumes.
#include "common.cuh"
#include "nccl_api.h"
#include <math.h>
#include <string.h>
#include <algorithm>
#include <numeric>
#include <chrono>
#include <cub/cub.cuh>

namespace gemb {

#define RNG_M 2147483647u

__host__ __device__ __forceinline__ uint32_t lcg_next(uint32_t s) {
    // 16807 * s mod (2^31 - 1), s in [1, m-1]  (same values as Schrage's form, bin@0x41bb0c)
    uint64_t p = (uint64_t)s * 16807ull;
    uint32_t r = (uint32_t)(p & RNG_M) + (uint32_t)(p >> 31);
    return r >= RNG_M ? r - RNG_M : r;
}
__host__ __device__ __forceinline__ uint32_t mulmod31(uint32_t a, uint32_t b) {
    return (uint32_t)(((uint64_t)a * (uint64_t)b) % (uint64_t)RNG_M);
}
__host__ __device__ __forceinline__ uint32_t lcg_skip(uint32_t seed, uint64_t k) {
    uint32_t base = 16807u, acc = 1u;
    while (k) {
        if (k & 1) acc = mulmod31(acc, base);
        base = mulmod31(base, base);
        k >>= 1;
    }
    return mulmod31(acc, seed);
}
__device__ __forceinline__ double lcg_uni(uint32_t s) { return __ddiv_rn((double)s, 2147483647.0); }

// ------------------------------------------------------------------------------ alias tables
// Vose's alias method exactly as GetNodeAlias: the d unnormalised weights weight(i), whose sequential sum is psum,
// become the thresholds U and the aliases K of one table.  LIFO Under/Over stacks share the table's `st` segment,
// growing from both ends.  fp64 in the oracle's operation order, no FMA contraction.  weight(i) may read U[i] (the
// second-order tables keep their weights there): it is read before U[i] is written.
template <class Weight>
__device__ __forceinline__ void vose(int d, Weight weight, double psum, int32_t *K, double *U, int32_t *st) {
    int nu = 0, no = 0;
    for (int i = 0; i < d; i++) {
        const double u = __dmul_rn(__ddiv_rn(weight(i), psum), (double)d);
        K[i] = 0;
        U[i] = u;
        if (u < 1.0) st[nu++] = i; else st[d - 1 - (no++)] = i;
    }
    while (nu > 0 && no > 0) {
        const int small = st[--nu];
        const int large = st[d - 1 - (--no)];
        K[small] = large;
        const double ul = __dadd_rn(__dadd_rn(U[large], U[small]), -1.0);
        U[large] = ul;
        if (ul < 1.0) st[nu++] = large; else st[d - 1 - (no++)] = large;
    }
    while (nu > 0) U[st[--nu]] = 1.0;
    while (no > 0) U[st[d - 1 - (--no)]] = 1.0;
}

// first order: thread per node, the node's table at its CSR rows
__global__ void alias_build_kernel(int64_t n, const int32_t *__restrict__ indptr, const double *__restrict__ w,
                                   int32_t *__restrict__ K, double *__restrict__ U, int32_t *__restrict__ scratch) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    const int64_t s = indptr[v];
    const int d = indptr[v + 1] - indptr[v];
    if (d == 0) return;
    double psum = 0.0;
    const auto weight = [=](int j) { return w ? w[s + j] : 1.0; };
    for (int j = 0; j < d; j++) psum = __dadd_rn(psum, weight(j));
    vose(d, weight, psum, K + s, U + s, scratch + s);
}

// Second order (p, q != 1), PreprocessNode (bin@0x411f40): every directed edge (t -> v) owns an alias table over v's
// out-neighbours x with the unnormalised weights  w(v,x)/p if x == t;  w(v,x) if x is an out-neighbour of t;  w(v,x)/q
// otherwise  -- the sum over edges of outdeg(v) entries the reference keeps in a hash map per node.  Here: one flat
// array, the table of CSR edge e at off2[e], built by one thread per edge, adjacency membership by binary search in t's
// sorted neighbour list.
__global__ void edge_degree_kernel(int64_t nnz, const int32_t *__restrict__ indptr, const int32_t *__restrict__ idx,
                                   long long *__restrict__ deg_out) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
        const int v = idx[e];
        deg_out[e] = (long long)(indptr[v + 1] - indptr[v]);
    }
}

__device__ __forceinline__ bool has_edge_sorted(const int32_t *__restrict__ idx, int lo, int hi, int x) {
    const int end = hi;
    while (lo < hi) { const int m = (lo + hi) >> 1; if (idx[m] < x) lo = m + 1; else hi = m; }
    return lo < end && idx[lo] == x;
}

__global__ void alias2_build_kernel(int64_t n, int64_t nnz, const int32_t *__restrict__ indptr, const int32_t *__restrict__ idx,
                                    const double *__restrict__ w, const long long *__restrict__ off2, double p, double q,
                                    int32_t *__restrict__ K2, double *__restrict__ U2, int32_t *__restrict__ scratch) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    // source node t of CSR position e: last row with indptr[row] <= e
    int64_t lo = 0, hi = n;
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if ((int64_t)indptr[m + 1] <= e) lo = m + 1; else hi = m; }
    const int t = (int)lo;
    const int v = idx[e];
    const int s = indptr[v], d = indptr[v + 1] - s;
    if (d == 0) return;
    const int ts = indptr[t], te = indptr[t + 1];
    const long long o = off2[e];
    double *U = U2 + o;
    double psum = 0.0;
    for (int j = 0; j < d; j++) {
        const int x = idx[s + j];
        const double wj = w ? w[s + j] : 1.0;
        double val;
        if (x == t) val = __ddiv_rn(wj, p);
        else if (has_edge_sorted(idx, ts, te, x)) val = wj;
        else val = __ddiv_rn(wj, q);
        U[j] = val;
        psum = __dadd_rn(psum, val);
    }
    vose(d, [=](int j) { return U[j]; }, psum, K2 + o, U, scratch + o);
}

// ------------------------------------------------------------------------------ walks
// Thread per walk w = i*N + j (round i, shuffled position j).  Stream offset (oracle mode 1):
//   (i+1)*(N-1) + w*(2*walk_len-3).
// Every step after the first draws from the table of the current node (first order: at indptr[cur]) or, SECOND, from
// the table of the CSR edge e just walked (off2[e], bin@0x411d73).
template <bool SECOND>
__global__ void walk_kernel(const int32_t *__restrict__ indptr, const int32_t *__restrict__ idx,
                            const int32_t *__restrict__ K, const double *__restrict__ U,
                            const long long *__restrict__ off2, const int32_t *__restrict__ order, int64_t N,
                            int walk_len, uint32_t seed, int64_t w_begin, int64_t w_end, int32_t *__restrict__ out) {
    const int64_t w = w_begin + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= w_end) return;
    int32_t *row = out + (w - w_begin) * walk_len;
    const int64_t i = w / N;
    const uint64_t per_walk = walk_len >= 2 ? (uint64_t)(2 * walk_len - 3) : 0;
    uint32_t st = lcg_skip(seed, (uint64_t)(i + 1) * (uint64_t)(N - 1) + (uint64_t)w * per_walk);
    int cur = order[w];
    int len = 0;
    row[len++] = cur;
    if (walk_len > 1) {
        int s = indptr[cur], d = indptr[cur + 1] - s;
        if (d > 0) {
            st = lcg_next(st);
            int64_t e = s + (int)(st % (uint32_t)d);         // step 1: uniform, ignores weights (bin@0x411b31)
            cur = idx[e];
            row[len++] = cur;
            while (len < walk_len) {
                s = indptr[cur];
                d = indptr[cur + 1] - s;
                if (d == 0) break;
                const long long o = SECOND ? off2[e] : s;
                st = lcg_next(st);
                const int x = (int)(int64_t)__dmul_rn(lcg_uni(st), (double)d);
                st = lcg_next(st);
                const double y = lcg_uni(st);
                const int nx = y < U[o + x] ? x : K[o + x];
                e = s + nx;
                cur = idx[e];
                row[len++] = cur;
            }
        }
    }
    for (; len < walk_len; len++) row[len] = 0;   // WalksVV is zero-initialised (SURVEY F10)
}

// ------------------------------------------------------------------------------ vocabulary
// first flat position and occurrence count of every node id in the (global) walk matrix
__global__ void vocab_kernel(const int32_t *__restrict__ walks, int64_t count, int64_t flat_offset,
                             unsigned long long *__restrict__ first_pos, unsigned long long *__restrict__ cnt) {
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < count;
         t += (int64_t)gridDim.x * blockDim.x) {
        const int id = walks[t];
        const unsigned long long pos = (unsigned long long)(t + flat_offset);
        if (pos < first_pos[id]) atomicMin(first_pos + id, pos);
        atomicAdd(cnt + id, 1ull);
    }
}

// SynPos[token i][j] = (GetUniDev() - 0.5) / d  with draws i*d + j + 1 of TRnd(seed)  (InitPosEmb)
__global__ void init_pos_kernel(int64_t V, int d, uint32_t seed, const int32_t *__restrict__ tok2node,
                                float *__restrict__ syn_pos) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    uint32_t st = lcg_skip(seed, (uint64_t)i * (uint64_t)d);
    float *row = syn_pos + (int64_t)tok2node[i] * d;
    for (int j = 0; j < d; j++) {
        st = lcg_next(st);
        row[j] = (float)__ddiv_rn(__dadd_rn(lcg_uni(st), -0.5), (double)d);
    }
}

// ------------------------------------------------------------------------------ SGNS
struct SgnsParams {
    const int32_t *walks;     // local walks, node ids
    int64_t n_walks_local;    // walks in this launch
    int64_t walk_offset;      // global index of local walk 0
    int64_t n_walks_total;    // all walks of an epoch (all ranks)
    int walk_len, d, win, iters, epoch;
    float *syn_pos, *syn_neg; // rows by node id
    const int32_t *KT;        // V  (token space): first-level lookup of RndUnigramInt
    const uint4 *ent;         // V: {thr, node(X), node(KT[X]), 0}: Y < UT[X]  <=>  draw < thr   (exact, see host)
    int64_t V;
    uint32_t seed;            // training TRnd seed
    int sequential;
    uint32_t *seq_state;      // sequential mode: carried RNG state across epochs/launches (device)
    unsigned long long *pair_counter;
};

#define SG_NEG 5
#define SG_MAXEXP 6.0f

template <int NV, bool VEC>
struct RowIO {
    // NV values per lane.  VEC: value v <-> dim (v/4)*128 + lane*4 + (v%4)  (float4 per lane);
    // scalar: value v <-> dim v*32 + lane.
    __device__ static __forceinline__ void load(const float *row, int d, int lane, float (&r)[NV]) {
        if (VEC) {
#pragma unroll
            for (int q = 0; q < NV / 4; q++) {
                const float4 t = __ldcg((const float4 *)(row + q * 128 + lane * 4));
                r[4 * q] = t.x; r[4 * q + 1] = t.y; r[4 * q + 2] = t.z; r[4 * q + 3] = t.w;
            }
        } else {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                const int dim = v * 32 + lane;
                r[v] = dim < d ? __ldcg(row + dim) : 0.f;
            }
        }
    }
    __device__ static __forceinline__ void store(float *row, int d, int lane, const float (&r)[NV]) {
        if (VEC) {
#pragma unroll
            for (int q = 0; q < NV / 4; q++)
                __stcg((float4 *)(row + q * 128 + lane * 4), make_float4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]));
        } else {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                const int dim = v * 32 + lane;
                if (dim < d) __stcg(row + dim, r[v]);
            }
        }
    }
};

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

// gradient * alpha, TrainModel bin@0x40dce8-0x40dd46: table lookup sigmoid quantised to 1e-4
__device__ __forceinline__ float sg_grad(float f, int label, float alpha) {
    if (f > SG_MAXEXP) return (float)(label - 1) * alpha;
    if (f < -SG_MAXEXP) return (float)label * alpha;
    const float fq = truncf(f * 10000.f) * 1e-4f;
    const float e = __expf(fq);
    return ((float)(label - 1) + __fdividef(1.f, 1.f + e)) * alpha;
}

__device__ __forceinline__ uint32_t mulmod_fold(uint32_t a, uint32_t b) {
    const uint64_t p = (uint64_t)a * (uint64_t)b;            // < 2^62
    uint64_t r = (p & RNG_M) + (p >> 31);                    // < 2^32
    r = (r & RNG_M) + (r >> 31);
    return (uint32_t)(r >= RNG_M ? r - RNG_M : r);
}

// one sample of a pair against the context row sp: g = gradient of <sp, r> for the sample's label; neu += g r, r += g sp.
// The positive sample (label 1) comes first and starts neu with an assignment: fmaf(g, r, 0) would turn a -0 into +0.
template <int NV, bool POSITIVE>
__device__ __forceinline__ void sgns_sample(const float (&sp)[NV], float (&r)[NV], float (&neu)[NV], float alpha) {
    float f = 0.f;
#pragma unroll
    for (int v = 0; v < NV; v++) f = fmaf(sp[v], r[v], f);
    f = warp_sum(f);
    const float g = sg_grad(f, POSITIVE ? 1 : 0, alpha);
#pragma unroll
    for (int v = 0; v < NV; v++) { neu[v] = POSITIVE ? g * r[v] : fmaf(g, r[v], neu[v]); r[v] = fmaf(g, sp[v], r[v]); }
}

// one (centre = word, context = ctx) pair: 1 positive + 5 negatives.  The 5 negative rows are loaded together, or,
// `seqpath`, one after the other through memory (needed when a negative row repeats inside the group).
template <int NV, bool VEC>
__device__ __forceinline__ void sgns_pair(const SgnsParams &P, int lane, int d, int ctx, const int (&tgt)[SG_NEG],
                                          bool seqpath, float alpha, float (&snw)[NV]) {
    float sp[NV], neu[NV];
    float *sp_row = P.syn_pos + (int64_t)ctx * d;
    RowIO<NV, VEC>::load(sp_row, d, lane, sp);
    if (!seqpath) {
        float sn[SG_NEG][NV];
#pragma unroll
        for (int j = 0; j < SG_NEG; j++)
            if (tgt[j] >= 0) RowIO<NV, VEC>::load(P.syn_neg + (int64_t)tgt[j] * d, d, lane, sn[j]);
        sgns_sample<NV, true>(sp, snw, neu, alpha);
#pragma unroll
        for (int j = 0; j < SG_NEG; j++) {
            if (tgt[j] < 0) continue;
            sgns_sample<NV, false>(sp, sn[j], neu, alpha);
            RowIO<NV, VEC>::store(P.syn_neg + (int64_t)tgt[j] * d, d, lane, sn[j]);
        }
    } else {
        sgns_sample<NV, true>(sp, snw, neu, alpha);
        for (int j = 0; j < SG_NEG; j++) {
            if (tgt[j] < 0) continue;
            float sn[NV];
            float *row = P.syn_neg + (int64_t)tgt[j] * d;
            RowIO<NV, VEC>::load(row, d, lane, sn);
            sgns_sample<NV, false>(sp, sn, neu, alpha);
            RowIO<NV, VEC>::store(row, d, lane, sn);
        }
    }
#pragma unroll
    for (int v = 0; v < NV; v++) sp[v] += neu[v];
    RowIO<NV, VEC>::store(sp_row, d, lane, sp);
}

// P is read in place from the parameter bank (__grid_constant__): a by-value copy of its fields into registers up front
// costs the d = 128 instantiation 8 registers.
template <int NV, bool VEC>
__global__ void __launch_bounds__(128)
sgns_kernel(const __grid_constant__ SgnsParams P) {
    extern __shared__ int32_t s_walks[];  // warps_per_block x walk_len
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int warps_per_block = blockDim.x >> 5;
    const int64_t warp_global = (int64_t)blockIdx.x * warps_per_block + wib;
    const int64_t total_warps = (int64_t)gridDim.x * warps_per_block;
    int32_t *wk = s_walks + wib * P.walk_len;
    const int d = P.d, L = P.walk_len, win = P.win;
    const int64_t all_words = P.n_walks_total * (int64_t)L;
    const double denom = (double)((int64_t)P.iters * all_words + 1);
    // upper bound of draws per walk in parallel mode: per word 1 + (2*win) * SG_NEG * 2
    const uint64_t stride = (uint64_t)L * (uint64_t)(1 + 2 * win * SG_NEG * 2);
    const uint32_t Vu = (uint32_t)P.V;
    // lane j < 5 draws negative j: its two TRnd values are draws 2j+1 and 2j+2 after the current state
    const uint32_t a_first = lane == 0 ? 16807u : lane == 1 ? lcg_skip(1u, 3) : lane == 2 ? lcg_skip(1u, 5)
                             : lane == 3 ? lcg_skip(1u, 7) : lcg_skip(1u, 9);
    const uint32_t a_ten = lcg_skip(1u, 10);
    uint32_t st = 0;
    if (P.sequential) st = *P.seq_state;
    unsigned long long pairs = 0;

    for (int64_t wl = warp_global; wl < P.n_walks_local; wl += total_warps) {
        const int64_t wg = P.walk_offset + wl;  // global walk index within the epoch
        for (int t = lane; t < L; t += 32) wk[t] = P.walks[wl * L + t];
        __syncwarp();
        if (!P.sequential)
            st = lcg_skip(P.seed, 0x40000000ull + ((uint64_t)P.epoch * (uint64_t)P.n_walks_total + (uint64_t)wg) * stride);
        for (int pos = 0; pos < L; pos++) {
            const int64_t wc = ((int64_t)P.epoch * P.n_walks_total + wg) * L + pos;  // WordCntAll
            const int64_t wc0 = wc - wc % 10000;
            double al = 0.025 * (1.0 - (double)wc0 / denom);
            if (al < 0.025 * 0.0001) al = 0.025 * 0.0001;
            const float alpha = (float)al;
            const int word = wk[pos];
            st = lcg_next(st);
            const int offset = (int)(st % (uint32_t)win);
            float snw[NV];
            float *snw_row = P.syn_neg + (int64_t)word * d;
            RowIO<NV, VEC>::load(snw_row, d, lane, snw);
            for (int a = offset; a < 2 * win + 1 - offset; a++) {
                if (a == win) continue;
                const int c = pos - win + a;
                if (c < 0 || c >= L) continue;
                const int ctx = wk[c];
                // ---- 5 negatives drawn by lanes 0..4 in parallel (RndUnigramInt: first lookup through KTable)
                int mine = -2 - lane;                                   // unique dummy: never matches
                if (lane < SG_NEG) {
                    const uint32_t s1 = mulmod_fold(st, a_first);
                    const uint32_t s2 = mulmod_fold(s1, 16807u);
                    const uint32_t i0 = (uint32_t)(((uint64_t)s1 * (uint64_t)Vu) / (uint64_t)RNG_M);
                    const int X = P.KT[i0];
                    const uint4 e = P.ent[X];
                    const int node = s2 < e.x ? (int)e.y : (int)e.z;
                    if (node != word) mine = node;                      // `if (Target == Word) continue;`
                }
                st = mulmod_fold(st, a_ten);
                int tgt[SG_NEG];
#pragma unroll
                for (int j = 0; j < SG_NEG; j++) tgt[j] = __shfl_sync(0xffffffffu, mine, j);
                const unsigned same = __match_any_sync(0xffffffffu, mine);
                const bool dup = __any_sync(0xffffffffu, lane < SG_NEG && mine >= 0 && __popc(same) > 1);
                sgns_pair<NV, VEC>(P, lane, d, ctx, tgt, dup, alpha, snw);
                pairs++;
            }
            RowIO<NV, VEC>::store(snw_row, d, lane, snw);
        }
        __syncwarp();
    }
    if (P.sequential && lane == 0 && warp_global == 0) *P.seq_state = st;
    if (lane == 0 && pairs) atomicAdd(P.pair_counter, pairs);
}

// ------------------------------------------------------------------------------ host pieces
// TVec::Shuffle per round (bin@0x40d220 branch: one GetUniDevInt per swap), cumulative across rounds;
// round i starts at stream offset i*(N-1) + i*N*(2*walk_len-3)  (oracle mode 1).
static void shuffle_rounds(const int32_t *nids, int64_t N, int num_walks, int walk_len, uint32_t seed,
                           int32_t *order_out) {
    std::vector<int32_t> order(nids, nids + N);
    const uint64_t per_walk = walk_len >= 2 ? (uint64_t)(2 * walk_len - 3) : 0;
    for (int64_t i = 0; i < num_walks; i++) {
        uint32_t st = lcg_skip(seed, (uint64_t)i * (uint64_t)(N - 1) + (uint64_t)i * (uint64_t)N * per_walk);
        for (int64_t j = 0; j < N - 1; j++) {
            st = lcg_next(st);
            const int64_t k = j + (int64_t)(st % (uint32_t)(N - j));
            std::swap(order[j], order[k]);
        }
        memcpy(order_out + i * N, order.data(), sizeof(int32_t) * N);
    }
}

// InitUnigramTable (bin@0x40e520): prob = count^0.75 via exp(log(c)*0.75), Vose over TOKEN order
static void unigram_alias(const std::vector<int64_t> &vocab, std::vector<int32_t> &KT, std::vector<double> &UT) {
    const int64_t V = (int64_t)vocab.size();
    std::vector<double> prob(V);
    double tw = 0;
    for (int64_t i = 0; i < V; i++) { prob[i] = exp(log((double)vocab[i]) * 0.75); tw += prob[i]; }
    for (int64_t i = 0; i < V; i++) prob[i] /= tw;
    KT.assign(V, 0);
    UT.assign(V, 0.0);
    std::vector<int32_t> under, over;
    under.reserve(V); over.reserve(V);
    for (int64_t i = 0; i < V; i++) {
        UT[i] = prob[i] * (double)V;
        if (UT[i] < 1) under.push_back((int32_t)i); else over.push_back((int32_t)i);
    }
    while (!under.empty() && !over.empty()) {
        const int32_t small = under.back(); under.pop_back();
        const int32_t large = over.back(); over.pop_back();
        KT[small] = large;
        UT[large] = UT[large] + UT[small] - 1;
        if (UT[large] < 1) under.push_back(large); else over.push_back(large);
    }
    for (int32_t i : under) UT[i] = 1;
    for (int32_t i : over) UT[i] = 1;
}

struct N2VDev {
    // walks only: fp64 weights; alias tables K/U (first order: a node's table at its CSR rows; second order: the table of
    // CSR edge e at off2[e]) and their Vose scratch; the start node of every walk
    DeviceBuffer<double> w, U;
    DeviceBuffer<int32_t> K, scratch, order;
    DeviceBuffer<long long> off2;    // second order only: nnz + 1 table offsets
    DeviceBuffer<int32_t> walks;
    DeviceBuffer<unsigned long long> first_pos, cnt, pairs;
    DeviceBuffer<int32_t> KT, tok2node;
    DeviceBuffer<uint4> ent;
    DeviceBuffer<float> syn_pos, syn_neg, pos0, delta;
    DeviceBuffer<uint32_t> seq_state;
};

static int check_graph_for_n2v(gemb_graph *g) {
    GEMB_ARG(g != nullptr, "graph");
    GEMB_ARG(g->row0 == 0 && g->n_local == g->n, "node2vec needs the whole graph on every rank (row0=0, n_local=n)");
    return GEMB_OK;
}

// first-order tables for p = q = 1, second-order tables (with D.off2) otherwise
static int build_alias(gemb_graph *g, const double *weights64, double p, double q, N2VDev &D) {
    gemb_ctx *c = g->ctx;
    const int64_t nnz = g->A.nnz, n = g->n;
    if (weights64 && nnz) GEMB_CUDA(D.w.upload(weights64, nnz, c->stream));
    if (p == 1.0 && q == 1.0) {
        GEMB_CUDA(D.K.alloc(std::max<int64_t>(nnz, 1)));
        GEMB_CUDA(D.U.alloc(std::max<int64_t>(nnz, 1)));
        GEMB_CUDA(D.scratch.alloc(std::max<int64_t>(nnz, 1)));
        return launch(c, alias_build_kernel, (unsigned)((n + 127) / 128), 128, 0, n, g->A.indptr, D.w.get(), D.K.get(), D.U.get(),
                      D.scratch.get());
    }
    GEMB_CUDA(D.off2.alloc(nnz + 1));
    long long T = 0;
    {
        DeviceBuffer<long long> deg;
        GEMB_CUDA(deg.alloc(nnz + 1));
        GEMB_CUDA(cudaMemsetAsync(deg.get(), 0, sizeof(long long) * (nnz + 1), c->stream));
        if (nnz) GEMB_TRY(launch(c, edge_degree_kernel, c->sm_count * 8, 256, 0, nnz, g->A.indptr, g->A.indices, deg.get()));
        size_t tb = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tb, deg.get(), D.off2.get(), nnz + 1, c->stream);
        DeviceBuffer<char> tmp;
        GEMB_CUDA(tmp.alloc(tb));
        GEMB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.get(), tb, deg.get(), D.off2.get(), nnz + 1, c->stream));
        count_launch();
        GEMB_TRY(copy_sync(c, &T, D.off2.get() + nnz, sizeof T, cudaMemcpyDeviceToHost));
    }
    // the reference needs the same sum_(t->v) outdeg(v) entries in host hash maps; here they must fit in HBM
    size_t free_b = 0, total_b = 0;
    GEMB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const double need = 16.0 * (double)T;
    if (need > 0.9 * ((double)free_b + (double)gemb_mem_cached_bytes())) {
        set_error("node2vec with p=%g q=%g: the second-order alias tables have %lld entries (%.1f GB, sum over edges (t->v) of "
                  "outdeg(v)) and do not fit in the %.1f GB of free device memory", p, q, T, need / 1e9, (double)free_b / 1e9);
        return GEMB_ERR_NOMEM;
    }
    GEMB_CUDA(D.K.alloc(std::max<long long>(T, 1)));
    GEMB_CUDA(D.U.alloc(std::max<long long>(T, 1)));
    GEMB_CUDA(D.scratch.alloc(std::max<long long>(T, 1)));
    if (nnz)
        GEMB_TRY(launch(c, alias2_build_kernel, (unsigned)((nnz + 127) / 128), 128, 0, n, nnz, g->A.indptr, g->A.indices, D.w.get(),
                        D.off2.get(), p, q, D.K.get(), D.U.get(), D.scratch.get()));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    D.scratch.reset();   // 4 of the 16 bytes per entry: freed before the walks allocate theirs
    return GEMB_OK;
}

static double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

// Alias tables (between events 0 and 1 of `ev`), then the walks [w_begin, w_end) into D.walks (device; event 2), then
// everything only the walks needed is released.  stats (optional): zeroed, with the alias and walk fields filled in.
template <int NEV>
static int alias_and_walks(gemb_graph *g, const double *weights64, double p, double q, const int32_t *nids, int64_t N,
                           int walk_len, int num_walks, uint32_t seed, int64_t w_begin, int64_t w_end, N2VDev &D,
                           const CallEvents<NEV> &ev, gemb_n2v_stats *stats) {
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaEventRecord(ev[0], c->stream));
    GEMB_TRY(build_alias(g, weights64, p, q, D));
    GEMB_CUDA(cudaEventRecord(ev[1], c->stream));
    auto t0 = std::chrono::steady_clock::now();
    std::vector<int32_t> order((size_t)num_walks * N);
    shuffle_rounds(nids, N, num_walks, walk_len, seed, order.data());
    const double sh_ms = ms_since(t0);
    GEMB_CUDA(D.order.upload(order.data(), order.size(), c->stream));
    const int64_t cnt = w_end - w_begin;
    GEMB_CUDA(D.walks.alloc(std::max<int64_t>(cnt * walk_len, 1)));
    if (cnt > 0) {
        const long long *off2 = D.off2.get();
        auto walk = off2 ? walk_kernel<true> : walk_kernel<false>;
        GEMB_TRY(launch(c, walk, (unsigned)((cnt + 127) / 128), 128, 0, g->A.indptr, g->A.indices, D.K.get(), D.U.get(), off2,
                        D.order.get(), N, walk_len, seed, w_begin, w_end, D.walks.get()));
    }
    GEMB_CUDA(cudaEventRecord(ev[2], c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));  // `order` (host) must outlive the async copy
    D.w.reset(); D.K.reset(); D.U.reset(); D.scratch.reset(); D.off2.reset(); D.order.reset();
    if (stats) {
        memset((char *)stats + sizeof(uint32_t), 0, sizeof(*stats) - sizeof(uint32_t));
        stats->alias_ms = ev.ms(0, 1);
        stats->shuffle_ms = sh_ms;
        stats->walk_ms = std::max(0.0, (double)ev.ms(1, 2) - sh_ms);   // the host shuffle runs while the stream works
        stats->n_walks = cnt;
        stats->walk_bytes = 24.0 * (double)cnt * (double)std::max(walk_len - 1, 0);
    }
    return GEMB_OK;
}

// Every warp stages its walk in shared memory: warps x walk_len int32.
static size_t sgns_smem_bytes(int threads, int walk_len) { return sizeof(int32_t) * (threads / 32) * (size_t)walk_len; }

static int launch_sgns(gemb_ctx *c, const SgnsParams &P, int blocks, int threads) {
    const int d = P.d, nv = (d + 31) / 32;
    auto kernel = sgns_kernel<16, false>;
    if (d % 128 == 0 && d <= 512)
        kernel = d == 128 ? sgns_kernel<4, true> : d == 256 ? sgns_kernel<8, true> : d == 384 ? sgns_kernel<12, true> : sgns_kernel<16, true>;
    else if (nv <= 8)
        kernel = nv <= 1 ? sgns_kernel<1, false> : nv <= 2 ? sgns_kernel<2, false> : nv <= 4 ? sgns_kernel<4, false> : sgns_kernel<8, false>;
    else if (nv > 16) {
        set_error("node2vec: d = %d is not supported (d <= 512)", d);
        return GEMB_ERR_UNSUPPORTED;
    }
    const size_t sh = sgns_smem_bytes(threads, P.walk_len);
    // beyond the default 48 KB the kernel has to opt in (gemb_node2vec checked sh against the device's opt-in limit)
    if (sh > 48 * 1024) GEMB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sh));
    return launch(c, kernel, blocks, threads, sh, P);
}

}  // namespace gemb

using namespace gemb;

extern "C" {

int gemb_n2v_alias(gemb_graph *g, const double *weights64, int32_t *K_out, double *U_out) {
    GEMB_TRY(check_graph_for_n2v(g));
    GEMB_ARG(K_out && U_out, "outputs");
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    N2VDev D;
    GEMB_TRY(build_alias(g, weights64, 1.0, 1.0, D));
    const int64_t nnz = g->A.nnz;
    GEMB_CUDA(cudaMemcpyAsync(K_out, D.K.get(), sizeof(int32_t) * nnz, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(U_out, D.U.get(), sizeof(double) * nnz, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

static int n2v_check_common(int64_t N, int walk_len, int num_walks, double p, double q, int32_t seed) {
    GEMB_ARG(N >= 1, "N");
    GEMB_ARG(walk_len >= 1 && num_walks >= 1, "walk_len / num_walks");
    GEMB_ARG(seed >= 1 && seed < 2147483647, "seed must be in [1, 2^31-2] (TRnd)");
    GEMB_ARG(p > 0.0 && q > 0.0, "p and q must be positive");
    return GEMB_OK;
}

int gemb_n2v_walks(gemb_graph *g, const double *weights64, const int32_t *nids, int64_t N, int walk_len,
                   int num_walks, double p, double q, int32_t seed, int64_t w_begin, int64_t w_end,
                   int32_t *walks_out, gemb_n2v_stats *stats) {
    GEMB_TRY(check_graph_for_n2v(g));
    GEMB_ARG(nids != nullptr, "nids");
    GEMB_TRY(n2v_check_common(N, walk_len, num_walks, p, q, seed));
    GEMB_ARG(0 <= w_begin && w_begin <= w_end && w_end <= N * (int64_t)num_walks, "walk range");
    GEMB_ARG(!stats || stats->struct_size == sizeof(gemb_n2v_stats), "stats.struct_size");
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    N2VDev D;
    CallEvents<3> ev;
    GEMB_CUDA(ev.create());
    GEMB_TRY(alias_and_walks(g, weights64, p, q, nids, N, walk_len, num_walks, (uint32_t)seed, w_begin, w_end, D, ev, stats));
    if (walks_out && w_end > w_begin)
        GEMB_CUDA(cudaMemcpyAsync(walks_out, D.walks.get(), sizeof(int32_t) * (size_t)(w_end - w_begin) * walk_len,
                                  cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    return GEMB_OK;
}

int gemb_node2vec(gemb_graph *g, const double *weights64, const int32_t *nids, int64_t N, int d, int walk_len,
                  int num_walks, int con_size, int max_iter, double p, double q, int32_t seed, int sequential,
                  int64_t n_rows, float *X_out, gemb_n2v_stats *stats) {
    GEMB_TRY(check_graph_for_n2v(g));
    GEMB_ARG(nids != nullptr, "nids");
    GEMB_TRY(n2v_check_common(N, walk_len, num_walks, p, q, seed));
    GEMB_ARG(d >= 1 && con_size >= 1 && max_iter >= 1, "d / con_size / max_iter");
    GEMB_ARG(n_rows >= g->n, "n_rows must cover every node id");
    GEMB_ARG(!stats || stats->struct_size == sizeof(gemb_n2v_stats), "stats.struct_size");
    gemb_ctx *c = g->ctx;
    GEMB_CUDA(cudaSetDevice(c->device));
    GEMB_ARG(!(sequential && c->nranks > 1), "sequential parity mode is single-GPU");
    // the SGNS kernel's limits, checked before any work: at most 16 values per lane, and the walks of a block in shared memory
    if (d > 512) {
        set_error("node2vec: d = %d is not supported (d <= 512)", d);
        return GEMB_ERR_UNSUPPORTED;
    }
    const int threads = sequential ? 32 : 128;
    int smem_optin = 0;
    GEMB_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    if (sgns_smem_bytes(threads, walk_len) > (size_t)smem_optin) {
        set_error("node2vec: walk_len = %d is not supported in %s mode (walk_len <= %d: the %d walk(s) trained by a block "
                  "are kept in its shared memory, at most %d bytes on this device)", walk_len,
                  sequential ? "sequential" : "Hogwild", smem_optin / (int)sgns_smem_bytes(threads, 1), threads / 32, smem_optin);
        return GEMB_ERR_UNSUPPORTED;
    }
    N2VDev D;
    CallEvents<6> ev;
    GEMB_CUDA(ev.create());

    // ---- walks: this rank's contiguous share of the num_walks*N walks of an epoch
    const int64_t total_walks = N * (int64_t)num_walks;
    const int64_t per = (total_walks + c->nranks - 1) / c->nranks;
    const int64_t w_begin = std::min<int64_t>(total_walks, per * c->rank);
    const int64_t w_end = std::min<int64_t>(total_walks, w_begin + per);
    const int64_t n_local = w_end - w_begin;
    GEMB_TRY(alias_and_walks(g, weights64, p, q, nids, N, walk_len, num_walks, (uint32_t)seed, w_begin, w_end, D, ev, stats));

    // ---- vocabulary: first appearance + counts (all ranks combined), host renumbering + Vose
    auto tv0 = std::chrono::steady_clock::now();
    const int64_t n_ids = g->n;
    GEMB_CUDA(D.first_pos.alloc(n_ids));
    GEMB_CUDA(D.cnt.alloc(n_ids));
    GEMB_CUDA(cudaMemsetAsync(D.first_pos.get(), 0xff, sizeof(unsigned long long) * n_ids, c->stream));
    GEMB_CUDA(cudaMemsetAsync(D.cnt.get(), 0, sizeof(unsigned long long) * n_ids, c->stream));
    if (n_local > 0)
        GEMB_TRY(launch(c, vocab_kernel, c->sm_count * 8, 256, 0, D.walks.get(), n_local * walk_len, w_begin * walk_len,
                        D.first_pos.get(), D.cnt.get()));
    if (c->nranks > 1) {
        NcclApi *api = nccl_api();
        if (!api) return GEMB_ERR_NCCL;
        ncclResult_t r = api->AllReduce(D.first_pos.get(), D.first_pos.get(), n_ids, ncclUint64, ncclMin, (ncclComm_t)c->comm, c->stream);
        if (r == ncclSuccess) r = api->AllReduce(D.cnt.get(), D.cnt.get(), n_ids, ncclUint64, ncclSum, (ncclComm_t)c->comm, c->stream);
        if (r != ncclSuccess) { set_error("nccl vocab allreduce: %s", api->GetErrorString(r)); return GEMB_ERR_NCCL; }
    }
    std::vector<unsigned long long> h_first(n_ids), h_cnt(n_ids);
    GEMB_CUDA(cudaMemcpyAsync(h_first.data(), D.first_pos.get(), sizeof(unsigned long long) * n_ids, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaMemcpyAsync(h_cnt.data(), D.cnt.get(), sizeof(unsigned long long) * n_ids, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    std::vector<int32_t> tok2node;
    tok2node.reserve(n_ids);
    for (int64_t i = 0; i < n_ids; i++) if (h_cnt[i] > 0) tok2node.push_back((int32_t)i);
    std::sort(tok2node.begin(), tok2node.end(), [&](int32_t a, int32_t b) { return h_first[a] < h_first[b]; });
    const int64_t V = (int64_t)tok2node.size();
    GEMB_ARG(V >= 1, "empty vocabulary");
    std::vector<int64_t> vocab(V);
    for (int64_t i = 0; i < V; i++) vocab[i] = (int64_t)h_cnt[tok2node[i]];
    std::vector<int32_t> KT;
    std::vector<double> UT;
    unigram_alias(vocab, KT, UT);
    // ent[X] = {thr, node(X), node(KT[X])} with thr the smallest draw s for which (double)s / m >= UT[X]:
    // `Y < UT[X]` of RndUnigramInt (Y = s / m in fp64) is then exactly `s < thr` in integers.
    std::vector<uint4> ent(V);
    for (int64_t i = 0; i < V; i++) {
        const double u = UT[i];
        int64_t t = (int64_t)ceil(u * 2147483647.0);
        if (t < 0) t = 0;
        if (t > 2147483647LL) t = 2147483647LL;
        while (t > 0 && (double)(t - 1) / 2147483647.0 >= u) t--;
        while (t < 2147483647LL && (double)t / 2147483647.0 < u) t++;
        ent[i] = make_uint4((uint32_t)t, (uint32_t)tok2node[i], (uint32_t)tok2node[KT[i]], 0u);
    }
    GEMB_CUDA(D.ent.upload(ent.data(), V, c->stream));
    GEMB_CUDA(D.KT.upload(KT.data(), V, c->stream));
    GEMB_CUDA(D.tok2node.upload(tok2node.data(), V, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    const double vocab_ms = ms_since(tv0);
    GEMB_CUDA(cudaEventRecord(ev[3], c->stream));

    // ---- embeddings
    const size_t tab = (size_t)n_rows * d;
    GEMB_CUDA(D.syn_pos.alloc(tab));
    GEMB_CUDA(D.syn_neg.alloc(tab));
    GEMB_CUDA(cudaMemsetAsync(D.syn_pos.get(), 0, sizeof(float) * tab, c->stream));
    GEMB_CUDA(cudaMemsetAsync(D.syn_neg.get(), 0, sizeof(float) * tab, c->stream));
    GEMB_TRY(launch(c, init_pos_kernel, (unsigned)((V + 127) / 128), 128, 0, V, d, (uint32_t)seed, D.tok2node.get(), D.syn_pos.get()));
    GEMB_CUDA(D.pairs.alloc(1));
    GEMB_CUDA(cudaMemsetAsync(D.pairs.get(), 0, sizeof(unsigned long long), c->stream));
    GEMB_CUDA(D.seq_state.alloc(1));
    {
        const uint32_t st0 = lcg_skip((uint32_t)seed, (uint64_t)V * (uint64_t)d);  // after InitPosEmb's V*d draws
        GEMB_TRY(copy_sync(c, D.seq_state.get(), &st0, sizeof st0, cudaMemcpyHostToDevice));
    }
    if (c->nranks > 1) {
        GEMB_CUDA(D.pos0.alloc(tab));
        GEMB_CUDA(D.delta.alloc(tab));
    }

    SgnsParams P;
    P.walks = D.walks.get(); P.n_walks_local = n_local; P.walk_offset = w_begin; P.n_walks_total = total_walks;
    P.walk_len = walk_len; P.d = d; P.win = con_size; P.iters = max_iter; P.epoch = 0;
    P.syn_pos = D.syn_pos.get(); P.syn_neg = D.syn_neg.get(); P.KT = D.KT.get(); P.ent = D.ent.get(); P.V = V;
    P.seed = (uint32_t)seed; P.sequential = sequential ? 1 : 0;
    P.seq_state = D.seq_state.get(); P.pair_counter = D.pairs.get();
    // Hogwild: concurrent walks race on embedding rows exactly as SNAP's OpenMP threads do.  Keep the
    // number of in-flight walks far below the vocabulary size so that lost updates stay as rare as in
    // the reference (<= 1 walk in flight per 32 tokens), up to 24 warps per SM.
    int blocks = sequential ? 1 : c->sm_count * 6;
    if (!sequential) {
        const int64_t max_warps = std::max<int64_t>(1, V / 32);
        blocks = (int)std::max<int64_t>(1, std::min<int64_t>(blocks, (max_warps + 3) / 4));
    }
    double comm_ms = 0;
    float *syn_pos = D.syn_pos.get(), *syn_neg = D.syn_neg.get(), *pos0 = D.pos0.get(), *delta = D.delta.get();
    for (int it = 0; it < max_iter; it++) {
        P.epoch = it;
        const int64_t tabn = (int64_t)tab;
        if (c->nranks > 1) {
            GEMB_CUDA(cudaMemcpyAsync(pos0, syn_pos, sizeof(float) * tab, cudaMemcpyDeviceToDevice, c->stream));
            GEMB_CUDA(cudaMemcpyAsync(delta, syn_neg, sizeof(float) * tab, cudaMemcpyDeviceToDevice, c->stream));
        }
        if (n_local > 0) GEMB_TRY(launch_sgns(c, P, blocks, threads));
        if (c->nranks > 1) {
            // embedding-"gradient" all-reduce once per epoch: table <- table0 + sum_ranks (table_r - table0)
            NcclApi *api = nccl_api();
            if (!api) return GEMB_ERR_NCCL;
            GEMB_TRY(c->t_comm.begin(c->stream));
            // syn_neg: delta held the pre-epoch copy
            GEMB_TRY(axpy_launch(c, tabn, -1.f, delta, syn_neg));        // syn_neg := d_neg
            ncclResult_t r = api->AllReduce(syn_neg, syn_neg, tab, ncclFloat, ncclSum, (ncclComm_t)c->comm, c->stream);
            GEMB_TRY(axpy_launch(c, tabn, 1.f, delta, syn_neg));         // + neg0
            GEMB_TRY(axpy_launch(c, tabn, -1.f, pos0, syn_pos));         // syn_pos := d_pos
            if (r == ncclSuccess) r = api->AllReduce(syn_pos, syn_pos, tab, ncclFloat, ncclSum, (ncclComm_t)c->comm, c->stream);
            GEMB_TRY(axpy_launch(c, tabn, 1.f, pos0, syn_pos));          // + pos0
            if (r != ncclSuccess) { set_error("nccl embedding allreduce: %s", api->GetErrorString(r)); return GEMB_ERR_NCCL; }
            GEMB_TRY(c->t_comm.end(c->stream));
        }
    }
    GEMB_CUDA(cudaEventRecord(ev[4], c->stream));
    if (X_out) GEMB_CUDA(cudaMemcpyAsync(X_out, syn_pos, sizeof(float) * tab, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaEventRecord(ev[5], c->stream));
    unsigned long long h_pairs = 0;
    GEMB_CUDA(cudaMemcpyAsync(&h_pairs, D.pairs.get(), sizeof h_pairs, cudaMemcpyDeviceToHost, c->stream));
    GEMB_CUDA(cudaStreamSynchronize(c->stream));
    if (c->nranks > 1) { comm_ms = c->t_comm.total_ms(); c->t_comm.reset(); }
    if (stats) {
        stats->vocab_ms = vocab_ms;
        stats->sgns_ms = ev.ms(3, 4);
        stats->total_ms = ev.ms(0, 4);
        stats->d2h_ms = ev.ms(4, 5);
        stats->comm_ms = comm_ms;
        stats->n_tokens = V;
        stats->pairs = (int64_t)h_pairs;
        stats->sgns_bytes = (double)h_pairs * 14.0 * 4.0 * (double)d;
    }
    return GEMB_OK;
}

}  // extern "C"
