// beam_select_sm100.cu -- one step of beam search on the device: the scoring and hypothesis bookkeeping of HF
// `beam_search` + `BeamSearchScorer.process` (transformers 4.31, early_stopping=False) as InterleavedForward._beam_search
// spells them out, and the in-place reorder of the generated positions of the KV cache.
//
// Scoring (one CTA per beam row).  The processed score of a token is log_softmax(x)[i], repetition-penalised if the id
// is in the row's generated history, -inf for an eos id while step < min_length, plus the row's beam score.  Like
// decode_select, the kernel keeps the penalty / ban facts as two V-bit maps in shared memory and recomputes the score
// from the fp32 row on every pass instead of staging a modified copy.  The row's top K (K = max(2, 1 + n_eos) * nb, the
// reference's candidate count) is found by a radix select over the order-preserving uint32 image of the score bits,
// 8 bits per pass, then collected; a sequence's global top K lies within the union of its rows' top-K lists.
//
// Candidate order.  A candidate is the 64-bit word (score key << 32) | (2^32 - 1 - flat), flat = row_in_group * V +
// token, so one unsigned comparison orders candidates by higher score first and, on exactly equal scores, by the lower
// flat index.  (torch.topk's order on exact ties is unspecified; this is the rule the kernel documents.)
//
// Bookkeeping (one CTA per sequence, second launch).  The nb lists are merged by rank, then thread 0 runs the scorer
// exactly as the eager loop does: an eos candidate of rank < nb becomes a hypothesis scored sum_logprobs /
// max(len, 1) ** length_penalty (in double, like the host), an eos candidate of rank >= nb is skipped, and non-eos
// candidates fill the nb next beams.  At most nb hypotheses are kept per sequence in slots that carry an insertion
// serial; a full set drops the first (lowest serial) of its lowest-scored hypotheses, as `min()` over the eager list
// does.  The generated-id history is reordered by parent with each thread owning whole columns of the nb rows of the
// sequence (read all rows into registers, then write), so the in-place permutation is race-free.
//
// Beam sample (HF 4.31 `beam_sample`).  Same bookkeeping; only the candidates differ.  Per row the score above is
// divided by the temperature, then top-k (ties at the k-th value kept) and top-p (decode_select's rule,
// min_tokens_to_keep = 2) remove tokens, and the draw is a Gumbel-top-k race: key = s - log(-log u) over the kept
// tokens.  The 2 * nb largest keys of a sequence's nb * V entries are an exact draw without replacement proportional to
// softmax(s) -- torch.multinomial without replacement runs the same race, topk(p / q) with q ~ Exp(1) -- and they lie
// in the union of the rows' top 2 * nb lists.  The sequence kernel keeps the top 2 * nb keys, orders them by s (higher
// first, then the lower flat index) and runs the scorer on them; a sequence left with fewer than nb non-eos candidates
// sets the sticky error flag (4.31 raises ValueError there).
#include <curand_philox4x32_x.h>

#include "common.cuh"

namespace mmfs {
namespace {

constexpr int kThreads = 512, kWarps = kThreads / 32;
constexpr int kMaxV = 1 << 17;                     // two V-bit maps in dynamic shared memory: <= 32 KiB
constexpr int kMaxBeams = 8, kMaxEos = 4;
constexpr int kMaxK = 5 * kMaxBeams;              // max(2, 1 + kMaxEos) * kMaxBeams
constexpr int kReorderThreads = 128;
constexpr float kFix = 1099511627776.f;           // 2^40: a weight in [0, 1] -> fixed-point mass (as decode_select)

__device__ __forceinline__ float recip(float p) { return __fdiv_rn(1.f, p); }   // as decode_select rounds s / p

// order-preserving image of an fp32 value: larger float <=> larger key (-0 is folded into +0 first)
__device__ __forceinline__ uint32_t float_key(float x) {
    const uint32_t u = __float_as_uint(x == 0.f ? 0.f : x);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

__device__ __forceinline__ void lse_merge(float &m, float &s, float om, float os) {
    if (om == -INFINITY) return;
    if (m == -INFINITY) { m = om; s = os; return; }
    if (om > m) { s = s * expf(m - om) + os; m = om; }
    else s += os * expf(om - m);
}

struct Row {
    const float *x;
    const uint32_t *pen, *ban;
    float max, logsum, p, inv_p, bs;
    bool any_pen;
    // log_softmax -> RepetitionPenaltyLogitsProcessor -> MinLengthLogitsProcessor -> + beam score
    __device__ __forceinline__ float score(int i) const {
        const uint32_t bit = 1u << (i & 31);
        if (ban[i >> 5] & bit) return -INFINITY;
        float s = (__ldg(x + i) - max) - logsum;
        if (any_pen && (pen[i >> 5] & bit)) s = s < 0.f ? s * p : s * inv_p;
        return s + bs;
    }
};

// Row set-up shared by both row kernels: the penalty / ban bit maps and log_softmax's max and log-sum of the row.
__device__ __forceinline__ Row load_row(const float *x, long t, float p, const int64_t *hist_r, const int64_t *eos,
                                        int n_eos, int min_length, float bs, int V, uint32_t *bits, float *red_m,
                                        float *red_s) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int W = (V + 31) >> 5;
    uint32_t *pen = bits, *ban = bits + W;
    const bool any_pen = p != 1.f;
    for (int i = tid; i < 2 * W; i += kThreads) bits[i] = 0u;
    __syncthreads();
    if (any_pen)
        for (long j = tid; j < t; j += kThreads) {
            const int64_t id = hist_r[j];
            if (id >= 0 && id < V) atomicOr(pen + (id >> 5), 1u << (id & 31));
        }
    if (t < min_length)
        for (int j = tid; j < n_eos; j += kThreads) {
            const int64_t id = eos[j];
            if (id >= 0 && id < V) atomicOr(ban + (id >> 5), 1u << (id & 31));
        }

    // max and sum of exp(x - max), online
    float m = -INFINITY, s = 0.f;
    for (int i = tid; i < V; i += kThreads) lse_merge(m, s, __ldg(x + i), 1.f);
#pragma unroll
    for (int o = 16; o; o >>= 1) lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) { red_m[warp] = m; red_s[warp] = s; }
    __syncthreads();                                                 // also publishes the bit maps
    if (tid == 0) {
        for (int w = 1; w < kWarps; ++w) lse_merge(m, s, red_m[w], red_s[w]);
        red_m[0] = m; red_s[0] = s;
    }
    __syncthreads();
    const Row row{x, pen, ban, red_m[0], logf(red_s[0]), p, recip(p), bs, any_pen};
    __syncthreads();                                                 // red_m / red_s may be reused
    return row;
}

struct SelectSmem {
    unsigned hist8[256];
    unsigned sel_prefix, sel_need, sel_eq, n_gt, taken;
    unsigned wcnt[kWarps], wofs[kWarps];
};
struct Sel {
    uint32_t thr;                                                    // the K-th largest key
    unsigned need, eq;                                               // how many of its ties are taken, of how many
};

// Radix select of the K-th largest key(i) over i < V (K <= V), most significant byte first.
template <typename KeyF>
__device__ __forceinline__ Sel radix_select(const KeyF &key, int V, unsigned K, SelectSmem &sm) {
    const int tid = threadIdx.x;
    unsigned prefix = 0, need = K;
    for (int level = 0; level < 4; ++level) {
        const int shift = 24 - 8 * level;
        for (int i = tid; i < 256; i += kThreads) sm.hist8[i] = 0u;
        __syncthreads();
        for (int i = tid; i < V; i += kThreads) {
            const uint32_t k = key(i);
            if (level == 0 || (k >> (shift + 8)) == prefix) atomicAdd(&sm.hist8[(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned above = 0;
            int d = 255;
            for (; d > 0 && above + sm.hist8[d] < need; --d) above += sm.hist8[d];
            sm.sel_prefix = (prefix << 8) | (unsigned)d;
            sm.sel_need = need - above;
            sm.sel_eq = sm.hist8[d];
        }
        __syncthreads();
        prefix = sm.sel_prefix;
        need = sm.sel_need;
        __syncthreads();                                             // hist8 / sel_* are rewritten next level
    }
    return Sel{prefix, need, sm.sel_eq};
}

// Calls emit(slot, i, key(i)) for the K largest keys, slots 0..K-1 in no particular order: every key above the
// threshold, then the `need` lowest token ids among the ties at it.
template <typename KeyF, typename EmitF>
__device__ __forceinline__ void collect_top(const KeyF &key, int V, unsigned K, Sel sel, SelectSmem &sm, EmitF &&emit) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t thr = sel.thr;
    const unsigned need = sel.need, n_above = K - need;
    if (tid == 0) { sm.n_gt = 0; sm.taken = 0; }
    __syncthreads();
    const bool all_ties = sel.eq == need;
    for (int i = tid; i < V; i += kThreads) {
        const uint32_t k = key(i);
        if (k > thr) emit(atomicAdd(&sm.n_gt, 1u), i, k);
        else if (all_ties && k == thr) emit(n_above + atomicAdd(&sm.taken, 1u), i, k);
    }
    if (all_ties) return;
    for (int base = 0; base < V; base += kThreads) {
        const int i = base + tid;
        const bool eq = i < V && key(i) == thr;
        const unsigned ball = __ballot_sync(0xffffffffu, eq);
        if (lane == 0) sm.wcnt[warp] = __popc(ball);
        __syncthreads();
        if (tid == 0) {
            unsigned acc = 0;
            for (int w = 0; w < kWarps; ++w) { sm.wofs[w] = acc; acc += sm.wcnt[w]; }
            sm.wcnt[0] = acc;                                        // chunk total, read after the next barrier
        }
        __syncthreads();
        const unsigned before = sm.taken;
        if (eq) {
            const unsigned rank = before + sm.wofs[warp] + __popc(ball & ((1u << lane) - 1u));
            if (rank < need) emit(n_above + rank, i, thr);
        }
        __syncthreads();
        if (tid == 0) sm.taken = before + sm.wcnt[0];
        __syncthreads();
        if (sm.taken >= need) break;
    }
}

__device__ __forceinline__ unsigned long long cand_word(uint32_t k, unsigned long long flat) {
    return ((unsigned long long)k << 32) | (0xffffffffull - flat);
}

__global__ void __launch_bounds__(kThreads) beam_rows_kernel(
    const float *__restrict__ logits, long ld, const int64_t *__restrict__ step_p, const double *__restrict__ prm,
    const float *__restrict__ beam_scores, const int64_t *__restrict__ hist, const uint8_t *__restrict__ done,
    const int64_t *__restrict__ eos, int n_eos, int min_length, unsigned long long *__restrict__ cand, int nb, int K,
    int V, int max_new) {
    extern __shared__ uint32_t bits[];                               // [pen: W words][ban: W words]
    __shared__ SelectSmem sm;
    __shared__ float red_m[kWarps], red_s[kWarps];

    const int r = blockIdx.x;
    const long t = *step_p;
    if (t < 0 || t >= max_new || done[r / nb]) return;
    const Row row = load_row(logits + (long)r * ld, t, (float)prm[0], hist + (long)r * max_new, eos, n_eos, min_length,
                             beam_scores[r], V, bits, red_m, red_s);
    const auto key = [&](int i) { return float_key(row.score(i)); };
    const unsigned long long jV = (unsigned long long)(r % nb) * (unsigned)V;
    unsigned long long *out = cand + (long)r * K;
    collect_top(key, V, (unsigned)K, radix_select(key, V, (unsigned)K, sm), sm,
                [&](unsigned slot, int i, uint32_t k) { out[slot] = cand_word(k, jV + (unsigned)i); });
}

// The top-p cut of decode_select_sm100.cu, same rule and same 2^-40 fixed point (see the comment at its top): the
// smallest weight key tau whose mass of all tokens with weight <= tau exceeds (1 - top_p) * Z, by a radix select over
// the fp32 bits of the weights with 256-bin histograms of mass; every token with weight key >= tau is kept.
// mass(i, key) returns token i's fixed-point mass and sets key to the bits of its weight.
struct TopPSmem {
    unsigned long long hist[256], below, thr;
    uint32_t prefix;
};
template <typename MassF>
__device__ __forceinline__ uint32_t top_p_cut(const MassF &mass, int V, double top_p, TopPSmem &sm) {
    const int tid = threadIdx.x;
    uint32_t prefix = 0;
    for (int level = 0; level < 4; ++level) {
        const int shift = 24 - 8 * level;
        for (int i = tid; i < 256; i += kThreads) sm.hist[i] = 0ull;
        __syncthreads();
        for (int i = tid; i < V; i += kThreads) {
            uint32_t key;
            const unsigned long long q = mass(i, key);
            if (q && (level == 0 || (key >> (shift + 8)) == prefix)) atomicAdd(&sm.hist[(key >> shift) & 255u], q);
        }
        __syncthreads();
        if (tid == 0) {
            if (level == 0) {                                        // Z = all mass; drop mass <= (1 - top_p) Z
                unsigned long long z = 0;
                for (int d = 0; d < 256; ++d) z += sm.hist[d];
                const double keep = 1.0 - top_p;
                sm.thr = keep > 0.0 ? (unsigned long long)(keep * (double)z) : 0ull;
                sm.below = 0;
            }
            unsigned long long acc = sm.below, at_cross = 0, at_last = 0;
            int cross = -1, last = 0;
            for (int d = 0; d < 256; ++d) {
                const unsigned long long m = sm.hist[d];
                if (cross < 0 && acc + m > sm.thr) { cross = d; at_cross = acc; }
                if (m) { last = d; at_last = acc; }
                acc += m;
            }
            // the first bin where the mass crosses the threshold; else (top_p <= 0) the heaviest-weight bin with mass
            sm.below = cross >= 0 ? at_cross : at_last;
            sm.prefix = (prefix << 8) | (uint32_t)(cross >= 0 ? cross : last);
        }
        __syncthreads();
        prefix = sm.prefix;
        __syncthreads();
    }
    return prefix;
}

__device__ __forceinline__ void top2_merge(float &a1, float &a2, float b1, float b2) {
    if (b1 > a1) { a2 = fmaxf(a1, b2); a1 = b1; }
    else a2 = fmaxf(a2, b1);
}

// Beam-sample rows: the warped score s of every token (beam_rows_kernel's score, times 1 / temperature), the top-k
// threshold (radix select over the score keys), the top-p cut over the top-k-kept set (top_p_cut, then lowered to the
// second largest weight: min_tokens_to_keep = 2), and the row's M = 2 * nb largest Gumbel keys s - log(-log u) over the
// kept tokens, u from Philox4x32-10 keyed by (seed, step, row, token) or from uniforms[row, token].  Each candidate
// is two words: the draw word (Gumbel key, flat) and the score word (s key, flat; key 0 when the token is not kept, so
// not drawable: a row with fewer than M kept tokens).
__global__ void __launch_bounds__(kThreads) beam_sample_rows_kernel(
    const float *__restrict__ logits, long ld, const int64_t *__restrict__ step_p, const double *__restrict__ prm,
    const int64_t *__restrict__ seed_p, const float *__restrict__ uniforms, const float *__restrict__ beam_scores,
    const int64_t *__restrict__ hist, const uint8_t *__restrict__ done, const int64_t *__restrict__ eos, int n_eos,
    int min_length, unsigned long long *__restrict__ cand, int nb, int M, int top_k, int V, int max_new) {
    extern __shared__ uint32_t bits[];                               // [pen: W words][ban: W words]
    __shared__ SelectSmem sm;
    __shared__ TopPSmem tp;
    __shared__ float red_m[kWarps], red_s[kWarps];

    const int r = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long t = *step_p;
    if (t < 0 || t >= max_new || done[r / nb]) return;
    const Row row = load_row(logits + (long)r * ld, t, (float)prm[0], hist + (long)r * max_new, eos, n_eos, min_length,
                             beam_scores[r], V, bits, red_m, red_s);
    const float inv_t = recip((float)prm[2]);                        // eager: scores / temperature
    const double top_p = prm[3];
    const auto warped = [&](int i) { return row.score(i) * inv_t; };

    // ---- the two largest warped scores (with multiplicity)
    float m1 = -INFINITY, m2 = -INFINITY;
    for (int i = tid; i < V; i += kThreads) top2_merge(m1, m2, warped(i), -INFINITY);
#pragma unroll
    for (int o = 16; o; o >>= 1) top2_merge(m1, m2, __shfl_xor_sync(0xffffffffu, m1, o), __shfl_xor_sync(0xffffffffu, m2, o));
    if (lane == 0) { red_m[warp] = m1; red_s[warp] = m2; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kWarps; ++w) top2_merge(m1, m2, red_m[w], red_s[w]);
        red_m[0] = m1; red_s[0] = m2;
    }
    __syncthreads();
    const float wmax = red_m[0], w2 = red_s[0];

    // ---- top-k: keep every score >= the k-th largest, ties included
    const int k = top_k > 0 && top_k < V ? max(top_k, 2) : V;
    const uint32_t kthr = k < V ? radix_select([&](int i) { return float_key(warped(i)); }, V, (unsigned)k, sm).thr : 0u;

    // ---- top-p over the top-k-kept set
    uint32_t tau = 0;
    if (top_p < 1.0 && wmax > -INFINITY) {
        tau = top_p_cut([&](int i, uint32_t &key) -> unsigned long long {
            const float s = warped(i);
            if (float_key(s) < kthr) { key = 0; return 0ull; }
            const float w = expf(s - wmax);
            key = __float_as_uint(w);
            return __float2ull_rn(w * kFix);
        }, V, top_p, tp);
        tau = min(tau, __float_as_uint(expf(w2 - wmax)));
    }

    // ---- the draw: the row's M largest Gumbel keys over the kept tokens
    const uint64_t seed = uniforms ? 0ull : (uint64_t)*seed_p;
    const uint32_t none = float_key(-INFINITY);
    const auto gkey = [&](int i) -> uint32_t {
        const float s = warped(i);
        if (s == -INFINITY || float_key(s) < kthr || (tau && __float_as_uint(expf(s - wmax)) < tau)) return none;
        float u;
        if (uniforms) {
            u = __ldg(uniforms + (long)r * V + i);
        } else {
            const uint4 q = curand_Philox4x32_10(make_uint4((uint32_t)i, (uint32_t)r, (uint32_t)t, (uint32_t)((uint64_t)t >> 32)),
                                                 make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
            u = (float)(2u * (q.x >> 9) + 1u) * 0x1p-24f;            // in (0, 1), exactly representable
        }
        return float_key(s - logf(-logf(u)));
    };
    const unsigned long long jV = (unsigned long long)(r % nb) * (unsigned)V;
    unsigned long long *out = cand + 2L * r * M;
    collect_top(gkey, V, (unsigned)M, radix_select(gkey, V, (unsigned)M, sm), sm, [&](unsigned slot, int i, uint32_t g) {
        const unsigned long long flat = jV + (unsigned)i;
        out[2 * slot] = cand_word(g, flat);
        out[2 * slot + 1] = cand_word(g > none ? float_key(warped(i)) : 0u, flat);
    });
}

// element k of a register array indexed at run time, without local memory
template <typename T>
__device__ __forceinline__ T pick(const T (&a)[kMaxBeams], int k) {
    T v = a[0];
#pragma unroll
    for (int j = 1; j < kMaxBeams; ++j)
        if (j == k) v = a[j];
    return v;
}

// sample == 0: cand holds the rows' top K score words (beam_rows_kernel); sample == 1: the rows' top K (draw word,
// score word) pairs (beam_sample_rows_kernel), and a shortage of continuing beams sets *error.
__global__ void __launch_bounds__(kThreads) beam_seq_kernel(
    const int64_t *__restrict__ step_p, const double *__restrict__ prm, float *__restrict__ beam_scores,
    int64_t *__restrict__ hist, int64_t *__restrict__ next_ids, int64_t *__restrict__ parent, uint8_t *__restrict__ done,
    double *__restrict__ hyp_scores, int64_t *__restrict__ hyp_ids, int64_t *__restrict__ hyp_meta,
    const int64_t *__restrict__ eos, int n_eos, long pad_id, const unsigned long long *__restrict__ cand, int nb, int K,
    int V, int max_new, int sample, int32_t *__restrict__ error) {
    __shared__ unsigned long long all[kMaxBeams * kMaxK];
    __shared__ unsigned long long top[kMaxK];
    __shared__ float s_score[kMaxBeams];
    __shared__ int64_t s_tok[kMaxBeams];
    __shared__ int s_par[kMaxBeams];                                 // parent row within the group
    __shared__ int s_src[kMaxBeams];                                 // per hypothesis slot: source row in the group, or -1
    __shared__ int s_was_done;

    const int b = blockIdx.x, tid = threadIdx.x;
    const long t = *step_p;
    if (t < 0 || t >= max_new) return;
    const long row0 = (long)b * nb;

    if (tid == 0) s_was_done = done[b];
    if (tid < kMaxBeams) s_src[tid] = -1;
    __syncthreads();
    if (s_was_done) {                                                // finished sequence: pad, score 0, parent b * nb
        if (tid < nb) { s_score[tid] = 0.f; s_tok[tid] = pad_id; s_par[tid] = 0; }
    } else {
        const int N = nb * K;
        if (!sample) {
            for (int i = tid; i < N; i += kThreads) all[i] = cand[row0 * K + i];
            __syncthreads();
            for (int i = tid; i < N; i += kThreads) {                // rank sort: every word is distinct (flat index)
                const unsigned long long c = all[i];
                int rank = 0;
                for (int j = 0; j < N; ++j) rank += all[j] > c;
                if (rank < K) top[rank] = c;
            }
        } else {                                                     // (draw word, score word) pairs, N <= 128
            unsigned long long *draw = all, *score = all + N, *drawn = all + 2 * N;
            for (int i = tid; i < N; i += kThreads) {
                draw[i] = cand[2 * (row0 * K + i)];
                score[i] = cand[2 * (row0 * K + i) + 1];
            }
            __syncthreads();
            for (int i = tid; i < N; i += kThreads) {                // the K largest draw keys ...
                int rank = 0;
                for (int j = 0; j < N; ++j) rank += draw[j] > draw[i];
                if (rank < K) drawn[rank] = score[i];
            }
            __syncthreads();
            for (int i = tid; i < K; i += kThreads) {                // ... ordered by score
                int rank = 0;
                for (int j = 0; j < K; ++j) rank += drawn[j] > drawn[i];
                top[rank] = drawn[i];
            }
        }
        __syncthreads();
        if (tid == 0) {
            const double lp = prm[1];
            double hs[kMaxBeams];
            long long serial[kMaxBeams];
            int count = 0;
            long long next_serial = 0;
            for (int j = 0; j < nb; ++j) {
                hs[j] = hyp_scores[row0 + j];
                serial[j] = hyp_meta[2 * (row0 + j) + 1];
                if (hyp_meta[2 * (row0 + j)] >= 0) {
                    ++count;
                    next_serial = max(next_serial, serial[j] + 1);
                }
            }
            const double len_norm = pow((double)max(t, 1L), lp);
            int k = 0;
            for (int rank = 0; rank < K && k < nb; ++rank) {
                const unsigned long long c = top[rank];
                if (!(c >> 32)) break;                               // key 0: a token beam_sample could not draw
                const float sc = key_float((uint32_t)(c >> 32));
                const unsigned flat = 0xffffffffu - (unsigned)(c & 0xffffffffull);
                const int j = (int)(flat / (unsigned)V);
                const int64_t tok = (int64_t)(flat % (unsigned)V);
                bool is_eos = false;
                for (int e = 0; e < n_eos; ++e) is_eos |= tok == eos[e];
                if (!is_eos) {
                    s_score[k] = sc; s_tok[k] = tok; s_par[k] = j; ++k;
                    continue;
                }
                if (rank >= nb) continue;
                const double score = (double)sc / len_norm;
                int slot = -1;
                if (count < nb) {                                    // a free slot
                    for (int q = 0; q < nb && slot < 0; ++q)
                        if (hyp_meta[2 * (row0 + q)] < 0 && s_src[q] < 0) slot = q;
                    ++count;
                } else {
                    int lo = -1;                                     // the first of the lowest-scored hypotheses
                    for (int q = 0; q < nb; ++q)
                        if (lo < 0 || hs[q] < hs[lo] || (hs[q] == hs[lo] && serial[q] < serial[lo])) lo = q;
                    if (score > hs[lo]) slot = lo;
                }
                if (slot < 0) continue;
                hs[slot] = score;
                serial[slot] = next_serial++;
                s_src[slot] = j;
                hyp_meta[2 * (row0 + slot)] = t;                     // the slot now reads as taken
                hyp_meta[2 * (row0 + slot) + 1] = serial[slot];
                hyp_scores[row0 + slot] = score;
            }
            if (k < nb && error) *error = 1;                         // beam_sample: 4.31 raises ValueError here
            for (; k < nb; ++k) { s_score[k] = 0.f; s_tok[k] = pad_id; s_par[k] = 0; }
            if (count >= nb) {                                       // BeamHypotheses.is_done, early_stopping=False
                double worst = hs[0];
                for (int q = 1; q < nb; ++q) worst = fmin(worst, hs[q]);
                const float best = key_float((uint32_t)(top[0] >> 32));
                if (worst >= (double)best / pow((double)(t + 1), lp)) done[b] = 1;
            }
        }
    }
    __syncthreads();

    // ---- history: hypotheses copy the old rows, then rows take their parent's ids and append the new token
    int par[kMaxBeams], src[kMaxBeams];
#pragma unroll
    for (int j = 0; j < kMaxBeams; ++j) { par[j] = j < nb ? s_par[j] : 0; src[j] = s_src[j]; }
    for (long q = tid; q < t; q += kThreads) {
        int64_t old[kMaxBeams];
#pragma unroll
        for (int j = 0; j < kMaxBeams; ++j) old[j] = j < nb ? hist[(row0 + j) * max_new + q] : 0;
#pragma unroll
        for (int j = 0; j < kMaxBeams; ++j) {
            if (j >= nb) break;
            if (src[j] >= 0) hyp_ids[(row0 + j) * max_new + q] = pick(old, src[j]);
            hist[(row0 + j) * max_new + q] = pick(old, par[j]);
        }
    }
    if (tid < nb) {
        const long r = row0 + tid;
        hist[r * max_new + t] = s_tok[tid];
        beam_scores[r] = s_score[tid];
        next_ids[r] = s_tok[tid];
        parent[r] = row0 + s_par[tid];
    }
}

// One CTA per (position, sequence, cache tensor); each thread owns 16-byte columns of the nb rows of the sequence, so
// reading every source row into registers before writing any destination row makes the permutation in place and
// race-free.  Rows whose parent is themselves are neither read nor written.
__global__ void __launch_bounds__(kReorderThreads) kv_beam_reorder_kernel(
    char *__restrict__ cache, long cache_stride, long row_stride, long pos_stride, int cols, const int64_t *__restrict__ parent,
    const int64_t *__restrict__ cur_p, const int64_t *__restrict__ step_p, const uint8_t *__restrict__ done, int nb) {
    const long t = *step_p, p = blockIdx.x;
    if (p >= t) return;
    const int g = blockIdx.y;
    if (done && done[g]) return;
    const long pos = *cur_p - t + p;
    int par[kMaxBeams];
    unsigned moved = 0, needed = 0;
#pragma unroll
    for (int j = 0; j < kMaxBeams; ++j) {
        par[j] = j;
        if (j < nb) {
            const long q = parent[(long)g * nb + j] - (long)g * nb;
            if (q >= 0 && q < nb && q != j) { par[j] = (int)q; moved |= 1u << j; needed |= 1u << q; }
        }
    }
    if (!moved) return;
    char *base = cache + blockIdx.z * cache_stride + (long)g * nb * row_stride + pos * pos_stride;
    for (int c = threadIdx.x; c < cols; c += kReorderThreads) {
        uint4 v[kMaxBeams];
#pragma unroll
        for (int j = 0; j < kMaxBeams; ++j)
            v[j] = (needed & (1u << j)) ? *reinterpret_cast<const uint4 *>(base + j * row_stride + 16L * c) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < kMaxBeams; ++j)
            if (moved & (1u << j)) *reinterpret_cast<uint4 *>(base + j * row_stride + 16L * c) = pick(v, par[j]);
    }
}

}  // namespace
}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_beam_select(const float *logits, long ld, const int64_t *step, const double *params,
                                float *beam_scores, int64_t *history, int64_t *next_ids, int64_t *parent, uint8_t *done,
                                double *hyp_scores, int64_t *hyp_ids, int64_t *hyp_meta, const int64_t *eos_ids,
                                int n_eos, long pad_id, int min_length, uint64_t *scratch, int B, int num_beams, int V,
                                int max_new, void *stream) {
    MMFS_CHECK_ARG(B > 0 && V > 0 && max_new > 0 && num_beams > 0, "beam_select: B, num_beams, V and max_new must be positive");
    MMFS_CHECK_ARG(num_beams <= kMaxBeams, "beam_select: num_beams %d exceeds %d", num_beams, kMaxBeams);
    MMFS_CHECK_ARG(n_eos >= 0 && n_eos <= kMaxEos, "beam_select: eos count %d outside [0, %d]", n_eos, kMaxEos);
    const int K = (n_eos + 1 > 2 ? n_eos + 1 : 2) * num_beams;
    MMFS_CHECK_ARG(V <= kMaxV, "beam_select: V %d exceeds %d", V, kMaxV);
    MMFS_CHECK_ARG(V >= K, "beam_select: V %d is below the candidate count K %d", V, K);
    MMFS_CHECK_ARG(ld >= V, "beam_select: row stride ld %ld < V %d", ld, V);
    MMFS_CHECK_ARG(logits && step && params && beam_scores && history && next_ids && parent && done && hyp_scores &&
                       hyp_ids && hyp_meta && scratch && (eos_ids || n_eos == 0),
                   "beam_select: null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = 2 * (size_t)((V + 31) / 32) * sizeof(uint32_t);
    auto *cand = reinterpret_cast<unsigned long long *>(scratch);
    beam_rows_kernel<<<B * num_beams, kThreads, smem, st>>>(logits, ld, step, params, beam_scores, history, done, eos_ids,
                                                            n_eos, min_length, cand, num_beams, K, V, max_new);
    MMFS_CUDA(cudaGetLastError());
    beam_seq_kernel<<<B, kThreads, 0, st>>>(step, params, beam_scores, history, next_ids, parent, done, hyp_scores, hyp_ids,
                                            hyp_meta, eos_ids, n_eos, pad_id, cand, num_beams, K, V, max_new, 0, nullptr);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

extern "C" int mmfs_beam_sample(const float *logits, long ld, const int64_t *step, const double *params,
                                const int64_t *seed, const float *uniforms, float *beam_scores, int64_t *history,
                                int64_t *next_ids, int64_t *parent, uint8_t *done, double *hyp_scores, int64_t *hyp_ids,
                                int64_t *hyp_meta, int32_t *error, const int64_t *eos_ids, int n_eos, long pad_id,
                                int min_length, int top_k, uint64_t *scratch, int B, int num_beams, int V, int max_new,
                                void *stream) {
    MMFS_CHECK_ARG(B > 0 && V > 0 && max_new > 0 && num_beams > 0, "beam_sample: B, num_beams, V and max_new must be positive");
    MMFS_CHECK_ARG(num_beams <= kMaxBeams, "beam_sample: num_beams %d exceeds %d", num_beams, kMaxBeams);
    MMFS_CHECK_ARG(n_eos >= 0 && n_eos <= kMaxEos, "beam_sample: eos count %d outside [0, %d]", n_eos, kMaxEos);
    MMFS_CHECK_ARG(top_k >= 0, "beam_sample: negative top_k %d", top_k);
    const int M = 2 * num_beams;
    MMFS_CHECK_ARG(V <= kMaxV, "beam_sample: V %d exceeds %d", V, kMaxV);
    MMFS_CHECK_ARG(V >= M, "beam_sample: V %d is below the candidate count 2 * num_beams %d", V, M);
    MMFS_CHECK_ARG(ld >= V, "beam_sample: row stride ld %ld < V %d", ld, V);
    MMFS_CHECK_ARG(logits && step && params && beam_scores && history && next_ids && parent && done && hyp_scores &&
                       hyp_ids && hyp_meta && error && scratch && (eos_ids || n_eos == 0) && (seed || uniforms),
                   "beam_sample: null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = 2 * (size_t)((V + 31) / 32) * sizeof(uint32_t);
    auto *cand = reinterpret_cast<unsigned long long *>(scratch);
    beam_sample_rows_kernel<<<B * num_beams, kThreads, smem, st>>>(logits, ld, step, params, seed, uniforms, beam_scores,
                                                                   history, done, eos_ids, n_eos, min_length, cand,
                                                                   num_beams, M, top_k, V, max_new);
    MMFS_CUDA(cudaGetLastError());
    beam_seq_kernel<<<B, kThreads, 0, st>>>(step, params, beam_scores, history, next_ids, parent, done, hyp_scores, hyp_ids,
                                            hyp_meta, eos_ids, n_eos, pad_id, cand, num_beams, M, V, max_new, 1, error);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

extern "C" int mmfs_kv_beam_reorder(void *cache, int n_caches, long cache_stride, int rows, long row_stride,
                                    long pos_stride, long row_bytes, int num_beams, const int64_t *parent,
                                    const int64_t *cur, const int64_t *step, const uint8_t *done, int max_positions,
                                    void *stream) {
    MMFS_CHECK_ARG(n_caches > 0 && rows > 0 && num_beams > 0 && row_bytes > 0 && max_positions > 0,
                   "kv_beam_reorder: n_caches, rows, num_beams, row_bytes and max_positions must be positive");
    MMFS_CHECK_ARG(num_beams <= kMaxBeams, "kv_beam_reorder: num_beams %d exceeds %d", num_beams, kMaxBeams);
    MMFS_CHECK_ARG(rows % num_beams == 0, "kv_beam_reorder: rows %d is not a multiple of num_beams %d", rows, num_beams);
    MMFS_CHECK_ARG(cache && parent && cur && step, "kv_beam_reorder: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)cache | (unsigned long)cache_stride | (unsigned long)row_stride | (unsigned long)pos_stride |
                    (unsigned long)row_bytes) % 16 == 0,
                   "kv_beam_reorder: the cache pointer, strides and row_bytes must be multiples of 16 bytes");
    MMFS_CHECK_ARG(rows / num_beams <= 65535 && n_caches <= 65535, "kv_beam_reorder: too many sequences or caches");
    const dim3 grid(max_positions, rows / num_beams, n_caches);
    kv_beam_reorder_kernel<<<grid, kReorderThreads, 0, (cudaStream_t)stream>>>(
        (char *)cache, cache_stride, row_stride, pos_stride, (int)(row_bytes / 16), parent, cur, step, done, num_beams);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}
