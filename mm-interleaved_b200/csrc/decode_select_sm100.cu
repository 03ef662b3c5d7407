// decode_select_sm100.cu -- one decode step's token choice: HF's logits processors (repetition penalty, min-length),
// then arg-max or temperature + top-p sampling, then the finished / pad bookkeeping, in one launch with one CTA per row.
//
// The processed score of a token is a pure function of its logit and two bits (already generated -> penalised; eos
// while step < min_length -> -inf), so the kernel keeps two V-bit maps in shared memory and re-reads the fp32 row on
// every pass (L1 / L2 resident after the first: 128 KB at the model's 32002 ids) instead of staging a modified copy.
// That also gives HF's "once per distinct id" penalty for free: a repeated id sets the same bit.
//
// Top-p without a sort.  With weights w_i = exp(x_i - max) (x = processed score / temperature), HF drops a token when
// the ascending cumulative softmax mass up to and including it is <= 1 - top_p.  The kept set is therefore every token
// with w_i >= tau, tau the smallest weight whose "mass of all tokens with weight <= tau" exceeds (1 - top_p) * Z.  tau
// is found by a radix select over the fp32 bits of w (non-negative floats order like their bit patterns): four passes
// of 256-bin histograms of MASS over the next 8 bits of the tokens matching the prefix found so far.  Masses are 2^-40
// fixed point summed with 64-bit integer atomics, so every sum is exact and independent of order: the result is
// run-to-run reproducible.  All tokens tied exactly at tau are kept (HF's sort keeps an arbitrary subset of them);
// the arg-max is always kept.  The draw is an inverse CDF over the kept set in vocabulary order, with the same fixed
// point masses: the first id whose running kept mass exceeds floor(u * kept mass), u from Philox4x32-10 keyed by
// (seed, row, step) or taken from `uniforms[row]`.
#include <curand_philox4x32_x.h>

#include "common.cuh"

namespace mmfs {
namespace {

constexpr int kThreads = 512, kWarps = kThreads / 32;
constexpr int kHistCopies = 4;            // warps w and w + 4k share histogram w % 4
constexpr int kMaxV = 1 << 17;            // two V-bit maps in dynamic shared memory: <= 32 KiB
constexpr float kFix = 1099511627776.f;   // 2^40: w in [0, 1] -> fixed-point mass

struct Params { float penalty, temperature, top_p; };

// eager's `scores / p` with a Python float p multiplies by the fp32 reciprocal of p (PyTorch turns a division by a
// host scalar into a multiplication); the kernel rounds the same way so greedy tokens match the eager loop bit for bit
__device__ __forceinline__ float recip(float p) { return __fdiv_rn(1.f, p); }

struct Row {
    const float *s;
    const uint32_t *pen, *ban;
    float p, inv_p;
    bool any_pen;
    // HF RepetitionPenaltyLogitsProcessor, then MinLengthLogitsProcessor
    __device__ __forceinline__ float score(int i) const {
        const float x = __ldg(s + i);
        const uint32_t bit = 1u << (i & 31);
        if (ban[i >> 5] & bit) return -INFINITY;
        if (any_pen && (pen[i >> 5] & bit)) return x < 0.f ? x * p : x * inv_p;
        return x;
    }
};

// f(i, score(i)) for i = lo, lo + stride, ... < hi; the loads of kUnroll elements are issued before any is used (one
// CTA per row: without that memory-level parallelism every pass is a chain of dependent load latencies)
constexpr int kUnroll = 8;
template <typename F>
__device__ __forceinline__ void visit(const Row &row, int lo, int hi, int stride, F &&f) {
    for (int base = lo; base < hi; base += kUnroll * stride) {
        float x[kUnroll];
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) x[k] = base + k * stride < hi ? row.score(base + k * stride) : 0.f;
#pragma unroll
        for (int k = 0; k < kUnroll; ++k)
            if (base + k * stride < hi) f(base + k * stride, x[k]);
    }
}

__device__ __forceinline__ void argmax_merge(float &v, int &i, float ov, int oi) {
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }      // first index wins ties, like torch.argmax
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long x) {
#pragma unroll
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    return x;
}

__device__ __forceinline__ unsigned long long warp_incl_scan(unsigned long long x, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    return x;
}

__global__ void __launch_bounds__(kThreads) decode_select_kernel(
    const float *__restrict__ logits, long ld, int64_t *__restrict__ out_ids, const int64_t *__restrict__ step_p,
    uint8_t *__restrict__ finished, int64_t *__restrict__ next_ids, const int64_t *__restrict__ eos, int n_eos,
    long pad_id, int min_length, const Params *__restrict__ prm, const int64_t *__restrict__ seed_p,
    const float *__restrict__ uniforms, int V, int max_new, int mode) {
    extern __shared__ uint32_t bits[];                            // [pen: W words][ban: W words]
    __shared__ unsigned long long hist[kHistCopies][256];
    __shared__ unsigned long long wsum[kWarps];
    __shared__ float red_v[kWarps];
    __shared__ int red_i[kWarps];
    __shared__ unsigned long long sel_below, sel_target;
    __shared__ uint32_t sel_prefix;
    __shared__ int sel_id, sel_warp;

    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long t = *step_p;
    if (t < 0 || t >= max_new) return;                            // nothing to write outside out_ids
    const int W = (V + 31) >> 5;
    uint32_t *pen = bits, *ban = bits + W;
    const Params P = *prm;
    const bool any_pen = P.penalty != 1.f;
    int64_t *hist_ids = out_ids + (long)b * max_new;

    for (int i = tid; i < 2 * W; i += kThreads) bits[i] = 0u;
    __syncthreads();
    if (any_pen)
        for (long j = tid; j < t; j += kThreads) {
            const int64_t id = hist_ids[j];
            if (id >= 0 && id < V) atomicOr(pen + (id >> 5), 1u << (id & 31));
        }
    if (t < min_length)
        for (int j = tid; j < n_eos; j += kThreads) {
            const int64_t id = eos[j];
            if (id >= 0 && id < V) atomicOr(ban + (id >> 5), 1u << (id & 31));
        }
    __syncthreads();

    const Row row{logits + (long)b * ld, pen, ban, P.penalty, recip(P.penalty), any_pen};
    const bool sample = mode == MMFS_SELECT_SAMPLE;
    const float inv_t = sample ? recip(P.temperature) : 1.f;      // eager: scores / temperature

    // ---- pass 1: arg-max of the processed (and, sampling, temperature-scaled) scores
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    visit(row, tid, V, kThreads, [&](int i, float x) { argmax_merge(bv, bi, sample ? x * inv_t : x, i); });
#pragma unroll
    for (int o = 16; o; o >>= 1) argmax_merge(bv, bi, __shfl_xor_sync(0xffffffffu, bv, o), __shfl_xor_sync(0xffffffffu, bi, o));
    if (lane == 0) { red_v[warp] = bv; red_i[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kWarps; ++w) argmax_merge(bv, bi, red_v[w], red_i[w]);
        red_v[0] = bv; red_i[0] = bi;
    }
    __syncthreads();
    const float vmax = red_v[0];
    int id = red_i[0];

    if (sample && vmax > -INFINITY) {
        // fixed-point weight of token i and the fp32 bits of exp(x - max) the radix select orders by
        auto weight = [&](float x, uint32_t &key) -> unsigned long long {
            const float w = expf(x * inv_t - vmax);
            key = __float_as_uint(w);
            return __float2ull_rn(w * kFix);
        };
        // ---- passes 2-5: radix select of tau, 8 bits per pass, most significant first
        unsigned long long below = 0, thr = 0;
        uint32_t prefix = 0;
        for (int level = 0; level < 4; ++level) {
            const int shift = 24 - 8 * level;
            for (int i = tid; i < kHistCopies * 256; i += kThreads) (&hist[0][0])[i] = 0ull;
            __syncthreads();
            visit(row, tid, V, kThreads, [&](int, float x) {
                uint32_t key;
                const unsigned long long q = weight(x, key);
                if (q && (level == 0 || (key >> (shift + 8)) == prefix)) atomicAdd(&hist[warp % kHistCopies][(key >> shift) & 255u], q);
            });
            __syncthreads();
            if (warp == 0) {                                      // lane l owns bins 8l .. 8l+7
                unsigned long long m[8], tot = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    m[k] = 0;
#pragma unroll
                    for (int c = 0; c < kHistCopies; ++c) m[k] += hist[c][8 * lane + k];
                    tot += m[k];
                }
                const unsigned long long incl = warp_incl_scan(tot, lane), excl = incl - tot;
                if (level == 0) {                                 // Z = all mass; drop mass <= (1 - top_p) Z
                    const double keep = 1.0 - (double)P.top_p;
                    thr = keep > 0.0 ? (unsigned long long)(keep * (double)__shfl_sync(0xffffffffu, incl, 31)) : 0ull;
                }
                int cross = -1, last = -1;
                unsigned long long acc = below + excl, at_cross = 0, at_last = 0;   // mass below bin k
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (cross < 0 && acc + m[k] > thr) { cross = k; at_cross = acc; }
                    if (m[k]) { last = k; at_last = acc; }
                    acc += m[k];
                }
                const unsigned cross_mask = __ballot_sync(0xffffffffu, cross >= 0);
                const unsigned last_mask = __ballot_sync(0xffffffffu, last >= 0);
                // first bin where the mass crosses the threshold; else (top_p <= 0) the heaviest-weight bin with mass
                const int owner = cross_mask ? __ffs(cross_mask) - 1 : 31 - __clz(last_mask);
                if (lane == owner) {
                    sel_below = cross_mask ? at_cross : at_last;
                    sel_prefix = (prefix << 8) | (uint32_t)(8 * lane + (cross_mask ? cross : last));
                }
            }
            __syncthreads();
            below = sel_below;
            prefix = sel_prefix;
            __syncthreads();                                      // hist / sel_* are rewritten next level
        }
        const uint32_t tau = prefix;

        // ---- pass 6: kept mass per warp range (vocabulary order), then the inverse CDF
        const int span = (((V + kWarps - 1) / kWarps) + 31) & ~31;
        const int lo = warp * span, hi = min(V, lo + span);
        unsigned long long acc = 0;
        visit(row, lo + lane, hi, 32, [&](int, float x) {
            uint32_t key;
            const unsigned long long q = weight(x, key);
            acc += key >= tau ? q : 0ull;
        });
        acc = warp_sum(acc);
        if (lane == 0) wsum[warp] = acc;
        __syncthreads();
        if (tid == 0) {
            unsigned long long kept = 0;
            for (int w = 0; w < kWarps; ++w) kept += wsum[w];
            unsigned long long target;
            if (uniforms) {
                const double u = fmin(fmax((double)uniforms[b], 0.0), 1.0);
                target = (unsigned long long)(u * (double)kept);
            } else {
                const uint64_t s = (uint64_t)*seed_p;
                const uint4 r = curand_Philox4x32_10(make_uint4((uint32_t)t, (uint32_t)((uint64_t)t >> 32), (uint32_t)b, 0u),
                                                     make_uint2((uint32_t)s, (uint32_t)(s >> 32)));
                target = __umul64hi(((unsigned long long)r.y << 32) | r.x, kept);
            }
            if (target >= kept) target = kept - 1;                // kept > 0: the arg-max has weight 1
            int w = 0;
            while (target >= wsum[w]) target -= wsum[w++];
            sel_warp = w;
            sel_target = target;
        }
        __syncthreads();
        if (warp == sel_warp) {
            unsigned long long run = 0;
            const unsigned long long target = sel_target;
            bool found = false;
            for (int base = lo; base < hi && !found; base += 32 * kUnroll) {
                float x[kUnroll];
#pragma unroll
                for (int k = 0; k < kUnroll; ++k) {
                    const int i = base + 32 * k + lane;
                    x[k] = i < hi ? row.score(i) : -INFINITY;          // weight 0 past the range
                }
#pragma unroll
                for (int k = 0; k < kUnroll; ++k) {
                    if (found) break;
                    uint32_t key;
                    unsigned long long q = weight(x[k], key);
                    if (key < tau) q = 0;
                    const unsigned long long incl = warp_incl_scan(q, lane);
                    const unsigned hit = __ballot_sync(0xffffffffu, run + incl > target);
                    if (hit) {
                        if (lane == 0) sel_id = base + 32 * k + __ffs(hit) - 1;
                        found = true;
                    }
                    run += __shfl_sync(0xffffffffu, incl, 31);
                }
            }
        }
        __syncthreads();
        id = sel_id;
    }

    // ---- bookkeeping: finished rows emit pad, finished |= id in eos, out_ids[b, step], next_ids[b]
    if (tid == 0) {
        bool fin = finished[b] != 0;
        long long tok = fin ? (long long)pad_id : (long long)id;
        for (int j = 0; j < n_eos; ++j) fin |= tok == eos[j];
        finished[b] = fin ? 1 : 0;
        hist_ids[t] = tok;
        next_ids[b] = tok;
    }
}

}  // namespace
}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_decode_select(const float *logits, long ld, int64_t *out_ids, const int64_t *step, uint8_t *finished,
                                  int64_t *next_ids, const int64_t *eos_ids, int n_eos, long pad_id, int min_length,
                                  const float *params, const int64_t *seed, const float *uniforms, int B, int V,
                                  int max_new, int mode, void *stream) {
    MMFS_CHECK_ARG(B > 0 && V > 0 && max_new > 0, "decode_select: B, V and max_new must be positive");
    MMFS_CHECK_ARG(V <= kMaxV, "decode_select: V %d exceeds %d", V, kMaxV);
    MMFS_CHECK_ARG(ld >= V, "decode_select: row stride ld %ld < V %d", ld, V);
    MMFS_CHECK_ARG(n_eos >= 0, "decode_select: negative eos count");
    MMFS_CHECK_ARG(mode == MMFS_SELECT_GREEDY || mode == MMFS_SELECT_SAMPLE, "decode_select: bad mode %d", mode);
    MMFS_CHECK_ARG(logits && out_ids && step && finished && next_ids && params && (eos_ids || n_eos == 0) &&
                       (seed || uniforms || mode == MMFS_SELECT_GREEDY),
                   "decode_select: null pointer argument");
    const size_t smem = 2 * (size_t)((V + 31) / 32) * sizeof(uint32_t);
    decode_select_kernel<<<B, kThreads, smem, (cudaStream_t)stream>>>(
        logits, ld, out_ids, step, finished, next_ids, eos_ids, n_eos, pad_id, min_length,
        reinterpret_cast<const Params *>(params), seed, uniforms, V, max_new, mode);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}
