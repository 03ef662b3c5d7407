// decode_common.cuh -- what the split-KV decode kernels share, over 16-bit / fp32 caches (attn_generic_sm100.cu) and
// E4M3 caches (kv_fp8_sm100.cu): the split geometry, the scratch layout, which cache row holds position j, and the
// epilogue that combines a CTA's warps and merges the splits of a (row, head).
//
// A launch over keys 0 .. last_key of `rows` query rows has grid (n_split, H, rows): every CTA reduces kDecKeys keys of
// one (row, head), kDecKPW per warp, and leaves an (m, l, acc[hd]) partial; the last CTA of a (row, head) to arrive merges
// them in split order and writes the output row.  The SHARED instantiations read a prompt stored once per group of G
// rows (see SharedLayout) and launch grid (n_split * G, H, rows / G) with blockIdx.x = split * G + g, so the G rows that
// read the same prefix tile are adjacent in launch order and share it through L2.  Only the addressing differs, so the
// output is bit-identical to the dense kernel's over the replicated cache.
#pragma once
#include "common.cuh"

namespace mmfs {

constexpr int kDecKeys = 256;                 // keys per CTA (one split)
constexpr int kDecWarps = 4;
constexpr int kDecKPW = kDecKeys / kDecWarps;

// The scratch buffer: one ticket per (row, head), padded to keep the partials 16-byte aligned, then one
// (acc[hd], m, l) partial per (row, head, split).
inline long decode_ticket_floats(int rows, int H) { return ((long)rows * H + 3) / 4 * 4; }
inline int decode_splits(int last_key) { return last_key / kDecKeys + 1; }

// the last key the single query row, at position `past`, sees; negative for a negative past
inline int decode_last_key(int causal, int past, int Tkv) { return causal ? (past < Tkv - 1 ? past : Tkv - 1) : Tkv - 1; }

// The SHARED cache: the query rows come in groups of G, one per prompt; row r's key / value at position j is row r / G
// of the (prompts, Tp, ...) prefix below *prefix_len (clamped to [0, Tp]), and row r of the (rows, max_new, ...)
// generated positions at min(j - prefix_len, max_new - 1) from there on.
struct SharedLayout {
    const long long *prefix_len = nullptr;
    int G = 1, Tp = 0, max_new = 1;           // as default-constructed: the dense cache, one row per group
};

inline dim3 decode_grid(int last_key, int rows, int H, const SharedLayout &sl) {
    return dim3(decode_splits(last_key) * sl.G, H, rows / sl.G);
}

// One CTA's split and query row, and the addressing of that row's cache
template <bool SHARED>
struct DecodeCta {
    int split, n_split, b, pb, plen, max_new;   // pb: the row's prompt (SHARED) or the row itself

    __device__ __forceinline__ explicit DecodeCta(const SharedLayout &sl)
        : split(SHARED ? blockIdx.x / sl.G : blockIdx.x), n_split(SHARED ? gridDim.x / sl.G : gridDim.x),
          b(SHARED ? blockIdx.z * sl.G + blockIdx.x % sl.G : blockIdx.z), pb(SHARED ? blockIdx.z : b),
          plen(SHARED ? (int)min(max(*sl.prefix_len, 0ll), (long long)sl.Tp) : 0), max_new(sl.max_new) {}

    // position j given this row's rows: `pre` = the dense cache's row b, or SHARED, the prefix row pb below plen and
    // `gen` = the generated row b after it
    template <typename P>
    __device__ __forceinline__ const P *at(const P *pre, long pre_ts, const P *gen, long gen_ts, int j) const {
        if constexpr (SHARED)
            return j < plen ? pre + (long)j * pre_ts : gen + (long)min(j - plen, max_new - 1) * gen_ts;
        else
            return pre + (long)j * pre_ts;
    }
    // position j of the whole (rows, T, ...) caches `pre` and `gen`
    template <typename P>
    __device__ __forceinline__ const P *at(const P *pre, long pre_bs, long pre_ts, const P *gen, long gen_bs, long gen_ts,
                                           int j) const {
        return at(pre + pb * pre_bs, pre_ts, gen + b * gen_bs, gen_ts, j);
    }
};

// The end of every decode kernel: each warp brings its running max m and sum l, and has left its accumulator in
// s_acc[warp * acc_ld + d], d < hd.  Thread = channel combines the warps into the CTA's partial; with one split that is
// the output row.  Otherwise the partial goes to the scratch `part`, and the last CTA of the (row, head) `bh` to take its
// ticket merges the (row, head)'s partials: the max M over the splits, then fmaf(exp(m_s - M), ., .) in split order, then
// num / den.  A fully masked row gives zeros.
template <typename T>
__device__ __forceinline__ void decode_epilogue(float m, float l, const float *s_acc, int acc_ld, int hd, float *part,
                                                unsigned *tickets, long bh, T *orow, int split, int n_split) {
    __shared__ float s_m[kDecWarps], s_l[kDecWarps];
    __shared__ int s_is_last;
    if ((threadIdx.x & 31) == 0) { s_m[threadIdx.x >> 5] = m; s_l[threadIdx.x >> 5] = l; }
    __syncthreads();
    float M = s_m[0];
#pragma unroll
    for (int w = 1; w < kDecWarps; ++w) M = fmaxf(M, s_m[w]);
    float den = 0.f;
    if (M != -INFINITY) {
#pragma unroll
        for (int w = 0; w < kDecWarps; ++w)
            if (s_m[w] != -INFINITY) den = fmaf(__expf(s_m[w] - M), s_l[w], den);
    }
    part += bh * n_split * (hd + 2);
    float *dst = part + (long)split * (hd + 2);
    for (int d = threadIdx.x; d < hd; d += blockDim.x) {
        float num = 0.f;
        if (M != -INFINITY) {
#pragma unroll
            for (int w = 0; w < kDecWarps; ++w)
                if (s_m[w] != -INFINITY) num = fmaf(__expf(s_m[w] - M), s_acc[w * acc_ld + d], num);
        }
        if (n_split == 1) orow[d] = from_op<T>(den > 0.f ? num / den : 0.f);
        else dst[d] = num;
    }
    if (n_split == 1) return;
    if (threadIdx.x == 0) { dst[hd] = M; dst[hd + 1] = den; }
    __threadfence();                                 // this thread's partial is visible device-wide ...
    __syncthreads();
    if (threadIdx.x == 0) s_is_last = atomicAdd(&tickets[bh], 1u) == (unsigned)(n_split - 1);   // ... before the ticket
    __syncthreads();
    if (!s_is_last) return;
    __threadfence();
    // the last CTA: L2 loads, the partials were written by other SMs
    float MM = -INFINITY;
    for (int s = 0; s < n_split; ++s) MM = fmaxf(MM, __ldcg(part + s * (hd + 2) + hd));
    float dd = 0.f;
    if (MM != -INFINITY)
#pragma unroll 4
        for (int s = 0; s < n_split; ++s) {
            const float ms = __ldcg(part + s * (hd + 2) + hd);
            if (ms != -INFINITY) dd = fmaf(__expf(ms - MM), __ldcg(part + s * (hd + 2) + hd + 1), dd);
        }
    for (int d = threadIdx.x; d < hd; d += blockDim.x) {
        float num = 0.f;
        if (MM != -INFINITY)
#pragma unroll 4
            for (int s = 0; s < n_split; ++s) {
                const float ms = __ldcg(part + s * (hd + 2) + hd);
                if (ms != -INFINITY) num = fmaf(__expf(ms - MM), __ldcg(part + s * (hd + 2) + d), num);
            }
        orow[d] = from_op<T>(dd > 0.f ? num / dd : 0.f);
    }
}

}  // namespace mmfs
