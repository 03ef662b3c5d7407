// attn_generic_sm100.cu -- bandwidth-oriented softmax(QK^T * scale + mask) V for the cases the
// tensor-core kernel (attn_fwd_sm100.cu) does not take: single-token decode over a KV cache
// (q_len = 1: a GEMV-shaped, HBM-bound problem -- no tensor cores needed) and small / odd shapes
// (head sizes other than 64/128, a few query rows).
//
// Semantics follow the reference's eager attention, LlamaAttention.forward
// (decoders/modeling_llama_mmfs.py:246-264): scores = (q * hd^-0.5) k^T + causal/padding mask,
// fp32 softmax, P V; and CLIPXAttention.forward (encoders/vit_adapter/xattn.py:47-141) when
// causal = 0 and no key mask.  Layout is the projection GEMMs' own (B, T, H, hd) -- no transposes.
// A query row whose keys are ALL masked (a left-padding position) returns zeros; the reference's
// finfo.min clamp makes such rows attend uniformly to every key, but those rows are padding and
// their outputs are never consumed (DESIGN.md, "Attention masks").
//
// One warp per (b, h, query row).  Keys are processed in chunks of 32*KPL: phase 1 gives every
// lane whole keys (row-contiguous 16-byte loads, q broadcast from shared memory), phase 2 gives
// every lane channels (coalesced V rows), online softmax across chunks.
#include "decode_common.cuh"
#include "sampler_common.cuh"   // MixFma (mixed-precision FMA)

namespace mmfs {

constexpr int kAttnChunk = 256;   // keys per chunk (8 per lane)
constexpr int kAttnWarps = 4;

// Prefix-shared segments (mmfs_attn_prefix_shared): k / v are the rows' own keys (Tkv = Tq), and row i walks the
// virtual key range j = 0 .. Tp + i - s, s = i / seg_len * seg_len: prefix key j below Tp (under `mask`), then own key
// s + j - Tp (under key_mask).  The other instantiations do not read `ps`, which comes last for that reason.
template <typename T>
struct PrefixSeg {
    const T *k, *v;                                   // (B, Tp, H, hd)
    long k_bs, k_ts, v_bs, v_ts;
    const uint8_t *mask;                              // (B, Tp) or null
    int Tp, seg_len;
};

template <typename T, bool PREFIX = false>
__global__ void __launch_bounds__(32 * kAttnWarps, PREFIX ? 8 : 0)   // PREFIX: 64 registers, no spills
attn_generic_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v, T *__restrict__ out,
                    const uint8_t *__restrict__ key_mask, long n_rows, int H, int Tq, int Tkv, int hd,
                    long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                    float scale, int causal, int past, PrefixSeg<T> ps) {
    extern __shared__ float s_dyn_f[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *s_q = s_dyn_f + warp * (hd + kAttnChunk);
    float *s_p = s_q + hd;
    const int cpl = (hd + 31) / 32;   // channels per lane (<= 8)

    for (long row = (long)blockIdx.x * kAttnWarps + warp; row < n_rows; row += (long)gridDim.x * kAttnWarps) {
        // PREFIX: 32-bit row arithmetic (the host keeps n_rows below 2^31), which spares the 64-bit division call
        const int i = PREFIX ? (int)row % Tq : (int)(row % Tq);
        const int h = PREFIX ? (int)row / Tq % H : (int)((row / Tq) % H);
        const int b = PREFIX ? (int)row / Tq / H : (int)(row / Tq / H);
        const T *qp = q + b * q_bs + i * q_ts + (long)h * hd;
        __syncwarp();
        for (int d = lane; d < hd; d += 32) s_q[d] = to_op(qp[d]) * scale;
        __syncwarp();
        int last_key = causal ? min(Tkv - 1, past + i) : Tkv - 1;
        int own0 = 0;                                 // PREFIX: own key of virtual key Tp
        if constexpr (PREFIX) {
            own0 = i / ps.seg_len * ps.seg_len - ps.Tp;
            last_key = i - own0;
        }
        float m_run = -INFINITY, l_run = 0.f;
        float acc[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] = 0.f;

        for (int j0 = 0; j0 <= last_key; j0 += kAttnChunk) {
            // phase 1: scores of up to kAttnChunk keys, lane owns keys j0 + lane + 32*t
            float cmax = -INFINITY;
            for (int t = 0; t < kAttnChunk / 32; ++t) {
                const int j = j0 + lane + 32 * t;
                float s = -INFINITY;
                if constexpr (PREFIX) {
                    const bool pre = j < ps.Tp;
                    if (j <= last_key && (pre ? (ps.mask == nullptr || ps.mask[(long)b * ps.Tp + j])
                                              : (key_mask == nullptr || key_mask[(long)b * Tkv + own0 + j]))) {
                        const T *kp = (pre ? ps.k + b * ps.k_bs + j * ps.k_ts : k + b * k_bs + (own0 + j) * k_ts) + (long)h * hd;
                        float dot = 0.f;
                        for (int d = 0; d < hd; ++d) dot += s_q[d] * to_op(kp[d]);
                        s = dot;
                    }
                } else if (j <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + j])) {
                    const T *kp = k + b * k_bs + j * k_ts + (long)h * hd;
                    float dot = 0.f;
                    for (int d = 0; d < hd; ++d) dot += s_q[d] * to_op(kp[d]);
                    s = dot;
                }
                s_p[lane + 32 * t] = s;
                cmax = fmaxf(cmax, s);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
            const float m_new = fmaxf(m_run, cmax);
            if (m_new == -INFINITY) { __syncwarp(); continue; }       // nothing visible yet
            const float corr = __expf(m_run - m_new);                 // m_run = -inf -> 0
            float csum = 0.f;
            for (int t = 0; t < kAttnChunk / 32; ++t) {
                const float p = __expf(s_p[lane + 32 * t] - m_new);   // masked (-inf) -> 0
                s_p[lane + 32 * t] = p;
                csum += p;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) csum += __shfl_xor_sync(0xffffffffu, csum, o);
            l_run = l_run * corr + csum;
            m_run = m_new;
            __syncwarp();
            // phase 2: acc[c] += p_j * v[j][channel], lane owns channels lane + 32*c
#pragma unroll
            for (int c = 0; c < 8; ++c) acc[c] *= corr;
            const int jn = min(kAttnChunk, last_key - j0 + 1);
            for (int jj = 0; jj < jn; ++jj) {
                const float p = s_p[jj];
                if (p == 0.f) continue;                                // warp-uniform (same smem word)
                const T *vp = v + b * v_bs + (long)(j0 + jj) * v_ts + (long)h * hd;
                if constexpr (PREFIX)
                    vp = j0 + jj < ps.Tp ? ps.v + b * ps.v_bs + (long)(j0 + jj) * ps.v_ts + (long)h * hd
                                         : v + b * v_bs + (long)(own0 + j0 + jj) * v_ts + (long)h * hd;
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < cpl && lane + 32 * c < hd) acc[c] += p * to_op(vp[lane + 32 * c]);
            }
            __syncwarp();
        }
        T *op = out + b * o_bs + i * o_ts + (long)h * hd;
        const float inv = l_run > 0.f ? 1.f / l_run : 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            if (c < cpl && lane + 32 * c < hd) op[lane + 32 * c] = from_op<T>(acc[c] * inv);
    }
}

// ------------------------------------------------------------------------------------------------------------
// Decode (q_len = 1 over a KV cache): split-KV ("flash decoding") on the skeleton of decode_common.cuh.  The
// row-per-warp kernel above gives a decode step B*H = 160 warps for the whole GPU, each walking 2k keys serially with
// scalar loads.  Here every CTA reduces 256 keys of one (b, h) -- lane = key for the scores (16-byte loads along the
// key row, q broadcast from shared memory), lane = channels for P V (coalesced V rows) -- and the last CTA of the
// (b, h) merges the partials.  HBM-bound: K and V are read exactly once.  The SHARED instantiations
// (mmfs_attn_decode_shared, the graphed beam search) read k / v as the (P, Tp, H, hd) prefix and `gen` as the
// (R, max_new, H, hd) generated rows.
// ------------------------------------------------------------------------------------------------------------
template <typename T>
struct Kv16 {                                         // a (rows, T, H, hd) K / V pair
    const T *k, *v;
    long k_bs, k_ts, v_bs, v_ts;
};

// A warp's 64 keys in two passes of 32; the CTA writes its (acc[hd], m, l) partial and attn_decode_merge_kernel merges
// them.  (Merging in the last CTA, as the other decode kernels do, costs this kernel registers and occupancy.)
template <typename T, bool SHARED = false>
__global__ void __launch_bounds__(32 * kDecWarps)
attn_decode_split_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v,
                         const uint8_t *__restrict__ key_mask, float *__restrict__ part, int H, int Tkv, int hd,
                         long q_bs, long k_bs, long k_ts, long v_bs, long v_ts, float scale, int last_key, Kv16<T> gen,
                         SharedLayout sl) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dec[];                  // q[hd] | per-warp partials [kDecWarps][hd + 2]
    float *s_q = s_dec, *s_red = s_dec + hd;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, h = blockIdx.y;
    const DecodeCta<SHARED> cta(sl);
    const int b = cta.b;
    const int cpl = hd / 32;                          // channels per lane in the P V phase (host: hd % 32 == 0, <= 8)
    const T *qp = q + b * q_bs + (long)h * hd;
    for (int d = threadIdx.x; d < hd; d += blockDim.x) s_q[d] = to_op(qp[d]) * scale;
    __syncthreads();

    float m_run = -INFINITY, l_run = 0.f;
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    const int kbase = cta.split * kDecKeys + warp * kDecKPW;
#pragma unroll 1
    for (int it = 0; it < kDecKPW / 32; ++it) {
        const int j0 = kbase + it * 32;
        if (j0 > last_key) break;                     // warp-uniform
        const int j = j0 + lane;
        float sc = -INFINITY;
        if (j <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + j])) {
            const T *kp = cta.at(k + (long)h * hd, k_bs, k_ts, gen.k + (long)h * hd, gen.k_bs, gen.k_ts, j);
            float dot = 0.f;
            for (int d0 = 0; d0 < hd; d0 += VEC) {
                float f[VEC];
                Vec16<T>::unpack(ldg_nc_v4(kp + d0), f);
#pragma unroll
                for (int e = 0; e < VEC; e += 4) {
                    const float4 qq = *reinterpret_cast<const float4 *>(s_q + d0 + e);
                    dot = fmaf(f[e], qq.x, dot); dot = fmaf(f[e + 1], qq.y, dot);
                    dot = fmaf(f[e + 2], qq.z, dot); dot = fmaf(f[e + 3], qq.w, dot);
                }
            }
            sc = dot;
        }
        float cmax = sc;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
        const float m_new = fmaxf(m_run, cmax);
        if (m_new == -INFINITY) continue;             // nothing visible in this pass (warp-uniform)
        const float corr = __expf(m_run - m_new);     // m_run = -inf -> 0
        const float pj = __expf(sc - m_new);          // masked (-inf) -> 0
        float psum = pj;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) psum += __shfl_xor_sync(0xffffffffu, psum, o);
        l_run = l_run * corr + psum;
        m_run = m_new;
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] *= corr;
        for (int jj = 0; jj < 32; ++jj) {
            const float pw = __shfl_sync(0xffffffffu, pj, jj);
            if (pw == 0.f) continue;                  // warp-uniform
            const T *vp = cta.at(v + (long)h * hd + lane * cpl, v_bs, v_ts, gen.v + (long)h * hd + lane * cpl, gen.v_bs,
                                 gen.v_ts, j0 + jj);
            bool done = false;
            if constexpr (sizeof(T) == 2) {
                if (cpl == 4) {                        // hd = 128, 16-bit: one 8-byte load per lane, 256 B per warp
                    const uint2 raw = *reinterpret_cast<const uint2 *>(vp);
                    float f[8];
                    Vec16<T>::unpack(make_uint4(raw.x, raw.y, 0u, 0u), f);
#pragma unroll
                    for (int c = 0; c < 4; ++c) acc[c] = fmaf(pw, f[c], acc[c]);
                    done = true;
                } else if (cpl == 2) {                 // hd = 64
                    const uint32_t raw = *reinterpret_cast<const uint32_t *>(vp);
                    float f[8];
                    Vec16<T>::unpack(make_uint4(raw, 0u, 0u, 0u), f);
                    acc[0] = fmaf(pw, f[0], acc[0]); acc[1] = fmaf(pw, f[1], acc[1]);
                    done = true;
                }
            }
            if (!done) {
#pragma unroll
                for (int c = 0; c < 8; ++c)
                    if (c < cpl) acc[c] = fmaf(pw, to_op(vp[c]), acc[c]);
            }
        }
    }
    // merge the four warps of the CTA
    float *mine = s_red + warp * (hd + 2);
    if (lane == 0) { mine[hd] = m_run; mine[hd + 1] = l_run; }
#pragma unroll
    for (int c = 0; c < 8; ++c)
        if (c < cpl) mine[lane * cpl + c] = acc[c];
    __syncthreads();
    float m_all = -INFINITY;
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) m_all = fmaxf(m_all, s_red[w * (hd + 2) + hd]);
    float *dst = part + (((long)b * H + h) * cta.n_split + cta.split) * (hd + 2);
    for (int d = threadIdx.x; d < hd + 2; d += blockDim.x) {
        float r = 0.f;
        if (d == hd) r = m_all;
        else if (m_all != -INFINITY) {
#pragma unroll
            for (int w = 0; w < kDecWarps; ++w) {
                const float mw = s_red[w * (hd + 2) + hd];
                if (mw != -INFINITY) r += __expf(mw - m_all) * s_red[w * (hd + 2) + (d < hd ? d : hd + 1)];
            }
        }
        dst[d] = r;                                   // d < hd: acc; d == hd: m; d == hd + 1: l
    }
}

// hd = 128, 16-bit elements (the Llama decode step): every load is a fully used 16-byte vector.
//   Q K^T : 8 lanes per key (2 x LDG.128 each = the key's 256 bytes), 4 keys per warp step; the products are mixed-precision FMA
//           (16-bit k x 16-bit q + fp32 accumulator, exact products, no unpack), the scale is applied to the fp32 dot;
//   P V   : 16 lanes per key (LDG.128 = 8 channels each), 2 keys per warp step.
// Loads are issued in explicit BATCHES of eight 16-byte vectors per lane (4 KB per warp), double-buffered in registers,
// with the key-validity bits balloted once per warp up front: the first version of this kernel tested the mask byte,
// branched and loaded key by key, which left two loads in flight per warp (SASS: LDG.U8 -> BRA -> 2 x LDG.128 -> SHFL per
// key).  A masked key inside the range is still loaded (clamped address)
// and discarded.
// A warp reduces 64 keys in one pass (no running rescale).
template <typename T>
__device__ __forceinline__ float dot16_mixed(const uint4 &ka, const uint4 &kb, const uint4 &qa, const uint4 &qb) {
    float d0 = 0.f, d1 = 0.f;
    const uint32_t kw[8] = {ka.x, ka.y, ka.z, ka.w, kb.x, kb.y, kb.z, kb.w};
    const uint32_t qw[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        MixFma<T>::fma(d0, (uint16_t)(kw[i] & 0xffffu), (uint16_t)(qw[i] & 0xffffu));
        MixFma<T>::fma(d1, (uint16_t)(kw[i] >> 16), (uint16_t)(qw[i] >> 16));
    }
    return d0 + d1;
}

// SHARED: 4 CTAs per SM (128 registers), which holds the generated rows' pointers without spilling
template <typename T, bool SHARED = false>
__global__ void __launch_bounds__(32 * kDecWarps, SHARED ? 4 : 5)
attn_decode_split128_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v,
                            const uint8_t *__restrict__ key_mask, float *__restrict__ part, unsigned *__restrict__ tickets,
                            T *__restrict__ out, int H, int Tkv, long q_bs, long k_bs, long k_ts, long v_bs, long v_ts,
                            long o_bs, float scale, int last_key, Kv16<T> gen, SharedLayout sl) {
    constexpr int WARPS = kDecWarps, HD = 128, KPW = kDecKPW;
    static_assert(KPW == 64, "the pipeline below walks a warp's keys in four batches of 16");
    __shared__ float s_p[WARPS][KPW];
    __shared__ __align__(16) float s_acc[WARPS][HD];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, h = blockIdx.y;
    const DecodeCta<SHARED> cta(sl);
    const int b = cta.b;
    const int k0 = cta.split * kDecKeys + warp * KPW;
    const int half = lane >> 4, ch = (lane & 15) * 8;
    float m = -INFINITY, l = 0.f;
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;

    unsigned ok_lo = 0u, ok_hi = 0u;                              // validity of keys k0 + 0..31 / k0 + 32..63
    if (k0 <= last_key) {                                         // warp-uniform
        const int ja = k0 + lane, jb = ja + 32;
        const bool oa = ja <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + ja]);
        const bool ob = jb <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + jb]);
        ok_lo = __ballot_sync(0xffffffffu, oa);
        ok_hi = __ballot_sync(0xffffffffu, ob);
    }
    if (ok_lo | ok_hi) {                                          // warp-uniform: at least one visible key
        const int sub = lane & 7, grp = lane >> 3;
        const T *qp = q + b * q_bs + (long)h * HD + sub * 16;    // this lane's 16 channels of q, kept packed
        const uint4 qa = ldg_nc_v4(qp), qb = ldg_nc_v4(qp + 8);
        // Software pipeline over eight batches (K0..K3, V0..V3) with two register buffers: the loads of batch i+1 are
        // issued BEFORE the arithmetic of batch i, and V0 is requested before the softmax reductions (V does not depend
        // on P), so every warp keeps one 4 KB batch in flight from its first instruction to its last.  (Without this
        // a warp has nothing in flight while it computes.)
        auto load_k = [&](uint4 (&r)[8], int bt) {
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const T *kp = cta.at(k + cta.pb * k_bs + (long)h * HD + sub * 16, k_ts, gen.k + b * gen.k_bs + (long)h * HD + sub * 16,
                                     gen.k_ts, min(k0 + bt * 16 + s * 4 + grp, last_key));
                r[2 * s] = ldg_nc_v4(kp);
                r[2 * s + 1] = ldg_nc_v4(kp + 8);
            }
        };
        auto load_v = [&](uint4 (&r)[8], int bt) {
#pragma unroll
            for (int s = 0; s < 8; ++s)
                r[s] = ldg_nc_v4(cta.at(v + cta.pb * v_bs + (long)h * HD + ch, v_ts, gen.v + b * gen.v_bs + (long)h * HD + ch,
                                        gen.v_ts, min(k0 + bt * 16 + s * 2 + half, last_key)));
        };
        auto scores = [&](const uint4 (&r)[8], int bt) {          // 4 steps of 4 keys
            const unsigned okw = (bt < 2 ? ok_lo : ok_hi) >> ((bt & 1) * 16);
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                float dot = dot16_mixed<T>(r[2 * s], r[2 * s + 1], qa, qb);
                dot += __shfl_xor_sync(0xffffffffu, dot, 1);
                dot += __shfl_xor_sync(0xffffffffu, dot, 2);
                dot += __shfl_xor_sync(0xffffffffu, dot, 4);
                const bool ok = (okw >> (s * 4 + grp)) & 1u;
                if (sub == 0) s_p[warp][bt * 16 + s * 4 + grp] = ok ? dot * scale : -INFINITY;
            }
        };
        auto pv = [&](const uint4 (&r)[8], int bt) {              // 8 steps of 2 keys, 16 lanes x 8 channels per key
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                const float pw = s_p[warp][bt * 16 + s * 2 + half];
                if (pw != 0.f) {                                  // a masked slot may hold anything (0 x NaN)
                    float f[8];
                    Vec16<T>::unpack(r[s], f);
#pragma unroll
                    for (int c = 0; c < 8; ++c) acc[c] = fmaf(pw, f[c], acc[c]);
                }
            }
        };
        uint4 ra[8], rb[8];
        load_k(ra, 0);
        load_k(rb, 1); scores(ra, 0);
        load_k(ra, 2); scores(rb, 1);
        load_k(rb, 3); scores(ra, 2);
        load_v(ra, 0); scores(rb, 3);
        __syncwarp();
        // ---- softmax over the warp's keys ----------------------------------------------------------------------
        const float s0 = s_p[warp][lane], s1 = s_p[warp][lane + 32];
        m = fmaxf(s0, s1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        const float p0 = __expf(s0 - m), p1 = __expf(s1 - m);   // masked (-inf) -> 0; m is finite here
        l = p0 + p1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
        __syncwarp();
        s_p[warp][lane] = p0;
        s_p[warp][lane + 32] = p1;
        __syncwarp();
        // ---- P V ---------------------------------------------------------------------------------------------
        load_v(rb, 1); pv(ra, 0);
        load_v(ra, 2); pv(rb, 1);
        load_v(rb, 3); pv(ra, 2);
        pv(rb, 3);
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 16);
    }
    if (lane < 16) {
        *reinterpret_cast<float4 *>(&s_acc[warp][ch]) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4 *>(&s_acc[warp][ch + 4]) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    decode_epilogue<T>(m, l, &s_acc[0][0], HD, HD, part, tickets, (long)b * H + h, out + b * o_bs + (long)h * HD,
                       cta.split, cta.n_split);
}

// (Alternative not taken: staging a warp's whole 64-key K and V tiles in shared memory with cp.async -- 32 KB per warp
// requested up front, 6 warps per SM -- leaves so few warps that the score / softmax / P V arithmetic out of shared
// memory is latency-exposed.)
template <typename T>
__global__ void attn_decode_merge_kernel(const float *__restrict__ part, T *__restrict__ out, int H, int hd, int n_split,
                                         long o_bs) {
    const int h = blockIdx.x, b = blockIdx.y;
    const float *p0 = part + (((long)b * H + h) * n_split) * (hd + 2);
    float m = -INFINITY;
    for (int s = 0; s < n_split; ++s) m = fmaxf(m, p0[s * (hd + 2) + hd]);
    for (int d = threadIdx.x; d < hd; d += blockDim.x) {
        float num = 0.f, den = 0.f;
        if (m != -INFINITY)
            for (int s = 0; s < n_split; ++s) {
                const float ms = p0[s * (hd + 2) + hd];
                if (ms == -INFINITY) continue;
                const float w = __expf(ms - m);
                num = fmaf(w, p0[s * (hd + 2) + d], num);
                den = fmaf(w, p0[s * (hd + 2) + hd + 1], den);
            }
        out[b * o_bs + (long)h * hd + d] = from_op<T>(den > 0.f ? num / den : 0.f);   // fully masked row -> zeros
    }
}

// B query rows; SHARED: B = P * sl.G rows, k / v the prefix and gen the generated rows
template <typename T, bool SHARED = false>
static int launch_attn_decode(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask, float *scratch,
                              int B, int H, int Tkv, int hd, long q_bs, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs,
                              float scale, int last_key, cudaStream_t st, const Kv16<T> &gen = {},
                              const SharedLayout &sl = {}) {
    const dim3 grid = decode_grid(last_key, B, H, sl);
    if constexpr (sizeof(T) == 2) {
        if (hd == 128 && ((uintptr_t)q % 16 == 0) && (q_bs % 8 == 0) && ((uintptr_t)scratch % 16 == 0)) {
            unsigned *tickets = reinterpret_cast<unsigned *>(scratch);
            if (decode_splits(last_key) > 1) MMFS_CUDA(cudaMemsetAsync(tickets, 0, sizeof(unsigned) * (size_t)B * H, st));
            attn_decode_split128_kernel<T, SHARED><<<grid, 32 * kDecWarps, 0, st>>>(
                (const T *)q, (const T *)k, (const T *)v, key_mask, scratch + decode_ticket_floats(B, H), tickets, (T *)out, H,
                Tkv, q_bs, k_bs, k_ts, v_bs, v_ts, o_bs, scale, last_key, gen, sl);
            MMFS_CUDA(cudaGetLastError());
            return MMFS_OK;
        }
    }
    const size_t smem = (size_t)(hd + kDecWarps * (hd + 2)) * sizeof(float);
    attn_decode_split_kernel<T, SHARED><<<grid, 32 * kDecWarps, smem, st>>>((const T *)q, (const T *)k, (const T *)v, key_mask,
                                                                           scratch, H, Tkv, hd, q_bs, k_bs, k_ts, v_bs, v_ts,
                                                                           scale, last_key, gen, sl);
    attn_decode_merge_kernel<T><<<dim3(H, B), hd < 128 ? 64 : 128, 0, st>>>(scratch, (T *)out, H, hd, decode_splits(last_key),
                                                                            o_bs);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_attn_generic(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                               int B, int H, int Tq, int Tkv, int hd, long q_bs, long q_ts, long k_bs, long k_ts,
                               long v_bs, long v_ts, long o_bs, long o_ts, float scale, int causal, int past, cudaStream_t st) {
    const long n_rows = (long)B * H * Tq;
    const int grid = capped_grid((n_rows + kAttnWarps - 1) / kAttnWarps, 16);
    const size_t smem = (size_t)kAttnWarps * (hd + kAttnChunk) * sizeof(float);
    attn_generic_kernel<T><<<grid, 32 * kAttnWarps, smem, st>>>((const T *)q, (const T *)k, (const T *)v, (T *)out, key_mask,
                                                              n_rows, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts,
                                                              o_bs, o_ts, scale, causal, past, PrefixSeg<T>{});
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

// mmfs_attn_prefix_shared's fallback (arguments checked there): the generic kernel's PREFIX instantiation
int attn_prefix_generic(const void *q, const void *k, const void *v, const void *k_prefix, const void *v_prefix, void *out,
                        const uint8_t *prefix_mask, const uint8_t *key_mask, int B, int H, int Tq, int Tp, int seg_len,
                        int hd, long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long kp_bs, long kp_ts,
                        long vp_bs, long vp_ts, long o_bs, long o_ts, float scale, int dtype, cudaStream_t st) {
    const long n_rows = (long)B * H * Tq;
    if (n_rows >= (1L << 31)) { set_error("attn_prefix_shared: %ld query rows", n_rows); return MMFS_EUNSUPPORTED; }
    return dispatch_dtype<kF32Types>(dtype, "attn_prefix_shared", [&](auto tag) {
        using T = typename decltype(tag)::type;
        const int grid = capped_grid((n_rows + kAttnWarps - 1) / kAttnWarps, 16);
        const size_t smem = (size_t)kAttnWarps * (hd + kAttnChunk) * sizeof(float);
        const PrefixSeg<T> ps{(const T *)k_prefix, (const T *)v_prefix, kp_bs, kp_ts, vp_bs, vp_ts, prefix_mask, Tp, seg_len};
        attn_generic_kernel<T, true><<<grid, 32 * kAttnWarps, smem, st>>>(
            (const T *)q, (const T *)k, (const T *)v, (T *)out, key_mask, n_rows, H, Tq, Tq, hd, q_bs, q_ts, k_bs, k_ts, v_bs,
            v_ts, o_bs, o_ts, scale, 0, 0, ps);
        MMFS_CUDA(cudaGetLastError());
        return MMFS_OK;
    });
}

}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_attn_generic(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                                 int B, int H, int Tq, int Tkv, int hd,
                                 long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                                 float scale, int causal, int past, int dtype, void *stream) {
    MMFS_CHECK_ARG(B >= 0 && H > 0 && Tq >= 0 && Tkv > 0 && hd > 0 && hd <= 256, "attn_generic: bad shape (hd <= 256)");
    if (B == 0 || Tq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && out, "attn_generic: null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kF32Types>(dtype, "attn_generic", [&](auto tag) {
        return launch_attn_generic<typename decltype(tag)::type>(q, k, v, out, key_mask, B, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts,
                                                                 v_bs, v_ts, o_bs, o_ts, scale, causal, past, st);
    });
}

extern "C" long mmfs_attn_decode_scratch_floats(int B, int H, int Tkv, int hd) {
    return decode_ticket_floats(B, H) + (long)B * H * decode_splits(Tkv - 1) * (hd + 2);
}

extern "C" int mmfs_attn_decode(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask, float *scratch,
                                int B, int H, int Tkv, int hd, long q_bs, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs,
                                float scale, int causal, int past, int dtype, void *stream) {
    MMFS_CHECK_ARG(B >= 0 && H > 0 && Tkv > 0 && hd > 0, "attn_decode: bad shape");
    if (B == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && out && scratch, "attn_decode: null pointer argument");
    const size_t es = dtype_size(dtype);
    if (dtype == MMFS_F64 || es == 0 || hd % 32 != 0 || hd > 256 || B > 65535 || H > 65535 ||
        ((uintptr_t)k | (uintptr_t)v) % 16 != 0 || (k_bs * es) % 16 != 0 || (k_ts * es) % 16 != 0 ||
        (v_bs * es) % 16 != 0 || (v_ts * es) % 16 != 0 || (hd * es) % 16 != 0) {
        set_error("attn_decode: needs f32/f16/bf16, hd %% 32 == 0 (<= 256), 16-byte aligned K / V rows");
        return MMFS_EUNSUPPORTED;
    }
    const int last_key = decode_last_key(causal, past, Tkv);
    MMFS_CHECK_ARG(last_key >= 0, "attn_decode: negative past");
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kF32Types>(dtype, "attn_decode", [&](auto tag) {
        return launch_attn_decode<typename decltype(tag)::type>(q, k, v, out, key_mask, scratch, B, H, Tkv, hd, q_bs, k_bs, k_ts,
                                                                v_bs, v_ts, o_bs, scale, last_key, st);
    });
}

extern "C" int mmfs_attn_decode_shared(const void *q, const void *k_prefix, const void *v_prefix, const void *k_gen,
                                       const void *v_gen, void *out, const uint8_t *key_mask, const long long *prefix_len,
                                       float *scratch, int R, int G, int H, int Tkv, int Tp, int max_new, int hd, long q_bs,
                                       long kp_bs, long kp_ts, long vp_bs, long vp_ts, long kg_bs, long kg_ts, long vg_bs,
                                       long vg_ts, long o_bs, float scale, int causal, int past, int dtype, void *stream) {
    MMFS_CHECK_ARG(R >= 0 && G > 0 && H > 0 && Tkv > 0 && Tp > 0 && hd > 0, "attn_decode_shared: bad shape");
    MMFS_CHECK_ARG(R % G == 0, "attn_decode_shared: R = %d rows are not whole groups of G = %d", R, G);
    MMFS_CHECK_ARG(max_new >= 1, "attn_decode_shared: max_new must be >= 1");
    if (R == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k_prefix && v_prefix && k_gen && v_gen && out && prefix_len && scratch,
                   "attn_decode_shared: null pointer argument");
    const size_t es = dtype_size(dtype);
    const long strides[8] = {kp_bs, kp_ts, vp_bs, vp_ts, kg_bs, kg_ts, vg_bs, vg_ts};
    bool aligned = (((uintptr_t)k_prefix | (uintptr_t)v_prefix | (uintptr_t)k_gen | (uintptr_t)v_gen) % 16 == 0);
    for (long s : strides) aligned = aligned && (s * (long)es) % 16 == 0;
    if (dtype == MMFS_F64 || es == 0 || hd % 32 != 0 || hd > 256 || R / G > 65535 || H > 65535 || !aligned ||
        (hd * es) % 16 != 0) {
        set_error("attn_decode_shared: needs f32/f16/bf16, hd %% 32 == 0 (<= 256), 16-byte aligned prefix / gen rows, R / G <= 65535");
        return MMFS_EUNSUPPORTED;
    }
    const int last_key = decode_last_key(causal, past, Tkv);
    MMFS_CHECK_ARG(last_key >= 0, "attn_decode_shared: negative past");
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kF32Types>(dtype, "attn_decode_shared", [&](auto tag) {
        using T = typename decltype(tag)::type;
        return launch_attn_decode<T, true>(q, k_prefix, v_prefix, out, key_mask, scratch, R, H, Tkv, hd, q_bs, kp_bs, kp_ts,
                                           vp_bs, vp_ts, o_bs, scale, last_key, st,
                                           Kv16<T>{(const T *)k_gen, (const T *)v_gen, kg_bs, kg_ts, vg_bs, vg_ts},
                                           SharedLayout{prefix_len, G, Tp, max_new});
    });
}
