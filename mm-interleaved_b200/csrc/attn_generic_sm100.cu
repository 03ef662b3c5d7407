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
#include "common.cuh"
#include "sampler_common.cuh"   // MixFma (mixed-precision FMA)

namespace mmfs {

constexpr int kAttnChunk = 256;   // keys per chunk (8 per lane)
constexpr int kAttnWarps = 4;

template <typename T>
__global__ void __launch_bounds__(32 * kAttnWarps)
attn_generic_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v, T *__restrict__ out,
                    const uint8_t *__restrict__ key_mask, long n_rows, int H, int Tq, int Tkv, int hd,
                    long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                    float scale, int causal, int past) {
    extern __shared__ float s_dyn_f[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *s_q = s_dyn_f + warp * (hd + kAttnChunk);
    float *s_p = s_q + hd;
    const int cpl = (hd + 31) / 32;   // channels per lane (<= 8)

    for (long row = (long)blockIdx.x * kAttnWarps + warp; row < n_rows; row += (long)gridDim.x * kAttnWarps) {
        const int i = (int)(row % Tq);
        const int h = (int)((row / Tq) % H);
        const int b = (int)(row / Tq / H);
        const T *qp = q + b * q_bs + i * q_ts + (long)h * hd;
        __syncwarp();
        for (int d = lane; d < hd; d += 32) s_q[d] = to_op(qp[d]) * scale;
        __syncwarp();
        const int last_key = causal ? min(Tkv - 1, past + i) : Tkv - 1;
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
                if (j <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + j])) {
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
// Decode (q_len = 1 over a KV cache): split-KV ("flash decoding").  The row-per-warp kernel above gives a decode step
// B*H = 160 warps for the whole GPU, each walking 2k keys serially with scalar loads.  Here grid = (ceil(Tkv / 256), H, B): every CTA reduces 256 keys of one (b, h) -- lane = key for the
// scores (16-byte loads along the key row, q broadcast from shared memory), lane = channels for P V (coalesced V
// rows) -- and writes an (m, l, acc[hd]) partial; a second kernel merges the partials.  HBM-bound: K and V are read
// exactly once.
// ------------------------------------------------------------------------------------------------------------
constexpr int kDecKeys = 256;     // keys per CTA
constexpr int kDecWarps = 4;      // 64 keys per warp, two passes of 32

template <typename T>
__global__ void __launch_bounds__(32 * kDecWarps)
attn_decode_split_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v,
                         const uint8_t *__restrict__ key_mask, float *__restrict__ part, int H, int Tkv, int hd,
                         long q_bs, long k_bs, long k_ts, long v_bs, long v_ts, float scale, int last_key) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dec[];                  // q[hd] | per-warp partials [kDecWarps][hd + 2]
    float *s_q = s_dec, *s_red = s_dec + hd;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z, n_split = gridDim.x;
    const int cpl = hd / 32;                          // channels per lane in the P V phase (host: hd % 32 == 0, <= 8)
    const T *qp = q + b * q_bs + (long)h * hd;
    for (int d = threadIdx.x; d < hd; d += blockDim.x) s_q[d] = to_op(qp[d]) * scale;
    __syncthreads();

    float m_run = -INFINITY, l_run = 0.f;
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;
    const int kbase = split * kDecKeys + warp * (kDecKeys / kDecWarps);
#pragma unroll 1
    for (int it = 0; it < kDecKeys / kDecWarps / 32; ++it) {
        const int j0 = kbase + it * 32;
        if (j0 > last_key) break;                     // warp-uniform
        const int j = j0 + lane;
        float sc = -INFINITY;
        if (j <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + j])) {
            const T *kp = k + b * k_bs + (long)j * k_ts + (long)h * hd;
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
        const T *vb = v + b * v_bs + (long)h * hd + lane * cpl;
        for (int jj = 0; jj < 32; ++jj) {
            const float pw = __shfl_sync(0xffffffffu, pj, jj);
            if (pw == 0.f) continue;                  // warp-uniform
            const T *vp = vb + (long)(j0 + jj) * v_ts;
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
    float *dst = part + (((long)b * H + h) * n_split + split) * (hd + 2);
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
// A warp reduces 64 keys in one pass (no running rescale); the CTA's four warps are combined in shared memory into one
// (m, l, acc[128]) partial, and the LAST CTA of a (b, h) to arrive (a ticket per (b, h) in the scratch buffer, zeroed by
// the launcher) merges the n_split partials and writes the output row -- no second kernel.
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

template <typename T, int WARPS>
__global__ void __launch_bounds__(32 * WARPS, WARPS == 4 ? 5 : 2)
attn_decode_split128_kernel(const T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v,
                            const uint8_t *__restrict__ key_mask, float *__restrict__ part, unsigned *__restrict__ tickets,
                            T *__restrict__ out, int H, int Tkv, long q_bs, long k_bs, long k_ts, long v_bs, long v_ts,
                            long o_bs, float scale, int last_key) {
    constexpr int HD = 128, KPW = kDecKeys / WARPS, NB = KPW / 16;   // 64 (4 warps) or 32 (8 warps) keys per warp
    static_assert((WARPS == 4 || WARPS == 8) && 32 * WARPS >= HD, "one thread per channel in the combine / merge steps");
    __shared__ float s_p[WARPS][KPW];
    __shared__ __align__(16) float s_acc[WARPS][HD];
    __shared__ float s_m[WARPS], s_l[WARPS];
    __shared__ int s_is_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z, n_split = gridDim.x;
    const int k0 = split * kDecKeys + warp * KPW;
    const int half = lane >> 4, ch = (lane & 15) * 8;
    float m = -INFINITY, l = 0.f;
    float acc[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) acc[c] = 0.f;

    unsigned ok_lo = 0u, ok_hi = 0u;                              // validity of keys k0 + 0..31 / k0 + 32..63
    if (k0 <= last_key) {                                         // warp-uniform
        const int ja = k0 + lane, jb = ja + 32;
        const bool oa = ja <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + ja]);
        const bool ob = KPW == 64 && jb <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + jb]);
        ok_lo = __ballot_sync(0xffffffffu, oa);
        ok_hi = __ballot_sync(0xffffffffu, ob);
    }
    if (ok_lo | ok_hi) {                                          // warp-uniform: at least one visible key
        const int sub = lane & 7, grp = lane >> 3;
        const T *qp = q + b * q_bs + (long)h * HD + sub * 16;    // this lane's 16 channels of q, kept packed
        const uint4 qa = ldg_nc_v4(qp), qb = ldg_nc_v4(qp + 8);
        const T *kb = k + b * k_bs + (long)h * HD + sub * 16;
        // Software pipeline over eight batches (K0..K3, V0..V3) with two register buffers: the loads of batch i+1 are
        // issued BEFORE the arithmetic of batch i, and V0 is requested before the softmax reductions (V does not depend
        // on P), so every warp keeps one 4 KB batch in flight from its first instruction to its last.  (Without this
        // a warp has nothing in flight while it computes.)
        const T *vb = v + b * v_bs + (long)h * HD + ch;
        auto load_k = [&](uint4 (&r)[8], int bt) {
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                const T *kp = kb + (long)min(k0 + bt * 16 + s * 4 + grp, last_key) * k_ts;
                r[2 * s] = ldg_nc_v4(kp);
                r[2 * s + 1] = ldg_nc_v4(kp + 8);
            }
        };
        auto load_v = [&](uint4 (&r)[8], int bt) {
#pragma unroll
            for (int s = 0; s < 8; ++s) r[s] = ldg_nc_v4(vb + (long)min(k0 + bt * 16 + s * 2 + half, last_key) * v_ts);
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
        if constexpr (NB == 4) {
            load_k(ra, 2); scores(rb, 1);
            load_k(rb, 3); scores(ra, 2);
            load_v(ra, 0); scores(rb, 3);
        } else {
            load_v(ra, 0); scores(rb, 1);
        }
        __syncwarp();
        // ---- softmax over the warp's keys ----------------------------------------------------------------------
        const float s0 = s_p[warp][lane], s1 = KPW == 64 ? s_p[warp][(lane + 32) % KPW] : -INFINITY;
        m = fmaxf(s0, s1);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        const float p0 = __expf(s0 - m), p1 = __expf(s1 - m);   // masked (-inf) -> 0; m is finite here
        l = p0 + p1;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
        __syncwarp();
        s_p[warp][lane] = p0;
        if constexpr (KPW == 64) s_p[warp][lane + 32] = p1;
        __syncwarp();
        // ---- P V ---------------------------------------------------------------------------------------------
        load_v(rb, 1); pv(ra, 0);
        if constexpr (NB == 4) {
            load_v(ra, 2); pv(rb, 1);
            load_v(rb, 3); pv(ra, 2);
            pv(rb, 3);
        } else {
            pv(rb, 1);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], 16);
    }
    if (lane < 16) {
        *reinterpret_cast<float4 *>(&s_acc[warp][ch]) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4 *>(&s_acc[warp][ch + 4]) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    }
    if (lane == 0) { s_m[warp] = m; s_l[warp] = l; }
    __syncthreads();
    // ---- the CTA's partial: thread = channel (threads past HD only take part in the barriers) ----------------------
    const int d = threadIdx.x;
    const bool chan = d < HD;
    float M = s_m[0];
#pragma unroll
    for (int w = 1; w < WARPS; ++w) M = fmaxf(M, s_m[w]);
    float num = 0.f, den = 0.f;
    if (M != -INFINITY && chan) {
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            if (s_m[w] == -INFINITY) continue;
            const float e = __expf(s_m[w] - M);
            num = fmaf(e, s_acc[w][d], num);
            den = fmaf(e, s_l[w], den);
        }
    }
    T *orow = out + b * o_bs + (long)h * HD;
    if (n_split == 1) {                                           // nothing to merge with
        if (chan) orow[d] = from_op<T>(den > 0.f ? num / den : 0.f);
        return;
    }
    float *dst = part + (((long)b * H + h) * n_split + split) * (HD + 2);
    if (chan) dst[d] = num;
    if (d == 0) { dst[HD] = M; dst[HD + 1] = den; }
    __threadfence();                                              // this thread's partial is visible device-wide ...
    __syncthreads();
    if (d == 0) s_is_last = atomicAdd(&tickets[b * H + h], 1u) == (unsigned)(n_split - 1);   // ... before the ticket
    __syncthreads();
    if (!s_is_last || !chan) return;
    __threadfence();
    // ---- last CTA of this (b, h): merge (L2 loads: the partials were written by other SMs) ---------------------
    const float *p0 = part + ((long)b * H + h) * n_split * (HD + 2);
    float MM = -INFINITY;
    for (int s = 0; s < n_split; ++s) MM = fmaxf(MM, __ldcg(p0 + s * (HD + 2) + HD));
    num = 0.f, den = 0.f;
    if (MM != -INFINITY) {
#pragma unroll 4
        for (int s = 0; s < n_split; ++s) {
            const float ms = __ldcg(p0 + s * (HD + 2) + HD);
            const float e = ms == -INFINITY ? 0.f : __expf(ms - MM);
            num = fmaf(e, __ldcg(p0 + s * (HD + 2) + d), num);
            den = fmaf(e, __ldcg(p0 + s * (HD + 2) + HD + 1), den);
        }
    }
    orow[d] = from_op<T>(den > 0.f ? num / den : 0.f);           // fully masked row -> zeros
}

// (Alternative not taken: staging a warp's whole 64-key K and V tiles in shared memory with cp.async -- 32 KB per warp
// requested up front, 6 warps per SM -- leaves so few warps that the score / softmax / P V arithmetic out of shared
// memory is latency-exposed; tools/decode_attn_ab.py compares the variants.)
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

static int g_dec_warps = 4;   // warps per 256-key CTA of the hd-128 decode kernel (mmfs_attn_decode_set_tuning)

static inline long decode_ticket_floats(int B, int H) { return ((long)B * H + 3) / 4 * 4; }   // keeps the partials 16-byte aligned

template <typename T>
static int launch_attn_decode(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask, float *scratch,
                              int B, int H, int Tkv, int hd, long q_bs, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs,
                              float scale, int last_key, cudaStream_t st) {
    const int n_split = (last_key + kDecKeys) / kDecKeys;           // keys 0 .. last_key
    dim3 grid(n_split, H, B);
    if constexpr (sizeof(T) == 2) {
        if (hd == 128 && ((uintptr_t)q % 16 == 0) && (q_bs % 8 == 0) && ((uintptr_t)scratch % 16 == 0)) {
            unsigned *tickets = reinterpret_cast<unsigned *>(scratch);          // [B * H], then the partials
            float *part = scratch + decode_ticket_floats(B, H);
            if (n_split > 1) MMFS_CUDA(cudaMemsetAsync(tickets, 0, sizeof(unsigned) * (size_t)B * H, st));
            if (g_dec_warps == 8)
                attn_decode_split128_kernel<T, 8><<<grid, 256, 0, st>>>((const T *)q, (const T *)k, (const T *)v, key_mask, part, tickets,
                                                                     (T *)out, H, Tkv, q_bs, k_bs, k_ts, v_bs, v_ts, o_bs, scale, last_key);
            else
                attn_decode_split128_kernel<T, 4><<<grid, 128, 0, st>>>((const T *)q, (const T *)k, (const T *)v, key_mask, part, tickets,
                                                                     (T *)out, H, Tkv, q_bs, k_bs, k_ts, v_bs, v_ts, o_bs, scale, last_key);
            MMFS_CUDA(cudaGetLastError());
            return MMFS_OK;
        }
    }
    const size_t smem = (size_t)(hd + kDecWarps * (hd + 2)) * sizeof(float);
    attn_decode_split_kernel<T><<<grid, 32 * kDecWarps, smem, st>>>((const T *)q, (const T *)k, (const T *)v, key_mask, scratch, H,
                                                                   Tkv, hd, q_bs, k_bs, k_ts, v_bs, v_ts, scale, last_key);
    attn_decode_merge_kernel<T><<<dim3(H, B), hd < 128 ? 64 : 128, 0, st>>>(scratch, (T *)out, H, hd, n_split, o_bs);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_attn_generic(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                               int B, int H, int Tq, int Tkv, int hd, long q_bs, long q_ts, long k_bs, long k_ts,
                               long v_bs, long v_ts, long o_bs, long o_ts, float scale, int causal, int past, cudaStream_t st) {
    const long n_rows = (long)B * H * Tq;
    const long blocks = (n_rows + kAttnWarps - 1) / kAttnWarps;
    const int grid = (int)(blocks < (long)num_sms() * 16 ? blocks : (long)num_sms() * 16);
    const size_t smem = (size_t)kAttnWarps * (hd + kAttnChunk) * sizeof(float);
    attn_generic_kernel<T><<<grid, 32 * kAttnWarps, smem, st>>>((const T *)q, (const T *)k, (const T *)v, (T *)out, key_mask,
                                                              n_rows, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts,
                                                              o_bs, o_ts, scale, causal, past);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
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
    switch (dtype) {
        case MMFS_F32: return launch_attn_generic<float>(q, k, v, out, key_mask, B, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, scale, causal, past, st);
        case MMFS_F16: return launch_attn_generic<__half>(q, k, v, out, key_mask, B, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, scale, causal, past, st);
        case MMFS_BF16: return launch_attn_generic<__nv_bfloat16>(q, k, v, out, key_mask, B, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, scale, causal, past, st);
        default: set_error("attn_generic: dtype %d unsupported", dtype); return MMFS_EINVAL;
    }
}

extern "C" int mmfs_attn_decode_set_tuning(int warps) {
    MMFS_CHECK_ARG(warps == 0 || warps == 4 || warps == 8, "attn_decode_set_tuning: warps 0 (default) / 4 / 8");
    g_dec_warps = warps == 0 ? 4 : warps;
    return MMFS_OK;
}

extern "C" long mmfs_attn_decode_scratch_floats(int B, int H, int Tkv, int hd) {
    // tickets [B * H] (hd-128 16-bit path) + one partial per (b, h, split)
    return decode_ticket_floats(B, H) + (long)B * H * ((Tkv + kDecKeys - 1) / kDecKeys) * (hd + 2);
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
    const int last_key = causal ? (past < Tkv - 1 ? past : Tkv - 1) : Tkv - 1;     // the single query row sits at position `past`
    MMFS_CHECK_ARG(last_key >= 0, "attn_decode: negative past");
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case MMFS_F32: return launch_attn_decode<float>(q, k, v, out, key_mask, scratch, B, H, Tkv, hd, q_bs, k_bs, k_ts, v_bs, v_ts, o_bs, scale, last_key, st);
        case MMFS_F16: return launch_attn_decode<__half>(q, k, v, out, key_mask, scratch, B, H, Tkv, hd, q_bs, k_bs, k_ts, v_bs, v_ts, o_bs, scale, last_key, st);
        default: return launch_attn_decode<__nv_bfloat16>(q, k, v, out, key_mask, scratch, B, H, Tkv, hd, q_bs, k_bs, k_ts, v_bs, v_ts, o_bs, scale, last_key, st);
    }
}
