// kv_fp8_sm100.cu -- the decoder's KV cache in FP8: keys and values stored as E4M3 bytes with one fp32 scale per
// (row, position, head), written by the RoPE + append kernel and read by split-KV decode attention.
//
// Quantisation (the rule of ops.quantize_kv_fp8): a head vector x of hd values gets the least power of two s with
// amax(|x|) / s <= 448 (1 for an all-zero vector); x8 = e4m3(x / s), round to nearest even.  x / s is exact, the
// cast never saturates, and x8 * s is exact in bf16 and fp16, so a model reading x8 * s is an ordinary 16-bit model
// whose keys and values happen to be those numbers.  The append kernel also writes x8 * s back over its k / v inputs
// (the QKV GEMM's output), so a prefill's attention over its own positions sees exactly what later steps read.
//
// Decode attention (one query row over the cache) is a split-KV kernel on the skeleton of decode_common.cuh, whose
// splits, cache addressing and split merge it shares with the 16-bit decode kernels.  Scales are folded into
// scalars: score_j = (q . k8_j) * (scale_k[j] * softmax_scale), and P V accumulates (p_j * scale_v[j]) * v8_j.  The
// e4m3 -> f16 conversion (cvt.rn.f16x2.e4m3x2) is exact and every sum is fp32.
#include <cuda_fp8.h>

#include "decode_common.cuh"

namespace mmfs {
namespace {

constexpr int kFp8MaxHd = 256;

template <typename T> __device__ __forceinline__ float rnd_t(float x) { return to_op(from_op<T>(x)); }

// two e4m3 bytes (the low 16 bits) -> two floats, exactly
__device__ __forceinline__ float2 e4m3x2_to_float2(uint32_t v16) {
    uint32_t r;
    asm("{\n\t.reg .b16 t;\n\tcvt.u16.u32 t, %1;\n\tcvt.rn.f16x2.e4m3x2 %0, t;\n\t}" : "=r"(r) : "r"(v16));
    return __half22float2(*reinterpret_cast<const __half2 *>(&r));
}

__device__ __forceinline__ void unpack_e4m3x16(const uint4 &v, float (&f)[16]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 a = e4m3x2_to_float2(w[i] & 0xffffu), b = e4m3x2_to_float2(w[i] >> 16);
        f[4 * i] = a.x; f[4 * i + 1] = a.y; f[4 * i + 2] = b.x; f[4 * i + 3] = b.y;
    }
}

__device__ __forceinline__ float e4m3_to_float(uint8_t b) { return e4m3x2_to_float2(b).x; }

// the least power of two s with amax / s <= 448, 1 for amax == 0: amax = m * 2^e with m in [0.5, 1) and 448 = 0.875 * 2^9
__device__ __forceinline__ float kv_scale_of(float amax) {
    if (!(amax > 0.f)) return 1.f;
    int e;
    const float m = frexpf(amax, &e);
    return ldexpf(1.f, m <= 0.875f ? e - 9 : e - 8);
}

// ---- RoPE + append ----------------------------------------------------------------------------------------------
// One warp per (token, q / k / v, head); lane owns the rotation pairs (d, d + hd/2) for d = lane + 32 i.  q is rotated in
// place with rope_append_kernel's arithmetic (bit-identical q); the rotated k and the v are quantised per head vector,
// their bytes and scales go to the cache at position slot + t, and x8 * s overwrites the k / v inputs.
template <typename T>
__global__ void __launch_bounds__(256) rope_append_fp8_kernel(
    T *__restrict__ q, T *__restrict__ k, T *__restrict__ v, const float *__restrict__ cos_t, const float *__restrict__ sin_t,
    const int64_t *__restrict__ pos, uint8_t *__restrict__ k8, uint8_t *__restrict__ v8, float *__restrict__ ks,
    float *__restrict__ vs, const int64_t *__restrict__ slot_dev, long slot_host, long n_tok, int H, int hd, int q_stride,
    int k_stride, int v_stride, long c_bs, long c_ts, long s_bs, long s_ts, int pos_per_batch, int T_len) {
    const int lane = threadIdx.x & 31;
    const int half = hd >> 1;
    const long n_items = n_tok * 3 * H;
    const long slot = slot_dev != nullptr ? (long)*slot_dev : slot_host;
    const long warps = ((long)gridDim.x * blockDim.x) >> 5;
    for (long item = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < n_items; item += warps) {
        const long tok = item / (3 * H);
        const int r = (int)(item - tok * 3 * H), which = r / H, h = r - which * H;   // which: 0 q, 1 k, 2 v
        T *x = (which == 0 ? q + tok * q_stride : which == 1 ? k + tok * k_stride : v + tok * v_stride) + (long)h * hd;
        float a[4], bv[4];                               // the pair (d, d + half) of d = lane + 32 i
        float amax = 0.f;
        const long p = pos[pos_per_batch ? tok : (tok % T_len)];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int d = lane + 32 * i;
            a[i] = 0.f; bv[i] = 0.f;
            if (d >= half) continue;
            const float x1 = to_op(x[d]), x2 = to_op(x[d + half]);
            if (which == 2) {
                a[i] = x1; bv[i] = x2;
            } else {
                const float c = rnd_t<T>(cos_t[p * hd + d]), s = rnd_t<T>(sin_t[p * hd + d]);
                a[i] = rnd_t<T>(rnd_t<T>(x1 * c) + rnd_t<T>(-x2 * s));
                bv[i] = rnd_t<T>(rnd_t<T>(x2 * c) + rnd_t<T>(x1 * s));
            }
            amax = fmaxf(amax, fmaxf(fabsf(a[i]), fabsf(bv[i])));
        }
        if (which == 0) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int d = lane + 32 * i;
                if (d < half) { x[d] = from_op<T>(a[i]); x[d + half] = from_op<T>(bv[i]); }
            }
            continue;                                    // warp-uniform
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        const float s = kv_scale_of(amax);
        const long b = tok / T_len, t = tok - b * T_len;
        uint8_t *dst = (which == 1 ? k8 : v8) + b * c_bs + (slot + t) * c_ts + (long)h * hd;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int d = lane + 32 * i;
            if (d >= half) continue;
            const __nv_fp8_storage_t q1 = __nv_cvt_float_to_fp8(a[i] / s, __NV_SATFINITE, __NV_E4M3);
            const __nv_fp8_storage_t q2 = __nv_cvt_float_to_fp8(bv[i] / s, __NV_SATFINITE, __NV_E4M3);
            dst[d] = q1;
            dst[d + half] = q2;
            x[d] = from_op<T>(e4m3_to_float(q1) * s);   // exact
            x[d + half] = from_op<T>(e4m3_to_float(q2) * s);
        }
        if (lane == 0) (which == 1 ? ks : vs)[b * s_bs + (slot + t) * s_ts + h] = s;
    }
}

// ---- decode attention -------------------------------------------------------------------------------------------
struct Fp8KV {                    // an e4m3 (rows, T, H, hd) K / V pair and its fp32 (rows, T, >= H) scales
    const uint8_t *k, *v;
    const float *ks, *vs;
    long bs, ts, sbs, sts;        // strides in elements: K / V rows and positions, scale rows and positions
};

// HD128: a key is 128 bytes, 8 lanes x one 16-byte load, 4 keys per warp step; K and V come in batches of 32 keys
// (eight 16-byte loads per lane, 4 KB per warp) double-buffered in registers.  Otherwise (hd % 32 == 0, <= 256): lane =
// key for the scores (q from shared memory), lane = hd / 32 channels for P V.  `g` is the SHARED layout's generated rows.
template <typename T, bool SHARED, bool HD128>
__global__ void __launch_bounds__(32 * kDecWarps, 4)
attn_decode_fp8_kernel(const T *__restrict__ q, Fp8KV c, Fp8KV g, SharedLayout sl, const uint8_t *__restrict__ key_mask,
                       float *__restrict__ part, unsigned *__restrict__ tickets, T *__restrict__ out, int H, int Tkv, int hd,
                       long q_bs, long o_bs, float scale, int last_key) {
    __shared__ float s_p[kDecWarps][kDecKPW];
    __shared__ __align__(16) float s_acc[kDecWarps][HD128 ? 128 : kFp8MaxHd];
    __shared__ __align__(16) float s_q[HD128 ? 4 : kFp8MaxHd];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, h = blockIdx.y;
    const DecodeCta<SHARED> cta(sl);
    const int b = cta.b;
    const int k0 = cta.split * kDecKeys + warp * kDecKPW;

    unsigned ok_lo = 0u, ok_hi = 0u;                 // validity of keys k0 + 0..31 / k0 + 32..63
    float ks_lo = 0.f, ks_hi = 0.f, vs_lo = 0.f, vs_hi = 0.f;   // their scales (lane = key); masked keys' are never used
    if (k0 <= last_key) {                            // warp-uniform
        const int ja = k0 + lane, jb = ja + 32;
        ok_lo = __ballot_sync(0xffffffffu, ja <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + ja]));
        ok_hi = __ballot_sync(0xffffffffu, jb <= last_key && (key_mask == nullptr || key_mask[(long)b * Tkv + jb]));
        const int ca = min(ja, last_key), cb = min(jb, last_key);
        ks_lo = *cta.at(c.ks + h, c.sbs, c.sts, g.ks + h, g.sbs, g.sts, ca);
        ks_hi = *cta.at(c.ks + h, c.sbs, c.sts, g.ks + h, g.sbs, g.sts, cb);
        vs_lo = *cta.at(c.vs + h, c.sbs, c.sts, g.vs + h, g.sbs, g.sts, ca);
        vs_hi = *cta.at(c.vs + h, c.sbs, c.sts, g.vs + h, g.sbs, g.sts, cb);
    }
    float m = -INFINITY, l = 0.f;
    auto softmax = [&]() {                           // over the warp's 64 scores in s_p, in place
        __syncwarp();
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
    };

    if constexpr (HD128) {
        float acc[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[i] = 0.f;
        const int sub = lane & 7, grp = lane >> 3;
        if (ok_lo | ok_hi) {                         // warp-uniform: at least one visible key
            float qf[16];
            {
                const T *qp = q + b * q_bs + (long)h * 128 + sub * 16;
                float f[8];
                Vec16<T>::unpack(ldg_nc_v4(qp), f);
#pragma unroll
                for (int i = 0; i < 8; ++i) qf[i] = f[i];
                Vec16<T>::unpack(ldg_nc_v4(qp + 8), f);
#pragma unroll
                for (int i = 0; i < 8; ++i) qf[8 + i] = f[i];
            }
            auto load = [&](uint4 (&r)[8], const uint8_t *pre, const uint8_t *gen, int bt) {
#pragma unroll
                for (int s = 0; s < 8; ++s)
                    r[s] = ldg_nc_v4(cta.at(pre + (long)h * 128 + sub * 16, c.bs, c.ts, gen + (long)h * 128 + sub * 16, g.bs,
                                            g.ts, min(k0 + bt * 32 + s * 4 + grp, last_key)));
            };
            auto scores = [&](const uint4 (&r)[8], int bt) {
                const unsigned okw = bt ? ok_hi : ok_lo;
                const float ksw = bt ? ks_hi : ks_lo;
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    float f[16];
                    unpack_e4m3x16(r[s], f);
                    float d0 = 0.f, d1 = 0.f;
#pragma unroll
                    for (int i = 0; i < 16; i += 2) { d0 = fmaf(f[i], qf[i], d0); d1 = fmaf(f[i + 1], qf[i + 1], d1); }
                    float dot = d0 + d1;
                    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
                    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
                    dot += __shfl_xor_sync(0xffffffffu, dot, 4);
                    const int kk = s * 4 + grp;
                    const float sk = __shfl_sync(0xffffffffu, ksw, kk);
                    if (sub == 0) s_p[warp][bt * 32 + kk] = ((okw >> kk) & 1u) ? dot * (sk * scale) : -INFINITY;
                }
            };
            auto pv = [&](const uint4 (&r)[8], int bt) {
                const float vsw = bt ? vs_hi : vs_lo;
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    const int kk = s * 4 + grp;
                    const float p = s_p[warp][bt * 32 + kk];
                    const float sv = __shfl_sync(0xffffffffu, vsw, kk);
                    if (p != 0.f) {                  // a masked slot is never read into the sums
                        const float pw = p * sv;
                        float f[16];
                        unpack_e4m3x16(r[s], f);
#pragma unroll
                        for (int i = 0; i < 16; ++i) acc[i] = fmaf(pw, f[i], acc[i]);
                    }
                }
            };
            uint4 ra[8], rb[8];
            load(ra, c.k, g.k, 0);
            load(rb, c.k, g.k, 1); scores(ra, 0);
            load(ra, c.v, g.v, 0); scores(rb, 1);
            softmax();
            load(rb, c.v, g.v, 1); pv(ra, 0);
            pv(rb, 1);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 8);
                acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], 16);
            }
        }
        if (lane < 8) {
#pragma unroll
            for (int i = 0; i < 16; i += 4)
                *reinterpret_cast<float4 *>(&s_acc[warp][lane * 16 + i]) = make_float4(acc[i], acc[i + 1], acc[i + 2], acc[i + 3]);
        }
    } else {
        for (int d = threadIdx.x; d < hd; d += blockDim.x) s_q[d] = to_op(q[b * q_bs + (long)h * hd + d]);
        __syncthreads();
        const int cpl = hd / 32;
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        if (ok_lo | ok_hi) {
#pragma unroll 1
            for (int hf = 0; hf < 2; ++hf) {
                const int j = min(k0 + hf * 32 + lane, last_key);
                const uint8_t *kp = cta.at(c.k + (long)h * hd, c.bs, c.ts, g.k + (long)h * hd, g.bs, g.ts, j);
                float dot = 0.f;
                for (int d0 = 0; d0 < hd; d0 += 16) {
                    float f[16];
                    unpack_e4m3x16(ldg_nc_v4(kp + d0), f);
#pragma unroll
                    for (int e = 0; e < 16; ++e) dot = fmaf(f[e], s_q[d0 + e], dot);
                }
                const bool ok = (((hf ? ok_hi : ok_lo) >> lane) & 1u) != 0u;
                s_p[warp][hf * 32 + lane] = ok ? dot * ((hf ? ks_hi : ks_lo) * scale) : -INFINITY;
            }
            softmax();
            for (int jj = 0; jj < kDecKPW; ++jj) {
                const float p = s_p[warp][jj];
                const float sv = __shfl_sync(0xffffffffu, jj < 32 ? vs_lo : vs_hi, jj & 31);
                if (p == 0.f) continue;              // warp-uniform; a masked slot is never read into the sums
                const uint8_t *vp = cta.at(c.v + (long)h * hd + lane * cpl, c.bs, c.ts, g.v + (long)h * hd + lane * cpl, g.bs,
                                           g.ts, k0 + jj);
                const float pw = p * sv;
#pragma unroll
                for (int i = 0; i < 8; ++i)
                    if (i < cpl) acc[i] = fmaf(pw, e4m3_to_float(vp[i]), acc[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (i < cpl) s_acc[warp][lane * cpl + i] = acc[i];
    }
    decode_epilogue<T>(m, l, &s_acc[0][0], HD128 ? 128 : kFp8MaxHd, hd, part, tickets, (long)b * H + h,
                       out + b * o_bs + (long)h * hd, cta.split, cta.n_split);
}

// B query rows; SHARED: B = P * sl.G rows, c the prefix and g the generated rows
template <typename T, bool SHARED>
int launch_decode_fp8(const void *q, const Fp8KV &c, const Fp8KV &g, const SharedLayout &sl, void *out,
                      const uint8_t *key_mask, float *scratch, int B, int H, int Tkv, int hd, long q_bs, long o_bs, float scale,
                      int last_key, cudaStream_t st) {
    const dim3 grid = decode_grid(last_key, B, H, sl);
    unsigned *tickets = reinterpret_cast<unsigned *>(scratch);
    float *part = scratch + decode_ticket_floats(B, H);
    if (decode_splits(last_key) > 1) MMFS_CUDA(cudaMemsetAsync(tickets, 0, sizeof(unsigned) * (size_t)B * H, st));
    bool done = false;
    if constexpr (sizeof(T) == 2) {
        if (hd == 128) {
            attn_decode_fp8_kernel<T, SHARED, true><<<grid, 32 * kDecWarps, 0, st>>>(
                (const T *)q, c, g, sl, key_mask, part, tickets, (T *)out, H, Tkv, hd, q_bs, o_bs, scale, last_key);
            done = true;
        }
    }
    if (!done)
        attn_decode_fp8_kernel<T, SHARED, false><<<grid, 32 * kDecWarps, 0, st>>>(
            (const T *)q, c, g, sl, key_mask, part, tickets, (T *)out, H, Tkv, hd, q_bs, o_bs, scale, last_key);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

bool fp8_rows_aligned(const Fp8KV &c) {
    return ((uintptr_t)c.k | (uintptr_t)c.v) % 16 == 0 && c.bs % 16 == 0 && c.ts % 16 == 0 &&
           ((uintptr_t)c.ks | (uintptr_t)c.vs) % 4 == 0;
}

// ---- dequantisation ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) kv_dequantize_kernel(const uint8_t *__restrict__ x8, const float *__restrict__ sc,
                                                            T *__restrict__ out, int T_len, int H, int hd, long n,
                                                            long x_bs, long x_ts, long s_bs, long s_ts, long o_bs, long o_ts) {
    const int per_pos = H * hd / 16;                 // 16-byte chunks of one position; a chunk lies in one head
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long bt = i / per_pos;
        const int e0 = (int)(i - bt * per_pos) * 16;
        const long b = bt / T_len, t = bt - b * T_len;
        const float s = sc[b * s_bs + t * s_ts + e0 / hd];
        float f[16];
        unpack_e4m3x16(ldg_nc_v4(x8 + b * x_bs + t * x_ts + e0), f);
        constexpr int VEC = 16 / (int)sizeof(T);
        T *o = out + b * o_bs + t * o_ts + e0;
#pragma unroll
        for (int c = 0; c < 16; c += VEC) {
            float y[VEC];
#pragma unroll
            for (int e = 0; e < VEC; ++e) y[e] = f[c + e] * s;
            *reinterpret_cast<uint4 *>(o + c) = Vec16<T>::pack(y);
        }
    }
}

}  // namespace
}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_rope_qk_append_fp8(void *q, void *k, void *v, const float *cos_table, const float *sin_table,
                                       const int64_t *position_ids, uint8_t *k_cache, uint8_t *v_cache, float *k_scale,
                                       float *v_scale, const int64_t *slot_dev, long slot_host, long n_tokens, int T_len,
                                       int H, int hd, int q_stride, int k_stride, int v_stride, long cache_bs,
                                       long cache_ts, long scale_bs, long scale_ts, int pos_per_batch, int dtype,
                                       void *stream) {
    MMFS_CHECK_ARG(n_tokens >= 0 && H > 0 && hd > 0 && T_len > 0 && slot_host >= 0, "rope_qk_append_fp8: bad shape");
    if (n_tokens == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && cos_table && sin_table && position_ids && k_cache && v_cache && k_scale && v_scale,
                   "rope_qk_append_fp8: null pointer argument");
    if (hd % 2 != 0 || hd > 256 || scale_ts < H || cache_ts < (long)H * hd) {
        set_error("rope_qk_append_fp8: needs an even head dim <= 256 and cache / scale positions holding H heads");
        return MMFS_EUNSUPPORTED;
    }
    return dispatch_dtype<kF32Types, MMFS_EUNSUPPORTED>(dtype, "rope_qk_append_fp8", [&](auto tag) {
        using T = typename decltype(tag)::type;
        const long warps = n_tokens * 3 * H;
        rope_append_fp8_kernel<T><<<capped_grid((warps + 7) / 8, 8), 256, 0, (cudaStream_t)stream>>>(
            (T *)q, (T *)k, (T *)v, cos_table, sin_table, position_ids, k_cache, v_cache, k_scale, v_scale, slot_dev, slot_host,
            n_tokens, H, hd, q_stride, k_stride, v_stride, cache_bs, cache_ts, scale_bs, scale_ts, pos_per_batch, T_len);
        MMFS_CUDA(cudaGetLastError());
        return MMFS_OK;
    });
}

extern "C" int mmfs_attn_decode_fp8(const void *q, const uint8_t *k, const uint8_t *v, const float *k_scale,
                                    const float *v_scale, void *out, const uint8_t *key_mask, float *scratch, int B, int H,
                                    int Tkv, int hd, long q_bs, long kv_bs, long kv_ts, long s_bs, long s_ts, long o_bs,
                                    float scale, int causal, int past, int dtype, void *stream) {
    MMFS_CHECK_ARG(B >= 0 && H > 0 && Tkv > 0 && hd > 0, "attn_decode_fp8: bad shape");
    if (B == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && k_scale && v_scale && out && scratch, "attn_decode_fp8: null pointer argument");
    const Fp8KV c{k, v, k_scale, v_scale, kv_bs, kv_ts, s_bs, s_ts};
    if (hd % 32 != 0 || hd > 256 || B > 65535 || H > 65535 || s_ts < H || !fp8_rows_aligned(c) ||
        ((uintptr_t)q % 16) != 0 || (q_bs * (long)dtype_size(dtype)) % 16 != 0) {
        set_error("attn_decode_fp8: needs hd %% 32 == 0 (<= 256), 16-byte aligned q and K / V rows, scale rows of >= H");
        return MMFS_EUNSUPPORTED;
    }
    const int last_key = decode_last_key(causal, past, Tkv);
    MMFS_CHECK_ARG(last_key >= 0, "attn_decode_fp8: negative past");
    return dispatch_dtype<kF32Types, MMFS_EUNSUPPORTED>(dtype, "attn_decode_fp8", [&](auto tag) {
        return launch_decode_fp8<typename decltype(tag)::type, false>(q, c, c, SharedLayout{}, out, key_mask, scratch, B, H,
                                                                      Tkv, hd, q_bs, o_bs, scale, last_key, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_attn_decode_shared_fp8(const void *q, const uint8_t *k_prefix, const uint8_t *v_prefix,
                                           const float *ks_prefix, const float *vs_prefix, const uint8_t *k_gen,
                                           const uint8_t *v_gen, const float *ks_gen, const float *vs_gen, void *out,
                                           const uint8_t *key_mask, const long long *prefix_len, float *scratch, int R, int G,
                                           int H, int Tkv, int Tp, int max_new, int hd, long q_bs, long p_bs, long p_ts,
                                           long ps_bs, long ps_ts, long g_bs, long g_ts, long gs_bs, long gs_ts, long o_bs,
                                           float scale, int causal, int past, int dtype, void *stream) {
    MMFS_CHECK_ARG(R >= 0 && G > 0 && H > 0 && Tkv > 0 && Tp > 0 && hd > 0, "attn_decode_shared_fp8: bad shape");
    MMFS_CHECK_ARG(R % G == 0, "attn_decode_shared_fp8: R = %d rows are not whole groups of G = %d", R, G);
    MMFS_CHECK_ARG(max_new >= 1, "attn_decode_shared_fp8: max_new must be >= 1");
    if (R == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k_prefix && v_prefix && ks_prefix && vs_prefix && k_gen && v_gen && ks_gen && vs_gen && out &&
                       prefix_len && scratch,
                   "attn_decode_shared_fp8: null pointer argument");
    const Fp8KV pre{k_prefix, v_prefix, ks_prefix, vs_prefix, p_bs, p_ts, ps_bs, ps_ts};
    const Fp8KV gen{k_gen, v_gen, ks_gen, vs_gen, g_bs, g_ts, gs_bs, gs_ts};
    if (hd % 32 != 0 || hd > 256 || R / G > 65535 || H > 65535 || ps_ts < H || gs_ts < H || !fp8_rows_aligned(pre) ||
        !fp8_rows_aligned(gen) || ((uintptr_t)q % 16) != 0 || (q_bs * (long)dtype_size(dtype)) % 16 != 0) {
        set_error("attn_decode_shared_fp8: needs hd %% 32 == 0 (<= 256), 16-byte aligned q and prefix / gen rows, scale "
                  "rows of >= H, R / G <= 65535");
        return MMFS_EUNSUPPORTED;
    }
    const int last_key = decode_last_key(causal, past, Tkv);
    MMFS_CHECK_ARG(last_key >= 0, "attn_decode_shared_fp8: negative past");
    return dispatch_dtype<kF32Types, MMFS_EUNSUPPORTED>(dtype, "attn_decode_shared_fp8", [&](auto tag) {
        return launch_decode_fp8<typename decltype(tag)::type, true>(q, pre, gen, SharedLayout{prefix_len, G, Tp, max_new},
                                                                     out, key_mask, scratch, R, H, Tkv, hd, q_bs, o_bs, scale,
                                                                     last_key, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_kv_dequantize_fp8(const uint8_t *x8, const float *scale, void *out, int B, int T_len, int H, int hd,
                                      long x_bs, long x_ts, long s_bs, long s_ts, long o_bs, long o_ts, int dtype,
                                      void *stream) {
    MMFS_CHECK_ARG(B >= 0 && T_len >= 0 && H > 0 && hd > 0, "kv_dequantize_fp8: bad shape");
    if (B == 0 || T_len == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x8 && scale && out, "kv_dequantize_fp8: null pointer argument");
    const long es = (long)dtype_size(dtype);
    if (hd % 16 != 0 || s_ts < H || ((uintptr_t)x8 | (uintptr_t)out) % 16 != 0 || x_bs % 16 != 0 || x_ts % 16 != 0 ||
        (o_bs * es) % 16 != 0 || (o_ts * es) % 16 != 0) {
        set_error("kv_dequantize_fp8: needs hd %% 16 == 0, 16-byte aligned rows and scale rows of >= H");
        return MMFS_EUNSUPPORTED;
    }
    return dispatch_dtype<kF32Types, MMFS_EUNSUPPORTED>(dtype, "kv_dequantize_fp8", [&](auto tag) {
        using T = typename decltype(tag)::type;
        const long n = (long)B * T_len * H * hd / 16;
        kv_dequantize_kernel<T><<<capped_grid((n + 255) / 256, 8), 256, 0, (cudaStream_t)stream>>>(
            x8, scale, (T *)out, T_len, H, hd, n, x_bs, x_ts, s_bs, s_ts, o_bs, o_ts);
        MMFS_CUDA(cudaGetLastError());
        return MMFS_OK;
    });
}
