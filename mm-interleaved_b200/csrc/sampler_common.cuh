// sampler_common.cuh -- pieces shared by the deformable-attention sampler kernels
// (msda_fwd_sm100.cu: the drop-in op; mmfs_sampler_sm100.cu: the fused MMFS sampler).
#pragma once
#include "common.cuh"

namespace mmfs {

// ------------------------------------------------------------------------------------
// Index math of one sampling point: cuh:287-291 (pixel coordinates, in-range predicate)
// and cuh:41-48 (floor, lerp fractions).
// ------------------------------------------------------------------------------------
template <typename OP> struct PointGeom {
    bool in_range;
    int h_low, w_low;
    OP lh, lw;
};

__device__ __forceinline__ PointGeom<float> point_geom(float x, float y, int H, int W) {
    // cuh:287-288  `loc_h * spatial_h - 0.5`: the product is an opmath (float) multiply
    // rounded on its own; the double literal then forces a separate subtraction (exact
    // in double, rounded once to float) -- equivalent to an un-fused float subtract.
    // __fmul_rn/__fsub_rn are never contracted into an FMA by nvcc.
    const float h_im = __fsub_rn(__fmul_rn(y, (float)H), 0.5f);
    const float w_im = __fsub_rn(__fmul_rn(x, (float)W), 0.5f);
    PointGeom<float> g;
    g.in_range = (h_im > -1.f) && (w_im > -1.f) && (h_im < (float)H) && (w_im < (float)W);  // cuh:291
    const float hf = floorf(h_im), wf = floorf(w_im);                                       // cuh:41-42
    g.h_low = (int)hf;
    g.w_low = (int)wf;
    g.lh = h_im - hf;  // cuh:46 (h - h_low; hf is integral, the subtraction is exact)
    g.lw = w_im - wf;
    return g;
}

__device__ __forceinline__ PointGeom<double> point_geom(double x, double y, int H, int W) {
    // double dispatch (cu:65): same source expression as the reference, so nvcc applies the
    // same contraction it applies there.
    const double h_im = y * H - 0.5;
    const double w_im = x * W - 0.5;
    PointGeom<double> g;
    g.in_range = (h_im > -1) && (w_im > -1) && (h_im < H) && (w_im < W);
    const double hf = floor(h_im), wf = floor(w_im);
    g.h_low = (int)hf;
    g.w_low = (int)wf;
    g.lh = h_im - hf;
    g.lw = w_im - wf;
    return g;
}

// corner k = 0..3 <-> reference v1..v4: (h_low,w_low) (h_low,w_high) (h_high,w_low) (h_high,w_high)
// validity predicates exactly as cuh:59,65,71,77.
__device__ __forceinline__ bool corner_valid(int corner, int h_low, int w_low, int H, int W) {
    const bool okh = (corner & 2) ? (h_low + 1 <= H - 1) : (h_low >= 0);
    const bool okw = (corner & 1) ? (w_low + 1 <= W - 1) : (w_low >= 0);
    return okh && okw;
}

__device__ __forceinline__ void fma2(float &a0, float &a1, float w0, float w1, float v0, float v1) {
    // two independent fp32 FMAs (Hopper has no packed fp32 pipe)
    a0 = __fmaf_rn(w0, v0, a0);
    a1 = __fmaf_rn(w1, v1, a1);
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// mbarrier + bulk async copy (TMA engine, SASS UBLKCP): one instruction stages a whole
// sampling-location / attention-weight row of the next output row into shared memory.
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                 "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// 512 bytes of zeros: taps that must not contribute (outside the map, invalid corner, masked
// image) are pointed here with weight 0, so the gather loop needs no predicates and a
// non-finite `value` entry can never leak through a 0 * inf product.
static __device__ uint4 g_zero_row[32];

struct __align__(16) Tap {  // mailbox record handed from the index-math lane to the fetching slot
    long long off;          // byte offset from the head slab origin (or to g_zero_row)
    float w0, w1;           // lerp weight * attention weight, duplicated for fma2
};

template <typename T> __device__ __forceinline__ float elem_to_f32(const T *p);
template <> __device__ __forceinline__ float elem_to_f32<float>(const float *p) { return *p; }
template <> __device__ __forceinline__ float elem_to_f32<__half>(const __half *p) { return __half2float(*p); }
template <> __device__ __forceinline__ float elem_to_f32<__nv_bfloat16>(const __nv_bfloat16 *p) { return __bfloat162float(*p); }

constexpr int kTapStride = 33;                      // 16-byte units between corner planes (bank skew)
constexpr int kTapsPerWarp = 4 * kTapStride;        // mailbox entries per warp (32 points x 4 corners)
constexpr int kWarpsPerCta = 8;


// ------------------------------------------------------------------------------------
// Phase 1 helper: the four taps of one sampling point (lane = point) into the warp mailbox.
// Corner planes are skewed by one 16-byte entry so that both the writes (lane = point) and the
// reads (slot = corner) are shared-memory bank-conflict free.
// ------------------------------------------------------------------------------------
__device__ __forceinline__ void emit_taps(Tap *taps, int lane, bool live, const PointGeom<float> &g, float a,
                                          int H, int W, int level_start, long long row_bytes, long long zero_off) {
    Tap t4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { t4[k].off = zero_off; t4[k].w0 = 0.f; t4[k].w1 = 0.f; }
    if (live) {
        const float hh = 1.f - g.lh, hw = 1.f - g.lw;                                       // cuh:48
        const long long o00 = (long long)(level_start + g.h_low * W + g.w_low) * row_bytes;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (corner_valid(k, g.h_low, g.w_low, H, W)) {
                t4[k].off = o00 + ((k & 2) ? (long long)W * row_bytes : 0ll) + ((k & 1) ? row_bytes : 0ll);
                const float wk = ((k & 2) ? g.lh : hh) * ((k & 1) ? g.lw : hw) * a;          // cuh:83
                t4[k].w0 = wk; t4[k].w1 = wk;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k)
        *reinterpret_cast<uint4 *>(&taps[k * kTapStride + lane]) = *reinterpret_cast<const uint4 *>(&t4[k]);
}

// ------------------------------------------------------------------------------------
// Phase 2: gather the 128 taps of a pass.  Slot s of the warp fetches tap (it*RPI + s) =
// (point, corner); every lane moves 16 bytes, i.e. one LDG.128 gathers RPI value rows.
// Groups of 8 fetches whose points are all dead (livemask) are skipped warp-uniformly.
// ------------------------------------------------------------------------------------
template <typename T, int D>
__device__ __forceinline__ void gather_pass(const Tap *taps, unsigned livemask, const char *vbase, int slot,
                                            float (&acc)[16 / sizeof(T)]) {
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int LPR = D / VEC;
    constexpr int RPI = 32 / LPR;
    constexpr int NIT = 128 / RPI;                 // fetch instructions per pass
    constexpr int G = NIT < 8 ? NIT : 8;           // fetches in flight per lane
    constexpr int PPG = (G * RPI) / 4;             // points covered by one group
#pragma unroll 1
    for (int g0 = 0; g0 < NIT; g0 += G) {
        const unsigned pm = (PPG >= 32) ? livemask : ((livemask >> ((g0 * RPI) / 4)) & ((1u << PPG) - 1u));
        if (pm == 0u) continue;                    // warp-uniform: these points are all dead
        Tap t[G];
        uint4 v[G];
#pragma unroll
        for (int it = 0; it < G; ++it) {
            const int tix = (g0 + it) * RPI + slot;        // tap index = point * 4 + corner
            *reinterpret_cast<uint4 *>(&t[it]) =
                *reinterpret_cast<const uint4 *>(&taps[(tix & 3) * kTapStride + (tix >> 2)]);
        }
#pragma unroll
        for (int it = 0; it < G; ++it) v[it] = ldg_nc_v4(vbase + t[it].off);
#pragma unroll
        for (int it = 0; it < G; ++it) {
            float f[VEC];
            Vec16<T>::unpack(v[it], f);
#pragma unroll
            for (int k = 0; k < VEC; k += 2) fma2(acc[k], acc[k + 1], t[it].w0, t[it].w1, f[k], f[k + 1]);
        }
    }
}

// Mixed-precision FMA: d = a(16-bit) * b(16-bit) + c(fp32) with one rounding.  Both 16-bit operands widen to fp32
// exactly, so an fp32 FMA on the widened values gives the same result; the saving is the 16-bit weight's register.
template <typename T> struct MixFma;
template <> struct MixFma<__nv_bfloat16> {
    __device__ __forceinline__ static void fma(float &acc, uint16_t v, uint16_t w) {
        acc = __fmaf_rn(__uint_as_float((uint32_t)v << 16), __uint_as_float((uint32_t)w << 16), acc);
    }
    __device__ __forceinline__ static uint16_t cvt(float w) { __nv_bfloat16 t = __float2bfloat16_rn(w); return *reinterpret_cast<uint16_t *>(&t); }
};
template <> struct MixFma<__half> {
    __device__ __forceinline__ static void fma(float &acc, uint16_t v, uint16_t w) {
        acc = __fmaf_rn(__half2float(__ushort_as_half(v)), __half2float(__ushort_as_half(w)), acc);
    }
    __device__ __forceinline__ static uint16_t cvt(float w) { __half t = __float2half_rn(w); return *reinterpret_cast<uint16_t *>(&t); }
};

// gather_pass with 16-bit tap weights (MMFS_MSDA_W16): 8 mixed-precision FMA per 16-byte fetch instead of 8 unpack + 8 FFMA
template <typename T, int D>
__device__ __forceinline__ void gather_pass_w16(const Tap *taps, unsigned livemask, const char *vbase, int slot,
                                                float (&acc)[16 / sizeof(T)]) {
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int LPR = D / VEC;
    constexpr int RPI = 32 / LPR;
    constexpr int NIT = 128 / RPI;
    constexpr int G = NIT < 8 ? NIT : 8;
    constexpr int PPG = (G * RPI) / 4;
    static_assert(VEC == 8, "16-bit element types only");
#pragma unroll 1
    for (int g0 = 0; g0 < NIT; g0 += G) {
        const unsigned pm = (PPG >= 32) ? livemask : ((livemask >> ((g0 * RPI) / 4)) & ((1u << PPG) - 1u));
        if (pm == 0u) continue;
        Tap t[G];
        uint4 v[G];
#pragma unroll
        for (int it = 0; it < G; ++it) {
            const int tix = (g0 + it) * RPI + slot;
            *reinterpret_cast<uint4 *>(&t[it]) =
                *reinterpret_cast<const uint4 *>(&taps[(tix & 3) * kTapStride + (tix >> 2)]);
        }
#pragma unroll
        for (int it = 0; it < G; ++it) v[it] = ldg_nc_v4(vbase + t[it].off);
#pragma unroll
        for (int it = 0; it < G; ++it) {
            const uint16_t w = MixFma<T>::cvt(t[it].w0);
            const uint32_t r[4] = {v[it].x, v[it].y, v[it].z, v[it].w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                MixFma<T>::fma(acc[2 * k], (uint16_t)(r[k] & 0xffffu), w);
                MixFma<T>::fma(acc[2 * k + 1], (uint16_t)(r[k] >> 16), w);
            }
        }
    }
}
// dispatch: 16-bit weights only for 16-bit element types and only on request
template <typename T, int D>
__device__ __forceinline__ void gather_pass_any(const Tap *taps, unsigned livemask, const char *vbase, int slot,
                                                float (&acc)[16 / sizeof(T)], bool w16) {
    if constexpr (sizeof(T) == 2) {
        if (w16) { gather_pass_w16<T, D>(taps, livemask, vbase, slot, acc); return; }
    }
    gather_pass<T, D>(taps, livemask, vbase, slot, acc);
}

// epilogue: sum the RPI slots, one rounding, 16-byte stores
template <typename T, int D>
__device__ __forceinline__ void store_row(float (&acc)[16 / sizeof(T)], T *out_row, int lane) {
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int LPR = D / VEC;
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1)
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], off);
    if (lane < LPR) stg_v4(out_row + lane * VEC, Vec16<T>::pack(acc));
}

// Persistent-grid work order shared by the sampler kernels.  A tile = kWarpsPerCta *
// rows_per_warp consecutive queries of ONE (b, m); tiles are numbered (b, m, q-tile) with the
// q-tile fastest.  CTA i of the persistent grid sits on SM (i % nsm) in its only wave, so giving
// CTA i the tiles ((i % nsm) * ctas_per_sm + i / nsm) + k * grid makes all CTAs resident on one
// SM walk neighbouring q-tiles of the same head: the head's value slab stays L1-resident.
struct RowCursor { int tile, r, b, m, q; bool ok; };
struct RowWalk {
    int itiles, igrid, qtiles, M, Lq, rows_per_warp, warp;
    __device__ __forceinline__ void settle(RowCursor &c) const {   // (tile, r) -> (b, m, q); skips rows past Lq
        for (;;) {
            if (c.tile >= itiles) { c.ok = false; return; }
            const int qt = c.tile % qtiles, bm = c.tile / qtiles;
            c.m = bm % M; c.b = bm / M;
            c.q = (qt * kWarpsPerCta + warp) * rows_per_warp + c.r;
            if (c.q < Lq) { c.ok = true; return; }
            c.r = 0; c.tile += igrid;  // the rest of this tile's rows are past Lq as well
        }
    }
    __device__ __forceinline__ RowCursor first(int ctas_per_sm, int nsm, int swizzle) const {
        long t0 = blockIdx.x;
        if (swizzle && gridDim.x == (unsigned)(nsm * ctas_per_sm))
            t0 = (long)(blockIdx.x % nsm) * ctas_per_sm + blockIdx.x / nsm;
        RowCursor c; c.tile = (int)t0; c.r = 0; c.b = c.m = c.q = 0; c.ok = false;
        settle(c);
        return c;
    }
    __device__ __forceinline__ RowCursor next(RowCursor c) const {
        if (++c.r == rows_per_warp) { c.r = 0; c.tile += igrid; settle(c); return c; }
        if (++c.q >= Lq) { c.r = 0; c.tile += igrid; settle(c); }   // same tile, next query: no divisions
        return c;
    }
};

// ------------------------------------------------------------------------------------
// Fused MMFS sampler: argument block + small numeric helpers shared by the generic kernel
// (mmfs_sampler_sm100.cu) and the specialised P = 8 / D = 64 kernel (mmfs_sampler_v2_sm100.cu).
// ------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ float round_to(float x) { return to_op(from_op<T>(x)); }
template <> __device__ __forceinline__ float round_to<float>(float x) { return x; }

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct SamplerArgs {
    const void *value;
    const int64_t *shapes, *starts;
    const void *qproj, *rtable;
    const uint8_t *relpos;
    const float *refpts, *scale_ratios;
    void *out;
    float *null_mass;
    void *loc_out, *attn_out;
    int S, M, n_img, n_lvl, Lq, P, Lq_r, Nr, Lr, R;
    float null_logit;
    unsigned flags;
    int rows_per_warp, qtiles;
    long ntiles;
    int ctas_per_sm, nsm, swizzle;
    int walk_dq, walk_dm, walk_db;   // specialised kernel: grid-stride decomposed into (q-tile, head, batch) steps
};


// Specialised fused sampler (16-bit element types, D = 64, P = 8, n_lvl in {3, 4}); returns MMFS_EUNSUPPORTED
// without touching the error text when the configuration is outside its domain (the caller then takes the
// generic kernel).
int launch_sampler_v2(const SamplerArgs &a, int N, int D, int dtype, cudaStream_t st);
int sampler_v2_set_tuning(int rows_per_warp, int wmode);

}  // namespace mmfs
