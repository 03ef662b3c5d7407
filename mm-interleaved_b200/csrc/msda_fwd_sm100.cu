// msda_fwd_sm100.cu -- multi-scale deformable attention forward for sm_90a.
//
// Replaces the reference's thread-per-output-scalar kernel
//   ops/src/cuda/ms_deform_im2col_cuda.cuh:240-302 (ms_deformable_im2col_gpu_kernel)
//   ops/src/cuda/ms_deform_im2col_cuda.cuh:36-87   (ms_deform_attn_im2col_bilinear)
// with a H100-first design (nothing here is translated from the reference kernel):
//
//   * one WARP per output row (b, q, m); every warp-level fetch moves 512 B: the warp is
//     split into RPI = 32 / (D*sizeof(T)/16) "slots", each slot fetches one 16-byte-
//     per-lane value row, so for D = 64 bf16 a single LDG.128 gathers the four
//     bilinear corners of a sampling point (4 fully used 128-byte lines);
//   * index math is done ONCE per (point, corner) -- lane = (point-in-chunk, corner) --
//     instead of once per channel, and handed to the fetching lanes through a 256-byte
//     per-warp shared-memory mailbox (or warp shuffles, template switch);
//   * CTAs are laid out (b, m, q-tile) with the q-tile fastest, so all warps of a CTA
//     -- and neighbouring CTAs -- walk the SAME head's value slab: it stays L1/L2
//     resident (the reference interleaves 2 heads per 128-thread block);
//   * all N batch entries in one launch, 64-bit base addressing, fp32 accumulation,
//     one rounding at the store; sampling locations / weights are streamed past L1;
//   * fetches of taps that cannot contribute (outside the map, masked image => weight
//     exactly 0) are predicated off, whole 8-point chunks are skipped warp-uniformly.
//
// The sampling-point index math (point_geom) is the single statement shared by the
// forward kernels and by the index-stream kernel that the parity tests compare
// bit-for-bit with oracle/msda_ref.c.
#include "sampler_common.cuh"

namespace mmfs {

// Shared-memory layout of one CTA (all offsets 16-byte aligned):
//   int4     lvl[L]                              {H, W, level_start, -}
//   per warp: uint64_t bar[2]                    mbarriers of the two staging buffers
//             T stage[2][stage_elems]            loc row (2*LP) then attn row (LP), padded to 16 B
//             Tap taps[kTapsPerWarp]             mailbox
template <typename T, int D>
__global__ void __launch_bounds__(32 * kWarpsPerCta, 3)
msda_fwd_rows_kernel(const T *__restrict__ value, const int64_t *__restrict__ shapes,
                     const int64_t *__restrict__ starts, const T *__restrict__ loc,
                     const T *__restrict__ attn, T *__restrict__ out,
                     int S, int M, int L, int Lq, int P, int p_shift, unsigned flags,
                     int rows_per_warp, int qtiles, long ntiles, int ctas_per_sm, int nsm,
                     int stage_elems, int bulk_ok) {
    constexpr int VEC = 16 / (int)sizeof(T);  // channels per lane
    constexpr int LPR = D / VEC;              // lanes per value row
    static_assert(D % VEC == 0 && LPR >= 1 && LPR <= 32 && (LPR & (LPR - 1)) == 0, "unsupported D");

    extern __shared__ int4 s_dyn[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int4 *s_lvl = s_dyn;
    const int per_warp_bytes = 16 + 2 * stage_elems * (int)sizeof(T) + kTapsPerWarp * (int)sizeof(Tap);
    char *wbase = reinterpret_cast<char *>(s_dyn + L) + warp * per_warp_bytes;
    uint64_t *bar = reinterpret_cast<uint64_t *>(wbase);
    T *stage = reinterpret_cast<T *>(wbase + 16);
    Tap *taps = reinterpret_cast<Tap *>(wbase + 16 + 2 * stage_elems * (int)sizeof(T));

    for (int l = threadIdx.x; l < L; l += blockDim.x)
        s_lvl[l] = make_int4((int)shapes[2 * l], (int)shapes[2 * l + 1], (int)starts[l], 0);
    if (lane == 0) {
        bar_init(&bar[0], 1);
        bar_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int LP = L * P;
    const long long row_bytes = (long long)M * D * (int)sizeof(T);
    const bool strict = flags & MMFS_MSDA_STRICT;
    const int slot = lane / LPR;
    const uint32_t loc_bytes = (uint32_t)(2 * LP * (int)sizeof(T)), att_bytes = (uint32_t)(LP * (int)sizeof(T));

    RowWalk walk;
    walk.itiles = (int)ntiles; walk.igrid = (int)gridDim.x; walk.qtiles = qtiles; walk.M = M; walk.Lq = Lq;
    walk.rows_per_warp = rows_per_warp; walk.warp = warp;

    auto stage_row = [&](int b, int m, int q, int buf) {  // whole warp calls; fills stage[buf]
        const size_t qm = ((size_t)b * Lq + q) * M + m;
        T *dst = stage + buf * stage_elems;
        const T *lsrc = loc + qm * (size_t)LP * 2;
        const T *asrc = attn + qm * (size_t)LP;
        if (bulk_ok) {   // bulk async copies (TMA engine): two instructions stage the whole row
            if (lane == 0) {
                bar_expect_tx(&bar[buf], loc_bytes + att_bytes);
                bulk_g2s(dst, lsrc, loc_bytes, &bar[buf]);
                bulk_g2s(dst + 2 * LP, asrc, att_bytes, &bar[buf]);
            }
        } else {         // rows not 16-byte aligned / sized: plain loads
            for (int i = lane; i < 2 * LP; i += 32) dst[i] = lsrc[i];
            for (int i = lane; i < LP; i += 32) dst[2 * LP + i] = asrc[i];
        }
    };

    RowCursor cur = walk.first(ctas_per_sm, nsm);
    unsigned n_staged = 0;  // rows staged so far: buffer = n & 1, parity = (n >> 1) & 1
    if (cur.ok) stage_row(cur.b, cur.m, cur.q, 0);

    while (cur.ok) {
        // look ahead: next valid row of this warp, staged into the other buffer right away
        const RowCursor nxt = walk.next(cur);
        const int b = cur.b, m = cur.m, q = cur.q;
        const int buf = n_staged & 1;
        const unsigned parity = (n_staged >> 1) & 1;
        if (nxt.ok) stage_row(nxt.b, nxt.m, nxt.q, buf ^ 1);
        if (bulk_ok) bar_wait(&bar[buf], parity); else __syncwarp();
        ++n_staged;

        const T *s_loc = stage + buf * stage_elems;
        const T *s_att = s_loc + 2 * LP;
        const char *slab = reinterpret_cast<const char *>(value + ((size_t)b * S * M + m) * D);
        const char *vbase = slab + (lane % LPR) * 16;   // per-lane gather base (one 64-bit add per fetch)
        const long long zero_off = reinterpret_cast<const char *>(g_zero_row) - slab;

        float acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = 0.f;

        for (int p0 = 0; p0 < LP; p0 += 32) {
            // ---- phase 1: one sampling point per lane, four taps each ----------------------
            const int j = p0 + lane;
            bool live = false;
            PointGeom<float> g;
            g.in_range = false; g.h_low = g.w_low = 0; g.lh = g.lw = 0.f;
            float a = 0.f;
            int4 lv = make_int4(1, 1, 0, 0);
            if (j < LP) {
                a = elem_to_f32(s_att + j);
                if (strict || a != 0.f) {   // masked images: weight exactly 0 -> no geometry, no fetch
                    const float x = elem_to_f32(s_loc + 2 * j), y = elem_to_f32(s_loc + 2 * j + 1);
                    lv = s_lvl[(p_shift >= 0) ? (j >> p_shift) : (j / P)];
                    g = point_geom(x, y, lv.x, lv.y);
                    live = g.in_range;
                }
            }
            const unsigned livemask = __ballot_sync(0xffffffffu, live);
            if (livemask == 0u) continue;  // e.g. 32 points of masked images: nothing to fetch
            __syncwarp();                  // previous pass finished reading the mailbox
            emit_taps(taps, lane, live, g, a, lv.x, lv.y, lv.z, row_bytes, zero_off);
            __syncwarp();
            // ---- phase 2 -------------------------------------------------------------------
            gather_pass<T, D>(taps, livemask, vbase, slot, acc);
        }

        store_row<T, D>(acc, out + (((size_t)b * Lq + q) * M + m) * D, lane);
        __syncwarp();  // all lanes done with stage[buf] before it is refilled two rows later
        cur = nxt;
    }
}

// ------------------------------------------------------------------------------------
// Small rows (L*P <= kSmallLP: the ViT-Adapter's injector / extractor, 12 and 4 points per row): one THREAD per
// (output row, 16-byte channel vector).  A warp-per-row pass would leave 20-28 of its 32 point lanes idle and pay the
// staging / mailbox / barrier sequence for 4 points; here a row costs its own loads only, the index math is repeated
// by the D*sizeof(T)/16 threads of a row (cheap at <= 16 points) and latency is hidden by occupancy, not by staging.
// Same index math (point_geom, corner_valid) and fp32 opmath as the row kernel; zero-weight points skipped alike.
// ------------------------------------------------------------------------------------
constexpr int kSmallLP = 16;

template <typename T, int D>
__global__ void __launch_bounds__(256)
msda_fwd_smallrow_kernel(const T *__restrict__ value, const int64_t *__restrict__ shapes,
                         const int64_t *__restrict__ starts, const T *__restrict__ loc,
                         const T *__restrict__ attn, T *__restrict__ out,
                         long total, int S, int M, int L, int Lq, int P, unsigned flags) {
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int LPR = D / VEC;
    const bool strict = flags & MMFS_MSDA_STRICT;
    const int LP = L * P;
    const long long row_elems = (long long)M * D;
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const long row = idx / LPR;                 // (b * Lq + q) * M + m
        const int v = (int)(idx % LPR);
        const int m = (int)(row % M);
        const long b = row / ((long)M * Lq);
        const T *loc_row = loc + row * LP * 2;
        const T *att_row = attn + row * LP;
        const T *slab = value + ((size_t)b * S * M + m) * D + v * VEC;
        float acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
        int j = 0;
        for (int l = 0; l < L; ++l) {
            const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1], start = (int)starts[l];
            for (int pp = 0; pp < P; ++pp, ++j) {
                const float a = elem_to_f32(att_row + j);
                if (!strict && a == 0.f) continue;
                const PointGeom<float> g = point_geom(elem_to_f32(loc_row + 2 * j), elem_to_f32(loc_row + 2 * j + 1), H, W);
                if (!g.in_range) continue;
                const float hh = 1.f - g.lh, hw = 1.f - g.lw;
                const T *p00 = slab + (long long)(start + g.h_low * W + g.w_low) * row_elems;
                uint4 vv[4];
                float wk[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const bool ok = corner_valid(k, g.h_low, g.w_low, H, W);
                    wk[k] = ok ? ((k & 2) ? g.lh : hh) * ((k & 1) ? g.lw : hw) * a : 0.f;
                    const T *pk = p00 + ((k & 2) ? (long long)W * row_elems : 0ll) + ((k & 1) ? row_elems : 0ll);
                    vv[k] = ok ? ldg_nc_v4(pk) : make_uint4(0u, 0u, 0u, 0u);
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    float f[VEC];
                    Vec16<T>::unpack(vv[k], f);
#pragma unroll
                    for (int c = 0; c < VEC; ++c) acc[c] = fmaf(wk[k], f[c], acc[c]);
                }
            }
        }
        stg_v4(out + row * D + v * VEC, Vec16<T>::pack(acc));
    }
}

// ------------------------------------------------------------------------------------
// Generic path (any D, f64): one thread per output scalar, index math per thread.
// ------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
msda_fwd_generic_kernel(const T *__restrict__ value, const int64_t *__restrict__ shapes,
                        const int64_t *__restrict__ starts, const T *__restrict__ loc,
                        const T *__restrict__ attn, T *__restrict__ out,
                        long total, int S, int M, int D, int L, int Lq, int P, unsigned flags) {
    using OP = typename OpMath<T>::type;
    const bool strict = flags & MMFS_MSDA_STRICT;
    for (long idx = (long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long)gridDim.x * blockDim.x) {
        const int c = (int)(idx % D);
        const long qm = idx / D;
        const int m = (int)(qm % M);
        const int b = (int)(qm / M / Lq);
        const T *vb = value + ((size_t)b * S * M + m) * D + c;
        const T *locp = loc + (size_t)qm * L * P * 2;
        const T *attp = attn + (size_t)qm * L * P;
        OP col = 0;
        for (int l = 0; l < L; ++l) {
            const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1], st = (int)starts[l];
            for (int p = 0; p < P; ++p) {
                const int j = l * P + p;
                const OP x = to_op(locp[2 * j]), y = to_op(locp[2 * j + 1]), a = to_op(attp[j]);
                const PointGeom<OP> g = point_geom(x, y, H, W);
                if (!g.in_range || (!strict && a == (OP)0)) continue;
                OP val = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (!corner_valid(k, g.h_low, g.w_low, H, W)) continue;
                    const int hc = g.h_low + (k >> 1), wc = g.w_low + (k & 1);
                    const OP fh = (k & 2) ? g.lh : (OP)1 - g.lh;
                    const OP fw = (k & 1) ? g.lw : (OP)1 - g.lw;
                    val += fh * fw * to_op(vb[(size_t)(st + hc * W + wc) * M * D]);
                }
                col += val * a;
            }
        }
        out[idx] = from_op<T>(col);
    }
}

// ------------------------------------------------------------------------------------
// Index stream (parity instrumentation; same point_geom / corner_valid as above).
// ------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
msda_index_stream_kernel(const int64_t *__restrict__ shapes, const int64_t *__restrict__ starts,
                         const T *__restrict__ loc, int32_t *__restrict__ idx,
                         long total, int M, int D, int L, int P) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int p = (int)(i % P);
        const int l = (int)((i / P) % L);
        const int m = (int)((i / P / L) % M);
        (void)p;
        const int H = (int)shapes[2 * l], W = (int)shapes[2 * l + 1];
        const float x = to_op(loc[2 * i]), y = to_op(loc[2 * i + 1]);
        const PointGeom<float> g = point_geom(x, y, H, W);
        int32_t rec[8] = {0, 0, 0, 0, -1, -1, -1, -1};
        if (g.in_range) {
            rec[0] = 1; rec[1] = g.h_low; rec[2] = g.w_low;
            const int w_stride = M * D, h_stride = W * w_stride;            // cuh:50-51
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (corner_valid(k, g.h_low, g.w_low, H, W)) {
                    rec[3] |= 1 << k;
                    rec[4 + k] = (g.h_low + (k >> 1)) * h_stride + (g.w_low + (k & 1)) * w_stride + m * D;
                }
        }
        int4 *o = reinterpret_cast<int4 *>(idx + i * 8);
        o[0] = make_int4(rec[0], rec[1], rec[2], rec[3]);
        o[1] = make_int4(rec[4], rec[5], rec[6], rec[7]);
    }
}

// ------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------
template <typename T, int D>
static int launch_rows(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
                       const void *attn, void *out, int N, int S, int M, int L, int Lq, int P,
                       unsigned flags, cudaStream_t st) {
    int p_shift = -1;
    if ((P & (P - 1)) == 0) { p_shift = 0; while ((1 << p_shift) < P) ++p_shift; }
    const int LP = L * P;
    const int stage_elems = ((3 * LP * (int)sizeof(T) + 15) / 16) * 16 / (int)sizeof(T);
    const size_t smem = (size_t)L * sizeof(int4) +
                        (size_t)kWarpsPerCta * (16 + 2 * (size_t)stage_elems * sizeof(T) + kTapsPerWarp * sizeof(Tap));
    if (smem > 200 * 1024) { set_error("msda: L*P = %d too large for the staging buffers", LP); return MMFS_EUNSUPPORTED; }
    constexpr auto kern = msda_fwd_rows_kernel<T, D>;
    int rc = ensure_dynamic_smem<kern>(smem);
    if (rc != MMFS_OK) return rc;
    // rows per warp per tile: short tiles -- neighbouring q-tiles of one head still share the L1-resident value slab
    // through the per-SM tile swizzle, and short tiles balance the tail of the persistent grid.  Tiny problems
    // (decode, Lq = 1) use 1.
    RowWalkPlan w;
    if ((rc = plan_row_walk(kern, smem, (long)N * M, Lq, 2, "msda", w)) != MMFS_OK) return rc;
    const bool bulk_ok = ((uintptr_t)loc % 16 == 0) && ((uintptr_t)attn % 16 == 0) &&
                         ((2 * LP * sizeof(T)) % 16 == 0) && ((LP * sizeof(T)) % 16 == 0);
    kern<<<w.grid, 32 * kWarpsPerCta, smem, st>>>(
        (const T *)value, shapes, starts, (const T *)loc, (const T *)attn, (T *)out, S, M, L, Lq, P, p_shift, flags,
        w.rows_per_warp, w.qtiles, w.ntiles, w.ctas_per_sm, w.nsm, stage_elems, bulk_ok ? 1 : 0);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_generic(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
                          const void *attn, void *out, int N, int S, int M, int D, int L, int Lq, int P,
                          unsigned flags, cudaStream_t st) {
    const long total = (long)N * Lq * M * D;
    const int grid = capped_grid((total + 255) / 256, 32);
    msda_fwd_generic_kernel<T><<<grid, 256, 0, st>>>((const T *)value, shapes, starts, (const T *)loc,
                                                       (const T *)attn, (T *)out, total, S, M, D, L, Lq, P, flags);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int dispatch_d(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
                      const void *attn, void *out, int N, int S, int M, int D, int L, int Lq, int P,
                      unsigned flags, cudaStream_t st) {
#define MMFS_CASE(DD) \
    case DD: return launch_rows<T, DD>(value, shapes, starts, loc, attn, out, N, S, M, L, Lq, P, flags, st);
    const bool aligned16 = ((uintptr_t)value % 16 == 0) && ((uintptr_t)out % 16 == 0);
    if (aligned16 && L * P <= kSmallLP && (D == 32 || D == 64 || D == 128)) {
        constexpr int VEC = 16 / (int)sizeof(T);
        const long total = (long)N * Lq * M * (D / VEC);
        const int grid = capped_grid((total + 255) / 256, 64);
        if (D == 32)
            msda_fwd_smallrow_kernel<T, 32><<<grid, 256, 0, st>>>((const T *)value, shapes, starts, (const T *)loc, (const T *)attn, (T *)out, total, S, M, L, Lq, P, flags);
        else if (D == 64)
            msda_fwd_smallrow_kernel<T, 64><<<grid, 256, 0, st>>>((const T *)value, shapes, starts, (const T *)loc, (const T *)attn, (T *)out, total, S, M, L, Lq, P, flags);
        else
            msda_fwd_smallrow_kernel<T, 128><<<grid, 256, 0, st>>>((const T *)value, shapes, starts, (const T *)loc, (const T *)attn, (T *)out, total, S, M, L, Lq, P, flags);
        MMFS_CUDA(cudaGetLastError());
        return MMFS_OK;
    }
    if (aligned16) {
        switch (D) {
            MMFS_CASE(32)
            MMFS_CASE(64)
            MMFS_CASE(128)
            default: break;
        }
    }
#undef MMFS_CASE
    return launch_generic<T>(value, shapes, starts, loc, attn, out, N, S, M, D, L, Lq, P, flags, st);
}

}  // namespace mmfs

using namespace mmfs;

static int check_msda_args(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
                           const void *attn, const void *out, int N, int S, int M, int D, int L, int Lq, int P, int dtype) {
    MMFS_CHECK_ARG(N >= 0 && Lq >= 0, "msda: negative batch (%d) or query count (%d)", N, Lq);
    MMFS_CHECK_ARG(S > 0 && M > 0 && D > 0 && L > 0 && P > 0,
                   "msda: non-positive dimension S=%d M=%d D=%d L=%d P=%d", S, M, D, L, P);
    MMFS_CHECK_ARG(dtype_size(dtype) != 0, "msda: unknown dtype code %d", dtype);
    if (N == 0 || Lq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value && shapes && starts && loc && attn && out, "msda: null pointer argument");
    if ((long)S * M * D >= (1L << 31) || (long)Lq * M * L * P * 2 >= (1L << 31) * 64L) {
        set_error("msda: per-batch slab too large for 32-bit row offsets (S=%d M=%d D=%d)", S, M, D);
        return MMFS_EUNSUPPORTED;
    }
    return MMFS_OK;
}

extern "C" int mmfs_msda_forward(const void *value, const int64_t *shapes, const int64_t *starts,
                                 const void *loc, const void *attn, void *out,
                                 int N, int S, int M, int D, int L, int Lq, int P,
                                 int dtype, unsigned flags, void *stream) {
    int rc = check_msda_args(value, shapes, starts, loc, attn, out, N, S, M, D, L, Lq, P, dtype);
    if (rc != MMFS_OK || N == 0 || Lq == 0) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kAllTypes>(dtype, "msda", [&](auto tag) {
        using T = typename decltype(tag)::type;
        if constexpr (std::is_same_v<T, double>)   // f64 has only the generic kernel
            return launch_generic<T>(value, shapes, starts, loc, attn, out, N, S, M, D, L, Lq, P, flags, st);
        else
            return dispatch_d<T>(value, shapes, starts, loc, attn, out, N, S, M, D, L, Lq, P, flags, st);
    });
}

extern "C" int mmfs_msda_index_stream(const int64_t *shapes, const int64_t *starts, const void *loc,
                                      int32_t *idx, int N, int M, int D, int L, int Lq, int P,
                                      int dtype, void *stream) {
    MMFS_CHECK_ARG(N >= 0 && Lq >= 0 && M > 0 && D > 0 && L > 0 && P > 0, "msda_index_stream: bad dimension");
    MMFS_CHECK_ARG(dtype == MMFS_F32 || dtype == MMFS_F16 || dtype == MMFS_BF16,
                   "msda_index_stream: dtype %d not supported (f32/f16/bf16 only)", dtype);
    const long total = (long)N * Lq * M * L * P;
    if (total == 0) return MMFS_OK;
    MMFS_CHECK_ARG(shapes && starts && loc && idx, "msda_index_stream: null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = capped_grid((total + 255) / 256, 32);
    return dispatch_dtype<kF32Types>(dtype, "msda_index_stream", [&](auto tag) {
        using T = typename decltype(tag)::type;
        msda_index_stream_kernel<T><<<grid, 256, 0, st>>>(shapes, starts, (const T *)loc, idx, total, M, D, L, P);
        MMFS_CUDA(cudaGetLastError());
        return MMFS_OK;
    });
}
