// msda_bwd_sm100.cu -- multi-scale deformable attention BACKWARD for sm_90a (training path; SURVEY.md 8f rank 4).
//
// Replaces ms_deform_attn_cuda_backward (ops/src/cuda/ms_deform_attn_cuda.cu:84-166) and the nine col2im kernels
// of ops/src/cuda/ms_deform_im2col_cuda.cuh:304-923 (+ launcher :959-1330) with ONE kernel that reuses the forward's
// machinery (sampler_common.cuh): a warp per (b, q, m) row, index math once per point, 16-byte gathers.
//   grad_value        scatter of go[c] * (lerp_k * a).  Two flavours:
//                     * DETERMINISTIC (mmfs_msda_backward_deterministic, the Python default): every contribution is
//                       converted to 64-bit fixed point (scale 2^(40 - ceil(log2 max|grad_out|)), exact power of two) and
//                       added with INTEGER atomics (red.global.add.u64) -- integer addition is associative, so the result
//                       does not depend on the order in which taps arrive and two runs are bit-identical; a final pass
//                       converts to fp32 with one rounding.  |contribution| < 2^40 and < 2^20 taps can meet in one pixel
//                       of one head, so the sum stays far inside int64.
//                     * red.global.add.v4.f32 into an fp32 buffer (mmfs_msda_backward) -- like the reference's atomicAdd
//                       (cuh:128-155): summation order, hence the last bits, vary from run to run.
//                     The reference too accumulates half inputs in fp32 and casts back (cu:122-129, 156-160; done by the
//                     Python shim here).
//   grad_sampling_loc one writer per (b,q,m,l,p): a*W*(-hh d1 + hh d2 - lh d3 + lh d4), a*H*(-hw d1 - lw d2 + hw d3 + lw d4)
//   grad_attn_weight  one writer: sum_k lerp_k d_k         with d_k = <grad_out row, value row of corner k> (cuh:90-162)
// The channel dot products d_k are reduced with warp shuffles inside each slot and handed to the point's lane
// through shared memory; no block-size-specialised reduction variants are needed.
#include "sampler_common.cuh"

namespace mmfs {

__device__ __forceinline__ void red_add_v4(float *addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_fixed(long long *addr, float x, float scale) {
    const long long q = __float2ll_rn(x * scale);          // scale is a power of two: x * scale is exact
    asm volatile("red.global.add.u64 [%0], %1;" ::"l"(addr), "l"(q) : "memory");
}
constexpr int kFixedBits = 40;

// max |grad_out| (order-independent: unsigned max on the bit patterns of non-negative floats), then the two powers of two
__global__ void absmax_kernel(const void *__restrict__ x, long n, int dtype, unsigned *__restrict__ out) {
    float m = 0.f;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float v;
        if (dtype == MMFS_F32) v = static_cast<const float *>(x)[i];
        else if (dtype == MMFS_F16) v = __half2float(static_cast<const __half *>(x)[i]);
        else v = __bfloat162float(static_cast<const __nv_bfloat16 *>(x)[i]);
        v = fabsf(v);
        if (v == v && v < INFINITY) m = fmaxf(m, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}
__global__ void fixed_scale_kernel(float *scratch) {   // scratch[0] = max|go| (in) -> scale; scratch[1] = 1 / scale
    const float amax = scratch[0];
    int e = 0;
    if (amax > 0.f) { frexpf(amax, &e); }               // amax = f * 2^e, f in [0.5, 1)  =>  amax < 2^e
    scratch[0] = ldexpf(1.f, kFixedBits - e);
    scratch[1] = ldexpf(1.f, e - kFixedBits);
}
__global__ void fixed_to_float_kernel(const long long *__restrict__ fx, float *__restrict__ out, long n, const float *scratch) {
    const double inv = (double)scratch[1];
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        out[i] = (float)((double)fx[i] * inv);
}

constexpr int kDotStride = 33;

template <typename T, int D, bool DET>
__global__ void __launch_bounds__(32 * kWarpsPerCta, 3)
msda_bwd_rows_kernel(const T *__restrict__ value, const int64_t *__restrict__ shapes, const int64_t *__restrict__ starts,
                     const T *__restrict__ loc, const T *__restrict__ attn, const T *__restrict__ grad_out,
                     void *__restrict__ grad_value_any, float *__restrict__ grad_loc, float *__restrict__ grad_attn,
                     const float *__restrict__ fixed_scale,
                     int S, int M, int L, int Lq, int P, int p_shift, int rows_per_warp, int qtiles, long ntiles,
                     int ctas_per_sm, int nsm) {
    float *grad_value = static_cast<float *>(grad_value_any);            // fp32 buffer (DET = false)
    long long *grad_fixed = static_cast<long long *>(grad_value_any);    // int64 fixed-point buffer (DET = true)
    const float fscale = DET ? fixed_scale[0] : 1.f;
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int LPR = D / VEC;
    constexpr int RPI = 32 / LPR;
    constexpr int NIT = 128 / RPI;
    extern __shared__ int4 s_dyn[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int4 *s_lvl = s_dyn;
    const int per_warp_bytes = kTapsPerWarp * (int)sizeof(Tap) + 4 * kDotStride * 4 + 16;
    char *wbase = reinterpret_cast<char *>(s_dyn + L) + warp * (((per_warp_bytes + 15) / 16) * 16);
    Tap *taps = reinterpret_cast<Tap *>(wbase);
    float *dots = reinterpret_cast<float *>(wbase + kTapsPerWarp * sizeof(Tap));   // [corner][point] skewed
    for (int l = threadIdx.x; l < L; l += blockDim.x)
        s_lvl[l] = make_int4((int)shapes[2 * l], (int)shapes[2 * l + 1], (int)starts[l], 0);
    __syncthreads();

    const int LP = L * P;
    const long long row_bytes = (long long)M * D * (int)sizeof(T);
    const int slot = lane / LPR, sub = lane % LPR;
    RowWalk walk;
    walk.itiles = (int)ntiles; walk.igrid = (int)gridDim.x; walk.qtiles = qtiles; walk.M = M; walk.Lq = Lq;
    walk.rows_per_warp = rows_per_warp; walk.warp = warp;

    for (RowCursor cur = walk.first(ctas_per_sm, nsm, 1); cur.ok; cur = walk.next(cur)) {
        const int b = cur.b, m = cur.m, q = cur.q;
        const size_t qm = ((size_t)b * Lq + q) * M + m;
        const T *locp = loc + qm * (size_t)LP * 2;
        const T *attp = attn + qm * (size_t)LP;
        const char *slab = reinterpret_cast<const char *>(value + ((size_t)b * S * M + m) * D);
        const char *vbase = slab + sub * 16;
        const size_t gv_off = ((size_t)b * S * M + m) * D + sub * VEC;           // element offset into the twin of the value slab
        const long long zero_off = reinterpret_cast<const char *>(g_zero_row) - slab;
        float go[VEC];   // this lane's channels of the incoming gradient row (same for every slot)
        Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(grad_out + qm * D + sub * VEC), go);

        for (int p0 = 0; p0 < LP; p0 += 32) {
            const int j = p0 + lane;
            bool live = false;
            PointGeom<float> g;
            g.in_range = false; g.h_low = g.w_low = 0; g.lh = g.lw = 0.f;
            float a = 0.f;
            int4 lv = make_int4(1, 1, 0, 0);
            if (j < LP) {
                a = to_op(attp[j]);
                const float x = to_op(locp[2 * j]), y = to_op(locp[2 * j + 1]);
                lv = s_lvl[(p_shift >= 0) ? (j >> p_shift) : (j / P)];
                g = point_geom(x, y, lv.x, lv.y);
                live = g.in_range;
            }
            const unsigned livemask = __ballot_sync(0xffffffffu, live);
            __syncwarp();
            if (livemask != 0u) {
                emit_taps(taps, lane, live, g, a, lv.x, lv.y, lv.z, row_bytes, zero_off);
#pragma unroll
                for (int k = 0; k < 4; ++k) dots[k * kDotStride + lane] = 0.f;
                __syncwarp();
#pragma unroll 4
                for (int it = 0; it < NIT; ++it) {
                    const int tix = it * RPI + slot;              // tap = point * 4 + corner
                    const int pt = tix >> 2, corner = tix & 3;
                    if (((livemask >> pt) & 1u) == 0u && RPI <= 4) continue;   // whole instruction dead (RPI <= 4: one point)
                    Tap t;
                    *reinterpret_cast<uint4 *>(&t) = *reinterpret_cast<const uint4 *>(&taps[corner * kTapStride + pt]);
                    const bool hit = t.off != zero_off;           // fetched corner of a live point
                    float f[VEC];
                    Vec16<T>::unpack(ldg_nc_v4(vbase + t.off), f);
                    float d = 0.f;
#pragma unroll
                    for (int k = 0; k < VEC; ++k) d = fmaf(go[k], f[k], d);
#pragma unroll
                    for (int o = 1; o < LPR; o <<= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
                    if (hit) {
                        const size_t e0 = gv_off + (size_t)(t.off / (long long)sizeof(T));
                        if (DET) {
#pragma unroll
                            for (int k = 0; k < VEC; ++k) red_add_fixed(grad_fixed + e0 + k, go[k] * t.w0, fscale);
                        } else {
#pragma unroll
                            for (int k = 0; k < VEC; k += 4)
                                red_add_v4(grad_value + e0 + k, go[k] * t.w0, go[k + 1] * t.w0, go[k + 2] * t.w0, go[k + 3] * t.w0);
                        }
                        if (sub == 0) dots[corner * kDotStride + pt] = d;
                    }
                }
                __syncwarp();
            }
            // ---- per-point gradients (lane = point) ----------------------------------------
            if (j < LP) {
                float gx = 0.f, gy = 0.f, gw = 0.f;
                if (live) {
                    const float d1 = dots[0 * kDotStride + lane], d2 = dots[1 * kDotStride + lane];
                    const float d3 = dots[2 * kDotStride + lane], d4 = dots[3 * kDotStride + lane];
                    const float lh = g.lh, lw = g.lw, hh = 1.f - lh, hw = 1.f - lw;
                    gw = hh * hw * d1 + hh * lw * d2 + lh * hw * d3 + lh * lw * d4;            // cuh:150-156
                    gx = (float)lv.y * a * (-hh * d1 + hh * d2 - lh * d3 + lh * d4);              // width  * grad_w_weight
                    gy = (float)lv.x * a * (-hw * d1 - lw * d2 + hw * d3 + lw * d4);              // height * grad_h_weight
                }
                grad_attn[qm * LP + j] = gw;
                grad_loc[(qm * LP + j) * 2] = gx;
                grad_loc[(qm * LP + j) * 2 + 1] = gy;
            }
            __syncwarp();
        }
    }
}

template <typename T, int D, bool DET>
static int launch_bwd_impl(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc, const void *attn,
                           const void *grad_out, void *gv, float *gl, float *ga, const float *fixed_scale, int N, int S, int M,
                           int L, int Lq, int P, cudaStream_t st) {
    int p_shift = -1;
    if ((P & (P - 1)) == 0) { p_shift = 0; while ((1 << p_shift) < P) ++p_shift; }
    const size_t per_warp = ((kTapsPerWarp * sizeof(Tap) + 4 * kDotStride * 4 + 16 + 15) / 16) * 16;
    const size_t smem = (size_t)L * sizeof(int4) + kWarpsPerCta * per_warp;
    auto kern = msda_bwd_rows_kernel<T, D, DET>;
    if (smem > 48 * 1024) MMFS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int ctas = 0;
    MMFS_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kern, 32 * kWarpsPerCta, smem));
    if (ctas < 1) { set_error("msda_backward: kernel does not fit"); return MMFS_EUNSUPPORTED; }
    const int nsm = num_sms();
    int rpw = 8;
    while (rpw > 1 && (long)N * M * ((Lq + kWarpsPerCta * rpw - 1) / (kWarpsPerCta * rpw)) < 2L * nsm * ctas) rpw >>= 1;
    const int qtiles = (Lq + kWarpsPerCta * rpw - 1) / (kWarpsPerCta * rpw);
    const long ntiles = (long)N * M * qtiles;
    if (ntiles > 0x3fffffffL) { set_error("msda_backward: too many tiles"); return MMFS_EUNSUPPORTED; }
    const long full = (long)nsm * ctas;
    kern<<<(unsigned)(ntiles < full ? ntiles : full), 32 * kWarpsPerCta, smem, st>>>(
        (const T *)value, shapes, starts, (const T *)loc, (const T *)attn, (const T *)grad_out, gv, gl, ga, fixed_scale,
        S, M, L, Lq, P, p_shift, rpw, qtiles, ntiles, ctas, nsm);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T, int D>
static int launch_bwd(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc, const void *attn,
                      const void *grad_out, void *gv, float *gl, float *ga, const float *fixed_scale, int N, int S, int M,
                      int L, int Lq, int P, cudaStream_t st) {
    if (fixed_scale != nullptr)
        return launch_bwd_impl<T, D, true>(value, shapes, starts, loc, attn, grad_out, gv, gl, ga, fixed_scale, N, S, M, L, Lq, P, st);
    return launch_bwd_impl<T, D, false>(value, shapes, starts, loc, attn, grad_out, gv, gl, ga, nullptr, N, S, M, L, Lq, P, st);
}

template <typename T>
static int dispatch_bwd(int D, const void *value, const int64_t *shapes, const int64_t *starts, const void *loc, const void *attn,
                        const void *grad_out, void *gv, float *gl, float *ga, const float *fs, int N, int S, int M, int L, int Lq, int P,
                        cudaStream_t st) {
    switch (D) {
        case 32: return launch_bwd<T, 32>(value, shapes, starts, loc, attn, grad_out, gv, gl, ga, fs, N, S, M, L, Lq, P, st);
        case 64: return launch_bwd<T, 64>(value, shapes, starts, loc, attn, grad_out, gv, gl, ga, fs, N, S, M, L, Lq, P, st);
        case 128: return launch_bwd<T, 128>(value, shapes, starts, loc, attn, grad_out, gv, gl, ga, fs, N, S, M, L, Lq, P, st);
        default: set_error("msda_backward: head size %d unsupported (32/64/128)", D); return MMFS_EUNSUPPORTED;
    }
}

}  // namespace mmfs

using namespace mmfs;

static int backward_entry(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc, const void *attn,
                          const void *grad_out, void *grad_value, float *grad_loc, float *grad_attn, const float *fixed_scale,
                          int N, int S, int M, int D, int L, int Lq, int P, int dtype, cudaStream_t st) {
    switch (dtype) {
        case MMFS_F32: return dispatch_bwd<float>(D, value, shapes, starts, loc, attn, grad_out, grad_value, grad_loc, grad_attn, fixed_scale, N, S, M, L, Lq, P, st);
        case MMFS_F16: return dispatch_bwd<__half>(D, value, shapes, starts, loc, attn, grad_out, grad_value, grad_loc, grad_attn, fixed_scale, N, S, M, L, Lq, P, st);
        case MMFS_BF16: return dispatch_bwd<__nv_bfloat16>(D, value, shapes, starts, loc, attn, grad_out, grad_value, grad_loc, grad_attn, fixed_scale, N, S, M, L, Lq, P, st);
        default: set_error("msda_backward: dtype %d unsupported (f32/f16/bf16)", dtype); return MMFS_EUNSUPPORTED;
    }
}

extern "C" int mmfs_msda_backward(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
                                  const void *attn, const void *grad_out, float *grad_value, float *grad_loc,
                                  float *grad_attn, int N, int S, int M, int D, int L, int Lq, int P, int dtype, void *stream) {
    MMFS_CHECK_ARG(N >= 0 && Lq >= 0 && S > 0 && M > 0 && D > 0 && L > 0 && P > 0, "msda_backward: bad dimension");
    if (N == 0 || Lq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value && shapes && starts && loc && attn && grad_out && grad_value && grad_loc && grad_attn,
                   "msda_backward: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)value | (uintptr_t)grad_out | (uintptr_t)grad_value) % 16 == 0, "msda_backward: 16-byte alignment required");
    return backward_entry(value, shapes, starts, loc, attn, grad_out, grad_value, grad_loc, grad_attn, nullptr,
                          N, S, M, D, L, Lq, P, dtype, (cudaStream_t)stream);
}

extern "C" int mmfs_msda_backward_deterministic(const void *value, const int64_t *shapes, const int64_t *starts, const void *loc,
                                                const void *attn, const void *grad_out, long long *grad_value_fixed,
                                                float *grad_value, float *grad_loc, float *grad_attn, float *scratch2,
                                                int N, int S, int M, int D, int L, int Lq, int P, int dtype, void *stream) {
    MMFS_CHECK_ARG(N >= 0 && Lq >= 0 && S > 0 && M > 0 && D > 0 && L > 0 && P > 0, "msda_backward_deterministic: bad dimension");
    if (N == 0 || Lq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value && shapes && starts && loc && attn && grad_out && grad_value_fixed && grad_value && grad_loc && grad_attn && scratch2,
                   "msda_backward_deterministic: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)value | (uintptr_t)grad_out | (uintptr_t)grad_value_fixed) % 16 == 0, "msda_backward_deterministic: 16-byte alignment required");
    MMFS_CHECK_ARG(dtype == MMFS_F32 || dtype == MMFS_F16 || dtype == MMFS_BF16, "msda_backward_deterministic: dtype %d unsupported", dtype);
    cudaStream_t st = (cudaStream_t)stream;
    const long n_go = (long)N * Lq * M * D, n_gv = (long)N * S * M * D;
    MMFS_CUDA(cudaMemsetAsync(scratch2, 0, 2 * sizeof(float), st));
    absmax_kernel<<<(unsigned)((n_go + 1023) / 1024 < 1184 ? (n_go + 1023) / 1024 : 1184), 256, 0, st>>>(grad_out, n_go, dtype, reinterpret_cast<unsigned *>(scratch2));
    fixed_scale_kernel<<<1, 1, 0, st>>>(scratch2);
    const int rc = backward_entry(value, shapes, starts, loc, attn, grad_out, grad_value_fixed, grad_loc, grad_attn, scratch2,
                                  N, S, M, D, L, Lq, P, dtype, st);
    if (rc != MMFS_OK) return rc;
    fixed_to_float_kernel<<<(unsigned)((n_gv + 1023) / 1024 < 2368 ? (n_gv + 1023) / 1024 : 2368), 256, 0, st>>>(grad_value_fixed, grad_value, n_gv, scratch2);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}
