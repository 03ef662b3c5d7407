// vit_bwd_sm100.cu -- backward kernels of the visual tokenizer's encoder (training path, 16-bit tensors, fp32 math).
//
//   mmfs_quick_gelu_backward       d/dh of h * sigmoid(1.702 h), CLIPMLP's activation (quick_gelu)
//   mmfs_resize_bilinear_backward  d/dx of F.interpolate(x, scale_factor=s, mode="bilinear", align_corners=False),
//                                  the ViT-Adapter's output resizes (vit_adapter_hf.py:150-152)
//
// Both are bandwidth kernels without atomics: each output element is computed by one thread in a fixed order and
// rounded once at the store, so two runs are bit-identical.
#include "common.cuh"

namespace mmfs {

// ---- quick-GELU backward: y = h * s, s = sigmoid(1.702 h)  ->  dh = dy * (s + 1.702 h s (1 - s)) -----------------------
__device__ __forceinline__ float quick_gelu_grad(float h, float dy) {
    const float s = 1.f / (1.f + expf(-1.702f * h));
    return dy * fmaf(1.702f * h * s, 1.f - s, s);
}

template <typename T>
__global__ void __launch_bounds__(256) quick_gelu_bwd_kernel(const T *__restrict__ h, const T *__restrict__ dy,
                                                             T *__restrict__ dh, long n) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const long nvec = n / VEC;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
        float a[VEC], d[VEC], o[VEC];
        Vec16<T>::unpack(ldg_nc_v4(h + i * VEC), a);
        Vec16<T>::unpack(ldg_nc_v4(dy + i * VEC), d);
#pragma unroll
        for (int k = 0; k < VEC; ++k) o[k] = quick_gelu_grad(a[k], d[k]);
        stg_v4(dh + i * VEC, Vec16<T>::pack(o));
    }
    for (long i = nvec * VEC + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)   // scalar tail
        dh[i] = from_op<T>(quick_gelu_grad(to_op(h[i]), to_op(dy[i])));
}

// ---- bilinear resize backward (gather form) ------------------------------------------------------------------------
// Source index of output index o along one axis, as PyTorch's upsample_bilinear2d computes it with align_corners=False
// and a given scale factor (area_pixel_compute_source_index, accumulation type float): r = max(scale * (o + 0.5) - 0.5,
// 0), i0 = (int)r, i1 = i0 + (i0 < in - 1), weights 1 - (r - i0) on i0 and r - i0 on i1 (i1 == i0 at the far edge).
// `scale` is 1 / scale_factor.
__device__ __forceinline__ float src_weight(int o, int i, float scale, int in) {
    float r = scale * ((float)o + 0.5f) - 0.5f;
    r = r < 0.f ? 0.f : r;
    const int i0 = (int)r;
    const int i1 = i0 + (i0 < in - 1 ? 1 : 0);
    const float l1 = r - (float)i0;
    return (i0 == i ? 1.f - l1 : 0.f) + (i1 == i ? l1 : 0.f);
}

// Output indices that can sample input index i: those with floor(r) in {i - 1, i}, widened by one on each side (the
// exact test is src_weight != 0).
__device__ __forceinline__ void out_range(int i, float scale, int out, int &lo, int &hi) {
    lo = max(0, (int)floorf(((float)i - 0.5f) / scale - 0.5f) - 1);
    hi = min(out - 1, (int)ceilf(((float)i + 1.5f) / scale - 0.5f) + 1);
}

// One thread per (image, input pixel, 8 channels): sums w_y * w_x * dy over the output pixels that sample the input
// pixel, rows then columns in increasing order, in fp32, and stores 8 channels of dx (B, Hin * Win, C) with one 16-byte
// store.  dy element (b, c, p) (p = oy * Wout + ox) is at dy[b * dy_bs + c * dy_cs + p * dy_ps]; kVec: dy_cs == 1 with
// 16-byte aligned pixels, read as one 16-byte vector.
template <typename T, bool kVec>
__global__ void __launch_bounds__(256) resize_bilinear_bwd_kernel(const T *__restrict__ dy, T *__restrict__ dx, int B,
                                                                  int C, int Hin, int Win, int Hout, int Wout, long dy_bs,
                                                                  long dy_cs, long dy_ps, float scale_h, float scale_w) {
    constexpr int VEC = 8;
    const int cg = C / VEC;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)B * Hin * Win * cg) return;
    const int c0 = (int)(t % cg) * VEC;
    const long pix = t / cg;
    const int ix = (int)(pix % Win), iy = (int)(pix / Win % Hin), b = (int)(pix / ((long)Win * Hin));
    int y_lo, y_hi, x_lo, x_hi;
    out_range(iy, scale_h, Hout, y_lo, y_hi);
    out_range(ix, scale_w, Wout, x_lo, x_hi);
    const T *base = dy + b * dy_bs + c0 * dy_cs;
    float acc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.f;
    for (int oy = y_lo; oy <= y_hi; ++oy) {
        const float wy = src_weight(oy, iy, scale_h, Hin);
        if (wy == 0.f) continue;
        float row[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) row[k] = 0.f;
        for (int ox = x_lo; ox <= x_hi; ++ox) {
            const float wx = src_weight(ox, ix, scale_w, Win);
            if (wx == 0.f) continue;
            const T *p = base + ((long)oy * Wout + ox) * dy_ps;
            float v[VEC];
            if constexpr (kVec) {
                Vec16<T>::unpack(ldg_nc_v4(p), v);
            } else {
#pragma unroll
                for (int k = 0; k < VEC; ++k) v[k] = to_op(p[k * dy_cs]);
            }
#pragma unroll
            for (int k = 0; k < VEC; ++k) row[k] = fmaf(wx, v[k], row[k]);
        }
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = fmaf(wy, row[k], acc[k]);
    }
    stg_v4(dx + pix * C + c0, Vec16<T>::pack(acc));
}

template <typename T>
static int launch_quick_gelu_bwd(const void *h, const void *dy, void *dh, long n, cudaStream_t st) {
    const long vecs = n / (16 / (long)sizeof(T)) + 1;
    quick_gelu_bwd_kernel<T><<<capped_grid((vecs + 255) / 256, 8), 256, 0, st>>>((const T *)h, (const T *)dy, (T *)dh, n);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_resize_bwd(const void *dy, void *dx, int B, int C, int Hin, int Win, int Hout, int Wout, long dy_bs,
                             long dy_cs, long dy_ps, float scale_h, float scale_w, bool vec, cudaStream_t st) {
    const long threads = (long)B * Hin * Win * (C / 8);
    const unsigned grid = (unsigned)((threads + 255) / 256);
    if (vec)
        resize_bilinear_bwd_kernel<T, true><<<grid, 256, 0, st>>>((const T *)dy, (T *)dx, B, C, Hin, Win, Hout, Wout, dy_bs,
                                                                   dy_cs, dy_ps, scale_h, scale_w);
    else
        resize_bilinear_bwd_kernel<T, false><<<grid, 256, 0, st>>>((const T *)dy, (T *)dx, B, C, Hin, Win, Hout, Wout, dy_bs,
                                                                    dy_cs, dy_ps, scale_h, scale_w);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_quick_gelu_backward(const void *h, const void *dy, void *dh, long n, int dtype, void *stream) {
    MMFS_CHECK_ARG(n >= 0, "quick_gelu_backward: bad shape");
    if (n == 0) return MMFS_OK;
    MMFS_CHECK_ARG(h && dy && dh, "quick_gelu_backward: null pointer argument");
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16) || ((uintptr_t)h | (uintptr_t)dy | (uintptr_t)dh) % 16 != 0) {
        set_error("quick_gelu_backward: needs bf16 / f16 and 16-byte aligned pointers (got dtype=%d)", dtype);
        return MMFS_EUNSUPPORTED;
    }
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "quick_gelu_backward", [&](auto tag) {
        return launch_quick_gelu_bwd<typename decltype(tag)::type>(h, dy, dh, n, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_resize_bilinear_backward(const void *dy, void *dx, int B, int C, int Hin, int Win, int Hout, int Wout,
                                             long dy_bs, long dy_cs, long dy_ps, float scale_h, float scale_w, int dtype,
                                             void *stream) {
    MMFS_CHECK_ARG(B >= 0 && C > 0 && Hin > 0 && Win > 0 && Hout > 0 && Wout > 0 && scale_h > 0.f && scale_w > 0.f,
                   "resize_bilinear_backward: bad shape");
    if (B == 0) return MMFS_OK;
    MMFS_CHECK_ARG(dy && dx, "resize_bilinear_backward: null pointer argument");
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16) || C % 8 != 0 || (uintptr_t)dx % 16 != 0) {
        set_error("resize_bilinear_backward: needs bf16 / f16, C %% 8 == 0 and a 16-byte aligned dx (got C=%d dtype=%d)", C,
                  dtype);
        return MMFS_EUNSUPPORTED;
    }
    const bool vec = dy_cs == 1 && (uintptr_t)dy % 16 == 0 && dy_bs % 8 == 0 && dy_ps % 8 == 0;
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "resize_bilinear_backward", [&](auto tag) {
        return launch_resize_bwd<typename decltype(tag)::type>(dy, dx, B, C, Hin, Win, Hout, Wout, dy_bs, dy_cs, dy_ps,
                                                               scale_h, scale_w, vec, (cudaStream_t)stream);
    });
}
