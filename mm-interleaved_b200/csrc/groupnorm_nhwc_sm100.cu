// groupnorm_nhwc_sm100.cu -- GroupNorm (+ optional SiLU) on NHWC activations, the normalisation in front of every
// UNet convolution of the denoise step (diffusers ResnetBlock2D / Transformer2DModel / conv_norm_out, called from
// the reference's patched forward, utils/monkey_patch/sd_unet_forward_monkey_patch.py:235-366).
//
// Why it exists: torch's CUDA group_norm always returns an NCHW tensor, so a channels-last UNet pays a layout
// round trip around every convolution; this kernel keeps the activations NHWC for the implicit-GEMM convolution
// (conv_igemm_sm100.cu) and folds the SiLU in.  Pure bandwidth work: two passes (statistics, apply), the second
// one hitting L2 for the map sizes of SD (<= 42 MB per tensor at batch 16).
//
// Thread mapping (both kernels): thread t owns the 16-byte channel vector t % (C/VEC) of every k-th pixel, so the
// per-channel scale/shift (apply) and the partial sums (statistics) live in registers and consecutive threads
// read consecutive 16-byte vectors of a pixel row (coalesced).  Statistics are fp32 sum / sum-of-squares, reduced
// in a fixed order (no atomics: results are reproducible run to run); the bf16 pipeline's rounding points
// (norm -> T, silu -> T) are kept so a bf16 run tracks diffusers' bf16 run.
#include "common.cuh"

namespace mmfs {

template <typename T> __device__ __forceinline__ float gn_rnd(float x) { return to_op(from_op<T>(x)); }
template <> __device__ __forceinline__ float gn_rnd<float>(float x) { return x; }

constexpr int kGnMaxChunks = 64;     // pixel chunks per image: the partial-statistics scratch is (B, kGnMaxChunks, G, 2) floats

// Pass 1: per (image, pixel chunk) partial sum / sum of squares of every group, written (not accumulated) to
// partial[b][chunk][g][0..1].  All reductions run in a fixed order -- registers over a thread's pixels, shared memory
// over the pixel lanes of a channel, then over the channels of a group -- so the result is bit-reproducible run to run
// (the first version used shared + global float atomics, whose order is not).
template <typename T>
__global__ void __launch_bounds__(1024) gn_stats_kernel(const T *__restrict__ x, float *__restrict__ partial, int HW, int C,
                                                         int G, int ppb, int cvecs, int lanes) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dyn[];                     // [lanes][C][2] thread partials, then [C][2] channel sums in place of lane 0
    const int b = blockIdx.y, p0 = blockIdx.x * ppb, p1 = min(HW, p0 + ppb);
    const int cv = threadIdx.x % cvecs, pl = threadIdx.x / cvecs;
    float s[VEC], ss[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) s[k] = ss[k] = 0.f;
    const T *base = x + ((size_t)b * HW) * C + (size_t)cv * VEC;
    if (pl < lanes) {
        int p = p0 + pl;
        for (; p + 3 * lanes < p1; p += 4 * lanes) {     // four independent 16-byte loads in flight
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = ldg_nc_v4(base + (size_t)(p + u * lanes) * C);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float f[VEC];
                Vec16<T>::unpack(v[u], f);
#pragma unroll
                for (int k = 0; k < VEC; ++k) { s[k] += f[k]; ss[k] = fmaf(f[k], f[k], ss[k]); }
            }
        }
        for (; p < p1; p += lanes) {
            float f[VEC];
            Vec16<T>::unpack(ldg_nc_v4(base + (size_t)p * C), f);
#pragma unroll
            for (int k = 0; k < VEC; ++k) { s[k] += f[k]; ss[k] = fmaf(f[k], f[k], ss[k]); }
        }
        float *mine = s_dyn + ((size_t)pl * C + (size_t)cv * VEC) * 2;
#pragma unroll
        for (int k = 0; k < VEC; ++k) { mine[2 * k] = s[k]; mine[2 * k + 1] = ss[k]; }
    }
    __syncthreads();
    if (pl == 0) {                                       // channel totals over the pixel lanes, lane order
        for (int l = 1; l < lanes; ++l) {
            const float *o = s_dyn + ((size_t)l * C + (size_t)cv * VEC) * 2;
#pragma unroll
            for (int k = 0; k < VEC; ++k) { s[k] += o[2 * k]; ss[k] += o[2 * k + 1]; }
        }
        float *mine = s_dyn + (size_t)cv * VEC * 2;
#pragma unroll
        for (int k = 0; k < VEC; ++k) { mine[2 * k] = s[k]; mine[2 * k + 1] = ss[k]; }
    }
    __syncthreads();
    const int cg = C / G;
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) {   // group totals over the group's channels, channel order
        const int g = i >> 1, which = i & 1;
        float acc = 0.f;
        for (int c = 0; c < cg; ++c) acc += s_dyn[(size_t)(g * cg + c) * 2 + which];
        partial[(((size_t)b * kGnMaxChunks + blockIdx.x) * G + g) * 2 + which] = acc;
    }
}

template <typename T>
__global__ void __launch_bounds__(1024) gn_apply_kernel(const T *__restrict__ x, const T *__restrict__ gamma,
                                                         const T *__restrict__ beta, const float *__restrict__ partial,
                                                         T *__restrict__ y, int HW, int C, int G, int ppb, int cvecs, int lanes,
                                                         float eps, int silu, int chunks) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float stats[];                     // [G][2] totals of this image (chunk order: reproducible)
    const int b = blockIdx.y, p0 = blockIdx.x * ppb, p1 = min(HW, p0 + ppb);
    const int cv = threadIdx.x % cvecs, pl = threadIdx.x / cvecs;
    for (int i = threadIdx.x; i < 2 * G; i += blockDim.x) {
        float acc = 0.f;
        for (int ch = 0; ch < chunks; ++ch) acc += partial[((size_t)b * kGnMaxChunks + ch) * 2 * G + i];
        stats[i] = acc;
    }
    __syncthreads();
    if (pl >= lanes) return;
    const int cg = C / G;
    const float inv_n = 1.f / ((float)cg * (float)HW);
    float sc[VEC], sh[VEC];
    {
        float gm[VEC], bt[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) { gm[k] = 1.f; bt[k] = 0.f; }
        if (gamma) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(gamma + cv * VEC), gm);
        if (beta) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(beta + cv * VEC), bt);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const int g = (cv * VEC + k) / cg;
            const float mean = stats[2 * g] * inv_n;
            const float var = fmaxf(stats[2 * g + 1] * inv_n - mean * mean, 0.f);
            const float r = rsqrtf(var + eps);
            sc[k] = r * gm[k];
            sh[k] = bt[k] - mean * sc[k];
        }
    }
    const size_t off = ((size_t)b * HW) * C + (size_t)cv * VEC;
    const T *xb = x + off;
    T *yb = y + off;
    auto one = [&](const uint4 &v, size_t p) {
        float f[VEC], o[VEC];
        Vec16<T>::unpack(v, f);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            float n = gn_rnd<T>(fmaf(f[k], sc[k], sh[k]));
            if (silu) n = __fdividef(n, 1.f + __expf(-n));
            o[k] = n;
        }
        stg_v4(yb + p * C, Vec16<T>::pack(o));
    };
    int p = p0 + pl;
    for (; p + 3 * lanes < p1; p += 4 * lanes) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = ldg_nc_v4(xb + (size_t)(p + u * lanes) * C);
#pragma unroll
        for (int u = 0; u < 4; ++u) one(v[u], (size_t)(p + u * lanes));
    }
    for (; p < p1; p += lanes) one(ldg_nc_v4(xb + (size_t)p * C), (size_t)p);
}

template <typename T>
static int gn_launch(const void *x, const void *gamma, const void *beta, void *y, float *stats, int B, int HW, int C, int G,
                     float eps, int silu, cudaStream_t st) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int cvecs = C / VEC;
    const int lanes = max(1, min(HW, 512 / cvecs));
    const int threads = cvecs * lanes;
    const int target_blocks = max(1, (num_sms() * 8) / B);               // ~8 CTAs' worth of work per SM over the batch
    int ppb = max(lanes * 4, (HW + target_blocks - 1) / target_blocks);
    ppb = max(ppb, (HW + kGnMaxChunks - 1) / kGnMaxChunks);
    ppb = min(ppb, HW);
    const int chunks = (HW + ppb - 1) / ppb;             // <= kGnMaxChunks
    const size_t smem_stats = (size_t)lanes * C * 2 * sizeof(float);
    constexpr auto kern = gn_stats_kernel<T>;
    const int rc = ensure_dynamic_smem<kern>(smem_stats);
    if (rc != MMFS_OK) return rc;
    dim3 grid(chunks, B);
    kern<<<grid, threads, smem_stats, st>>>((const T *)x, stats, HW, C, G, ppb, cvecs, lanes);
    gn_apply_kernel<T><<<grid, threads, 2 * G * sizeof(float), st>>>((const T *)x, (const T *)gamma, (const T *)beta, stats, (T *)y,
                                                                    HW, C, G, ppb, cvecs, lanes, eps, silu, chunks);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

}  // namespace mmfs

extern "C" int mmfs_groupnorm_nhwc(const void *x, const void *gamma, const void *beta, void *y, float *stats, int B, int HW,
                                   int C, int G, float eps, int silu, int dtype, void *stream) {
    using namespace mmfs;
    MMFS_CHECK_ARG(x && y && stats, "groupnorm: null pointer");
    MMFS_CHECK_ARG(B > 0 && HW > 0 && C > 0 && G > 0 && C % G == 0 && B <= 65535, "groupnorm: bad sizes B=%d HW=%d C=%d G=%d", B, HW, C, G);
    const size_t es = dtype_size(dtype);
    if (dtype == MMFS_F64 || es == 0 || C % (16 / (int)es) != 0 || C / (16 / (int)es) > 1024) {
        set_error("groupnorm: unsupported dtype %d / channel count %d (need C %% (16/sizeof) == 0, C*sizeof <= 16 KiB)", dtype, C);
        return MMFS_EUNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kF32Types>(dtype, "groupnorm", [&](auto tag) {
        return gn_launch<typename decltype(tag)::type>(x, gamma, beta, y, stats, B, HW, C, G, eps, silu, st);
    });
}
