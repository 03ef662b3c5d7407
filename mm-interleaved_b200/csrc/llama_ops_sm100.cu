// llama_ops_sm100.cu -- HBM-bound element-wise / row-wise kernels of the Llama-MMFS decoder layer.
//
//   mmfs_rmsnorm      LlamaRMSNorm.forward               decoders/modeling_llama_mmfs.py:53-70
//   mmfs_rope_qk      apply_rotary_pos_emb / rotate_half decoders/modeling_llama_mmfs.py:158-172
//   mmfs_swiglu       LlamaMLP: act_fn(gate) * up        decoders/modeling_llama_mmfs.py:188-189
//   mmfs_layernorm    nn.LayerNorm (CLIP / Q-Former / MMFSBlock norms)
//   mmfs_geglu        diffusers GEGLU: value * gelu(gate) (the SD UNet's feed-forward)
//   mmfs_rmsnorm_backward, mmfs_swiglu_backward, mmfs_layernorm_backward, mmfs_geglu_backward
//                     their gradients (training path, 16-bit tensors, fp32 math)
//
// Each mimics the rounding points of the reference's tensor pipeline in the storage type T (a
// tensor op in bf16 rounds its result to bf16), so a bf16 run tracks the reference's bf16 run and
// an fp32 run tracks its fp32 run.  All are pure bandwidth kernels: 16-byte vector loads/stores,
// one pass over the data, warp-shuffle + shared-memory row reductions, grid = rows.
#include "common.cuh"

namespace mmfs {

template <typename T> __device__ __forceinline__ float rnd(float x) { return to_op(from_op<T>(x)); }
template <> __device__ __forceinline__ float rnd<float>(float x) { return x; }

__device__ __forceinline__ float block_sum(float v, float *s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float t = (lane < nw) ? s_red[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    __syncthreads();
    return t;
}

// ---- RMSNorm: y = w * cast_T(x * rsqrt(mean(x^2) + eps)) -------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                       T *__restrict__ y, int cols, float eps) {
    constexpr int VEC = 16 / (int)sizeof(T);
    __shared__ float s_red[32];
    const size_t row = blockIdx.x;
    const T *xr = x + row * cols;
    T *yr = y + row * cols;
    const int nvec = cols / VEC;
    float ss = 0.f;
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        float f[VEC];
        Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(xr + i * VEC), f);
#pragma unroll
        for (int k = 0; k < VEC; ++k) ss += f[k] * f[k];
    }
    for (int i = nvec * VEC + threadIdx.x; i < cols; i += blockDim.x) { const float v = to_op(xr[i]); ss += v * v; }
    const float var = block_sum(ss, s_red) / (float)cols;      // variance in fp32 (:62)
    const float r = rsqrtf(var + eps);
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {     // second pass hits L1/L2
        float f[VEC], g[VEC], o[VEC];
        Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(xr + i * VEC), f);
        Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(w + i * VEC), g);
#pragma unroll
        for (int k = 0; k < VEC; ++k) o[k] = g[k] * rnd<T>(f[k] * r);   // cast to weight dtype, then weight * (:65-69)
        *reinterpret_cast<uint4 *>(yr + i * VEC) = Vec16<T>::pack(o);
    }
    for (int i = nvec * VEC + threadIdx.x; i < cols; i += blockDim.x)
        yr[i] = from_op<T>(to_op(w[i]) * rnd<T>(to_op(xr[i]) * r));
}

// Single-pass variant: 128 threads per row, the row stays in registers (up to kRmsChunks 16-byte vectors per thread:
// 8192 bf16 / 4096 fp32 columns), one shared-memory exchange between the four warps.  HBM traffic = read + write once.
constexpr int kRmsChunks = 8;
constexpr int kRmsThreads = 128;

template <typename T>
__global__ void __launch_bounds__(kRmsThreads) rmsnorm_reg_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                                  T *__restrict__ y, int cols, float eps) {
    constexpr int VEC = 16 / (int)sizeof(T);
    __shared__ float s_red[kRmsThreads / 32];
    const size_t row = blockIdx.x;
    const T *xr = x + row * cols;
    T *yr = y + row * cols;
    const int nvec = cols / VEC;                      // host: cols % VEC == 0, nvec <= kRmsThreads * kRmsChunks
    uint4 v[kRmsChunks], wv[kRmsChunks];          // the weight vectors travel with x: one memory round trip, not two
#pragma unroll
    for (int c = 0; c < kRmsChunks; ++c) {
        const int i = threadIdx.x + c * kRmsThreads;
        if (i < nvec) {
            v[c] = ldg_nc_v4(xr + i * VEC);
            wv[c] = ldg_nc_v4(w + i * VEC);
        }
    }
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < kRmsChunks; ++c)
        if (threadIdx.x + c * kRmsThreads < nvec) {
            float f[VEC];
            Vec16<T>::unpack(v[c], f);
#pragma unroll
            for (int k = 0; k < VEC; ++k) ss = fmaf(f[k], f[k], ss);
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = ss;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < kRmsThreads / 32; ++i) tot += s_red[i];
    const float r = rsqrtf(tot / (float)cols + eps);
#pragma unroll
    for (int c = 0; c < kRmsChunks; ++c) {
        const int i = threadIdx.x + c * kRmsThreads;
        if (i < nvec) {
            float f[VEC], g[VEC], o[VEC];
            Vec16<T>::unpack(v[c], f);
            Vec16<T>::unpack(wv[c], g);
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = g[k] * rnd<T>(f[k] * r);
            stg_v4(yr + i * VEC, Vec16<T>::pack(o));
        }
    }
}

// ---- LayerNorm (biased variance, fp32 statistics) ------------------------------------------------------
// Warp per row: the row lives in registers (16-byte vector loads), mean and centred variance are two warp
// reductions, one pass over HBM.  Rows of up to 32 * VEC * kLnChunks elements (2048 bf16 / 1024 fp32) take this
// path -- every LayerNorm on the interleaved path (64 ... 1280 columns); longer or unaligned rows use the block kernel.
constexpr int kLnChunks = 8;

// CH = 16-byte vectors per lane (1, 2, 4 or 8: rows of up to 32*CH*VEC elements).  The row is kept as raw 16-byte
// registers and unpacked three times (sum, centred squares, output): 4 registers per vector instead of 8 floats, so
// the common CH <= 4 instantiations stay under 64 registers and 32+ warps per SM hide the load latency (holding the
// row as floats for CH = 8 always needs 126 registers, i.e. 16 warps per SM).
template <typename T, int CH>
__global__ void __launch_bounds__(256, CH == 8 ? 2 : 4) layernorm_warp_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                              const T *__restrict__ b, T *__restrict__ y, long rows, int cols, float eps) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int lane = threadIdx.x & 31;
    const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const T *xr = x + row * cols;
    T *yr = y + row * cols;
    const int nvec = cols / VEC;                 // host guarantees cols % VEC == 0 and nvec <= 32 * CH
    uint4 v[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) {
        const int i = lane + 32 * c;
        v[c] = (i < nvec) ? ldg_nc_v4(xr + i * VEC) : make_uint4(0u, 0u, 0u, 0u);
    }
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c) {               // padding vectors are zeros: they add nothing to the sum
        float f[VEC];
        Vec16<T>::unpack(v[c], f);
#pragma unroll
        for (int k = 0; k < VEC; ++k) s += f[k];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)cols;
    float ss = 0.f;
#pragma unroll
    for (int c = 0; c < CH; ++c)
        if (lane + 32 * c < nvec) {
            float f[VEC];
            Vec16<T>::unpack(v[c], f);
#pragma unroll
            for (int k = 0; k < VEC; ++k) { const float d = f[k] - mean; ss = fmaf(d, d, ss); }
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float r = rsqrtf(ss / (float)cols + eps);
#pragma unroll
    for (int c = 0; c < CH; ++c) {
        const int i = lane + 32 * c;
        if (i < nvec) {
            float f[VEC], g[VEC], bb[VEC], o[VEC];
            Vec16<T>::unpack(v[c], f);
            if (w) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(w + i * VEC), g);
            if (b) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(b + i * VEC), bb);
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = (f[k] - mean) * r * (w ? g[k] : 1.f) + (b ? bb[k] : 0.f);
            stg_v4(yr + i * VEC, Vec16<T>::pack(o));
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) layernorm_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                         const T *__restrict__ b, T *__restrict__ y, int cols, float eps) {
    __shared__ float s_red[32];
    const size_t row = blockIdx.x;
    const T *xr = x + row * cols;
    T *yr = y + row * cols;
    float s = 0.f;
    for (int i = threadIdx.x; i < cols; i += blockDim.x) s += to_op(xr[i]);
    const float mean = block_sum(s, s_red) / (float)cols;
    float ss = 0.f;
    for (int i = threadIdx.x; i < cols; i += blockDim.x) { const float d = to_op(xr[i]) - mean; ss += d * d; }
    const float r = rsqrtf(block_sum(ss, s_red) / (float)cols + eps);
    for (int i = threadIdx.x; i < cols; i += blockDim.x) {
        const float n = (to_op(xr[i]) - mean) * r;
        yr[i] = from_op<T>(n * (w ? to_op(w[i]) : 1.f) + (b ? to_op(b[i]) : 0.f));
    }
}

// ---- RoPE on q and k, in place, (B, T, H, hd) layout (the GEMM output layout: no transposes) -------
//   q_embed = q * cos + rotate_half(q) * sin, rotate_half(x) = cat(-x2, x1)       (:158-172)
template <typename T>
__global__ void __launch_bounds__(256) rope_qk_kernel(T *__restrict__ q, T *__restrict__ k, const float *__restrict__ cos_t,
                                                       const float *__restrict__ sin_t, const int64_t *__restrict__ pos,
                                                       long n_tok, int H, int hd, int q_stride, int k_stride, int pos_per_batch,
                                                       int T_len) {
    // one CTA per token (grid-stride), one thread per (q-or-k, head, chunk of VEC rotation pairs): two 16-byte loads
    // (x1 | x2 halves), two 16-byte stores; the token's cos/sin row is fp32 and read through L1 by every head.
    // All index math is 32-bit and per token, so the kernel is pure load/store.
    constexpr int VEC = 16 / (int)sizeof(T);
    const int half = hd >> 1;
    const int chunks = half / VEC;
    const int per_tok = 2 * H * chunks;
    // blockDim.x is a multiple of `chunks` whenever chunks is a power of two <= 32 (head sizes 64 / 128): a thread then
    // keeps the same rotation chunk for every head it visits and loads the token's cos / sin values once per token
    const bool hoist = (blockDim.x % chunks) == 0;
    for (long tok = blockIdx.x; tok < n_tok; tok += gridDim.x) {
        const long p = pos[pos_per_batch ? tok : (tok % T_len)];
        const float *cp = cos_t + p * hd, *sp = sin_t + p * hd;
        T *qt = q + tok * q_stride, *kt = k + tok * k_stride;
        float cs[VEC], sn[VEC];
        auto load_table = [&](int c) {
#pragma unroll
            for (int i = 0; i < VEC; i += 4) {
                const float4 a = *reinterpret_cast<const float4 *>(cp + c * VEC + i);
                const float4 b = *reinterpret_cast<const float4 *>(sp + c * VEC + i);
                cs[i] = rnd<T>(a.x); cs[i + 1] = rnd<T>(a.y); cs[i + 2] = rnd<T>(a.z); cs[i + 3] = rnd<T>(a.w);   // tables cast to
                sn[i] = rnd<T>(b.x); sn[i + 1] = rnd<T>(b.y); sn[i + 2] = rnd<T>(b.z); sn[i + 3] = rnd<T>(b.w);   // x.dtype (:141-144)
            }
        };
        if (hoist) load_table(threadIdx.x % chunks);
        for (int it = threadIdx.x; it < per_tok; it += blockDim.x) {
            const int c = it % chunks;
            const int hh = it / chunks;                 // 0 .. 2H-1: q heads then k heads
            T *x = (hh >= H ? kt + (size_t)(hh - H) * hd : qt + (size_t)hh * hd) + c * VEC;
            float x1[VEC], x2[VEC], o1[VEC], o2[VEC];
            const uint4 v1 = *reinterpret_cast<const uint4 *>(x), v2 = *reinterpret_cast<const uint4 *>(x + half);
            if (!hoist) load_table(c);
            Vec16<T>::unpack(v1, x1);
            Vec16<T>::unpack(v2, x2);
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                o1[i] = rnd<T>(x1[i] * cs[i]) + rnd<T>(-x2[i] * sn[i]);
                o2[i] = rnd<T>(x2[i] * cs[i]) + rnd<T>(x1[i] * sn[i]);
            }
            *reinterpret_cast<uint4 *>(x) = Vec16<T>::pack(o1);
            *reinterpret_cast<uint4 *>(x + half) = Vec16<T>::pack(o2);
        }
    }
}

// RoPE + KV-cache append in one pass (extension; a static cache replaces the reference's torch.cat append,
// modeling_llama_mmfs.py:236-239): q is rotated in place, the ROTATED k and the v of every token go straight into
// the cache row of the token -- row (slot + t) of batch entry b, where slot is a host integer (prefill / eager decode:
// the number of positions already cached) or is read from device memory (the graphed decode step).  Same arithmetic
// as rope_qk_kernel; saves the in-place write of k plus two copy kernels per layer and token.
template <typename T>
__global__ void __launch_bounds__(256) rope_append_kernel(T *__restrict__ q, const T *__restrict__ k, const T *__restrict__ v,
                                                           const float *__restrict__ cos_t, const float *__restrict__ sin_t,
                                                           const int64_t *__restrict__ pos, T *__restrict__ k_cache,
                                                           T *__restrict__ v_cache, const int64_t *__restrict__ slot_dev,
                                                           long slot_host, long n_tok, int H, int hd, int q_stride, int k_stride,
                                                           int v_stride, long cache_bs, long cache_ts, int pos_per_batch, int T_len) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int half = hd >> 1;
    const int chunks = half / VEC;
    const int n_rot = 2 * H * chunks;                     // rotation items: q heads then k heads
    const int n_copy = H * hd / VEC;                      // v vectors
    const long slot = slot_dev != nullptr ? (long)*slot_dev : slot_host;
    for (long tok = blockIdx.x; tok < n_tok; tok += gridDim.x) {
        const long p = pos[pos_per_batch ? tok : (tok % T_len)];
        const float *cp = cos_t + p * hd, *sp = sin_t + p * hd;
        const long b = tok / T_len, tt = tok - b * T_len;
        T *qt = q + tok * q_stride;
        const T *kt = k + tok * k_stride, *vt = v + tok * v_stride;
        T *kc = k_cache + b * cache_bs + (slot + tt) * cache_ts, *vc = v_cache + b * cache_bs + (slot + tt) * cache_ts;
        for (int it = threadIdx.x; it < n_rot + n_copy; it += blockDim.x) {
            if (it >= n_rot) {                            // v: plain copy
                const int i = (it - n_rot) * VEC;
                *reinterpret_cast<uint4 *>(vc + i) = *reinterpret_cast<const uint4 *>(vt + i);
                continue;
            }
            const int c = it % chunks, hh = it / chunks;
            const bool is_k = hh >= H;
            const T *src = (is_k ? kt + (size_t)(hh - H) * hd : qt + (size_t)hh * hd) + c * VEC;
            T *dst = (is_k ? kc + (size_t)(hh - H) * hd : qt + (size_t)hh * hd) + c * VEC;
            float cs[VEC], sn[VEC], x1[VEC], x2[VEC], o1[VEC], o2[VEC];
#pragma unroll
            for (int i = 0; i < VEC; i += 4) {
                const float4 a = *reinterpret_cast<const float4 *>(cp + c * VEC + i);
                const float4 bb = *reinterpret_cast<const float4 *>(sp + c * VEC + i);
                cs[i] = rnd<T>(a.x); cs[i + 1] = rnd<T>(a.y); cs[i + 2] = rnd<T>(a.z); cs[i + 3] = rnd<T>(a.w);
                sn[i] = rnd<T>(bb.x); sn[i + 1] = rnd<T>(bb.y); sn[i + 2] = rnd<T>(bb.z); sn[i + 3] = rnd<T>(bb.w);
            }
            Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(src), x1);
            Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(src + half), x2);
#pragma unroll
            for (int i = 0; i < VEC; ++i) {
                o1[i] = rnd<T>(x1[i] * cs[i]) + rnd<T>(-x2[i] * sn[i]);
                o2[i] = rnd<T>(x2[i] * cs[i]) + rnd<T>(x1[i] * sn[i]);
            }
            *reinterpret_cast<uint4 *>(dst) = Vec16<T>::pack(o1);
            *reinterpret_cast<uint4 *>(dst + half) = Vec16<T>::pack(o2);
        }
    }
}

// silu in fp32: exact expf / division for fp32 tensors; ex2.approx + rcp.approx for 16-bit tensors, whose result is
// rounded to 8 / 11 significand bits right after (relative error of the fast path ~2^-21).
template <typename T> __device__ __forceinline__ float silu_op(float g) { return __fdividef(g, 1.f + __expf(-g)); }
template <> __device__ __forceinline__ float silu_op<float>(float g) { return g / (1.f + expf(-g)); }

// GEGLU (diffusers FeedForward of the SD UNet): out = value * gelu(gate) with [value | gate] halves and the exact
// erf GELU -- the same kernel with ACT = 1 and the gate in the second half.
template <typename T, int ACT> __device__ __forceinline__ float glu_act(float g) {
    if (ACT == 0) return silu_op<T>(g);
    return 0.5f * g * (1.f + erff(g * 0.70710678118654752f));
}

template <typename T, int ACT = 0, bool GATE_SECOND = false>
__global__ void __launch_bounds__(256) swiglu_kernel(const T *__restrict__ gu, T *__restrict__ out, long rows, int I) {
    // CTA per row (grid-stride): no 64-bit index division, two independent (gate, up) vector pairs in flight per thread
    // gridDim.y > 1 (few rows, e.g. a decode step): a row is cut into column slices so that it spreads over many SMs
    constexpr int VEC = 16 / (int)sizeof(T);
    const int per = (I / VEC + gridDim.y - 1) / gridDim.y;
    const int v0 = blockIdx.y * per, nvec = min(I / VEC, v0 + per);
    for (long r = blockIdx.x; r < rows; r += gridDim.x) {
        const T *g_row = gu + r * 2 * I + (GATE_SECOND ? I : 0), *u_row = gu + r * 2 * I + (GATE_SECOND ? 0 : I);
        T *o_row = out + r * I;
        int i = v0 + threadIdx.x;
        for (; i + (int)blockDim.x < nvec; i += 2 * blockDim.x) {
            const int j = i + blockDim.x;
            const uint4 g0 = ldg_nc_v4(g_row + i * VEC), u0 = ldg_nc_v4(u_row + i * VEC);
            const uint4 g1 = ldg_nc_v4(g_row + j * VEC), u1 = ldg_nc_v4(u_row + j * VEC);
            float g[VEC], u[VEC], o[VEC];
            Vec16<T>::unpack(g0, g); Vec16<T>::unpack(u0, u);
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = rnd<T>(glu_act<T, ACT>(g[k])) * u[k];   // act_fn(gate) is a tensor in T
            stg_v4(o_row + i * VEC, Vec16<T>::pack(o));
            Vec16<T>::unpack(g1, g); Vec16<T>::unpack(u1, u);
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = rnd<T>(glu_act<T, ACT>(g[k])) * u[k];
            stg_v4(o_row + j * VEC, Vec16<T>::pack(o));
        }
        if (i < nvec) {
            float g[VEC], u[VEC], o[VEC];
            Vec16<T>::unpack(ldg_nc_v4(g_row + i * VEC), g); Vec16<T>::unpack(ldg_nc_v4(u_row + i * VEC), u);
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = rnd<T>(glu_act<T, ACT>(g[k])) * u[k];
            stg_v4(o_row + i * VEC, Vec16<T>::pack(o));
        }
    }
}

template <typename T>
static int launch_rmsnorm(const void *x, const void *w, void *y, long rows, int cols, float eps, cudaStream_t st) {
    if (cols % (16 / (int)sizeof(T)) == 0 && cols / (16 / (int)sizeof(T)) <= kRmsThreads * kRmsChunks)
        rmsnorm_reg_kernel<T><<<(unsigned)rows, kRmsThreads, 0, st>>>((const T *)x, (const T *)w, (T *)y, cols, eps);
    else
        rmsnorm_kernel<T><<<(unsigned)rows, 256, 0, st>>>((const T *)x, (const T *)w, (T *)y, cols, eps);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_layernorm(const void *x, const void *w, const void *b, void *y, long rows, int cols, float eps, cudaStream_t st) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const bool vec_ok = (cols % VEC == 0) && (cols / VEC <= 32 * kLnChunks) &&
                        (((uintptr_t)x | (uintptr_t)y | (uintptr_t)w | (uintptr_t)b) % 16 == 0);
    if (vec_ok) {
        const int nvec = cols / VEC;
        const unsigned grid = (unsigned)((rows + 7) / 8);
#define MMFS_LN(CH) layernorm_warp_kernel<T, CH><<<grid, 256, 0, st>>>((const T *)x, (const T *)w, (const T *)b, (T *)y, rows, cols, eps)
        if (nvec <= 32) MMFS_LN(1); else if (nvec <= 64) MMFS_LN(2); else if (nvec <= 128) MMFS_LN(4); else MMFS_LN(8);
#undef MMFS_LN
    } else
        layernorm_kernel<T><<<(unsigned)rows, 256, 0, st>>>((const T *)x, (const T *)w, (const T *)b, (T *)y, cols, eps);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_rope(void *q, void *k, const float *cos_t, const float *sin_t, const int64_t *pos, long n_tok, int T_len,
                       int H, int hd, int qs, int ks, int ppb, cudaStream_t st) {
    const int per_tok = H * 2 * ((hd / 2) / (16 / (int)sizeof(T)));
    const int threads = per_tok >= 256 ? 256 : ((per_tok + 31) / 32) * 32;
    rope_qk_kernel<T><<<capped_grid(n_tok, 32), threads, 0, st>>>((T *)q, (T *)k, cos_t, sin_t, pos, n_tok, H, hd, qs, ks, ppb,
                                                                  T_len);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

// swiglu: silu over [gate | up]; geglu: gelu over [value | gate]
template <typename T>
static int launch_glu(const void *in, void *out, long rows, int inter, bool geglu, cudaStream_t st) {
    const int nvec = inter / (16 / (int)sizeof(T));
    const int threads = nvec >= 512 ? 256 : (nvec >= 64 ? 64 : 32);
    const int gx = capped_grid(rows, 64);
    int gy = 1;                                   // fewer CTAs than SMs: slice the columns (two vectors per thread)
    if (gx < num_sms()) { gy = (nvec + 2 * threads - 1) / (2 * threads); if (gy > 64) gy = 64; if (gy < 1) gy = 1; }
    const dim3 grid(gx, gy);
    if (geglu)
        swiglu_kernel<T, 1, true><<<grid, threads, 0, st>>>((const T *)in, (T *)out, rows, inter);
    else
        swiglu_kernel<T, 0, false><<<grid, threads, 0, st>>>((const T *)in, (T *)out, rows, inter);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_rope_append(void *q, const void *k, const void *v, const float *cos_t, const float *sin_t, const int64_t *pos,
                              void *kc, void *vc, const int64_t *slot_dev, long slot_host, long n_tok, int T_len, int H, int hd,
                              int qs, int ks, int vs, long cbs, long cts, int ppb, cudaStream_t st) {
    const int items = H * ((hd / 2) / (16 / (int)sizeof(T))) * 2 + H * hd / (16 / (int)sizeof(T));
    const int threads = items >= 256 ? 256 : ((items + 31) / 32) * 32;
    rope_append_kernel<T><<<capped_grid(n_tok, 32), threads, 0, st>>>((T *)q, (const T *)k, (const T *)v, cos_t, sin_t, pos, (T *)kc,
                                                                      (T *)vc, slot_dev, slot_host, n_tok, H, hd, qs, ks, vs, cbs,
                                                                      cts, ppb, T_len);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}


// ---- RMSNorm backward: dx = r * (g - x * r^2 * mean(g * x)), g = dy * w; dweight = sum over rows of dy * cast_T(x * r) --
// CTA p of kRmsBwdParts takes rows p, p + parts, ... in that order and keeps its dweight partial in shared memory
// (every thread owns the same columns for every row, so no synchronisation); the partials are summed per column in
// part order by rmsnorm_dw_reduce_kernel.  The part count depends only on `rows`, so the sum is run-to-run reproducible.
constexpr int kRmsBwdParts = MMFS_RMSNORM_BWD_PARTS;
constexpr int kRmsBwdMaxCols = 8192;

template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                          const T *__restrict__ dy, T *__restrict__ dx,
                                                          float *__restrict__ partials, long rows, int cols, float eps) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dw[];                           // cols floats, only with partials
    __shared__ float s_red[32];
    const int nvec = cols / VEC;
    if (partials)
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
#pragma unroll
            for (int k = 0; k < VEC; ++k) s_dw[i * VEC + k] = 0.f;
    for (long row = blockIdx.x; row < rows; row += gridDim.x) {
        const T *xr = x + row * cols, *dyr = dy + row * cols;
        float ss = 0.f, sg = 0.f;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float f[VEC], g[VEC], d[VEC];
            Vec16<T>::unpack(ldg_nc_v4(xr + i * VEC), f);
            Vec16<T>::unpack(ldg_nc_v4(w + i * VEC), g);
            Vec16<T>::unpack(ldg_nc_v4(dyr + i * VEC), d);
#pragma unroll
            for (int k = 0; k < VEC; ++k) { ss = fmaf(f[k], f[k], ss); sg = fmaf(d[k] * g[k], f[k], sg); }
        }
        ss = block_sum(ss, s_red);
        sg = block_sum(sg, s_red);
        const float r = rsqrtf(ss / (float)cols + eps);         // the forward's statistic
        const float coef = r * r * r * sg / (float)cols;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float f[VEC], g[VEC], d[VEC], o[VEC];
            Vec16<T>::unpack(ldg_nc_v4(xr + i * VEC), f);
            Vec16<T>::unpack(ldg_nc_v4(w + i * VEC), g);
            Vec16<T>::unpack(ldg_nc_v4(dyr + i * VEC), d);
#pragma unroll
            for (int k = 0; k < VEC; ++k) o[k] = fmaf(r * d[k], g[k], -f[k] * coef);
            stg_v4(dx + row * cols + i * VEC, Vec16<T>::pack(o));
            if (partials)
#pragma unroll
                for (int k = 0; k < VEC; ++k) s_dw[i * VEC + k] = fmaf(d[k], rnd<T>(f[k] * r), s_dw[i * VEC + k]);
        }
    }
    if (partials)
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
#pragma unroll
            for (int k = 0; k < VEC; ++k) partials[(long)blockIdx.x * cols + i * VEC + k] = s_dw[i * VEC + k];
}

template <typename T>
__global__ void __launch_bounds__(256) rmsnorm_dw_reduce_kernel(const float *__restrict__ partials, T *__restrict__ dw,
                                                                int parts, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float s = 0.f;
    for (int p = 0; p < parts; ++p) s += partials[(long)p * cols + c];
    dw[c] = from_op<T>(s);
}

// ---- LayerNorm backward: xhat = (x - mean) r, g = dy * w; dx = r * (g - mean(g) - xhat * mean(g * xhat));
// dweight = sum over rows of dy * xhat, dbias = sum over rows of dy.  The statistics are recomputed from x in fp32 (the
// forward rounds only its output).  Same part scheme as the RMSNorm backward: CTA p takes rows p, p + parts, ... and keeps
// its dweight / dbias partials in shared memory; layernorm_dwdb_reduce_kernel sums them per column in part order.  The
// CTA is as wide as a row's 16-byte vectors (32 .. 256 threads), so that the 64-wide qk-norm rows do not idle 7 warps.
template <typename T>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const T *__restrict__ x, const T *__restrict__ w,
                                                            const T *__restrict__ dy, T *__restrict__ dx,
                                                            float *__restrict__ partials, long rows, int cols, float eps) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_part[];                         // [dweight | dbias] x cols floats, only with partials
    __shared__ float s_red[32];
    const int nvec = cols / VEC;
    float *s_dw = s_part, *s_db = s_part + cols;
    if (partials)                                             // every thread owns the same columns for every row
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
#pragma unroll
            for (int k = 0; k < VEC; ++k) s_dw[i * VEC + k] = s_db[i * VEC + k] = 0.f;
    const float inv_n = 1.f / (float)cols;
    for (long row = blockIdx.x; row < rows; row += gridDim.x) {
        const T *xr = x + row * cols, *dyr = dy + row * cols;
        float s = 0.f;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float f[VEC];
            Vec16<T>::unpack(ldg_nc_v4(xr + i * VEC), f);
#pragma unroll
            for (int k = 0; k < VEC; ++k) s += f[k];
        }
        const float mean = block_sum(s, s_red) * inv_n;
        float ss = 0.f, sg = 0.f, sgx = 0.f;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float f[VEC], g[VEC], d[VEC];
            Vec16<T>::unpack(ldg_nc_v4(xr + i * VEC), f);
            Vec16<T>::unpack(ldg_nc_v4(w + i * VEC), g);
            Vec16<T>::unpack(ldg_nc_v4(dyr + i * VEC), d);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float c = f[k] - mean, gk = d[k] * g[k];
                ss = fmaf(c, c, ss);
                sg += gk;
                sgx = fmaf(gk, c, sgx);
            }
        }
        ss = block_sum(ss, s_red);
        sg = block_sum(sg, s_red);
        sgx = block_sum(sgx, s_red);
        const float r = rsqrtf(ss * inv_n + eps);               // the forward's statistic
        const float mg = sg * inv_n, mgx = sgx * r * inv_n;     // mean(g), mean(g * xhat)
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float f[VEC], g[VEC], d[VEC], o[VEC];
            Vec16<T>::unpack(ldg_nc_v4(xr + i * VEC), f);
            Vec16<T>::unpack(ldg_nc_v4(w + i * VEC), g);
            Vec16<T>::unpack(ldg_nc_v4(dyr + i * VEC), d);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float xh = (f[k] - mean) * r;
                o[k] = r * (fmaf(d[k], g[k], -mg) - xh * mgx);
                if (partials) {
                    s_dw[i * VEC + k] = fmaf(d[k], xh, s_dw[i * VEC + k]);
                    s_db[i * VEC + k] += d[k];
                }
            }
            stg_v4(dx + row * cols + i * VEC, Vec16<T>::pack(o));
        }
    }
    if (partials)
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                partials[(long)blockIdx.x * cols + i * VEC + k] = s_dw[i * VEC + k];
                partials[((long)gridDim.x + blockIdx.x) * cols + i * VEC + k] = s_db[i * VEC + k];
            }
}

template <typename T>
__global__ void __launch_bounds__(256) layernorm_dwdb_reduce_kernel(const float *__restrict__ partials, T *__restrict__ dw,
                                                                    T *__restrict__ db, int parts, int cols) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float sw = 0.f, sb = 0.f;
    for (int p = 0; p < parts; ++p) {
        sw += partials[(long)p * cols + c];
        sb += partials[((long)parts + p) * cols + c];
    }
    if (dw) dw[c] = from_op<T>(sw);
    if (db) db[c] = from_op<T>(sb);
}

// ---- SwiGLU backward: out = silu(g) * u  ->  dg = d * u * s * (1 + g * (1 - s)), du = d * silu(g), s = sigmoid(g) ----
template <typename T>
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const T *__restrict__ gu, const T *__restrict__ d_out,
                                                         T *__restrict__ d_gu, long rows, int I) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int nvec = I / VEC;
    for (long r = blockIdx.x; r < rows; r += gridDim.x)
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float g[VEC], u[VEC], d[VEC], dg[VEC], du[VEC];
            Vec16<T>::unpack(ldg_nc_v4(gu + r * 2 * I + i * VEC), g);
            Vec16<T>::unpack(ldg_nc_v4(gu + r * 2 * I + I + i * VEC), u);
            Vec16<T>::unpack(ldg_nc_v4(d_out + r * I + i * VEC), d);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                const float s = 1.f / (1.f + expf(-g[k]));
                dg[k] = d[k] * u[k] * s * fmaf(g[k], 1.f - s, 1.f);
                du[k] = d[k] * g[k] * s;
            }
            stg_v4(d_gu + r * 2 * I + i * VEC, Vec16<T>::pack(dg));
            stg_v4(d_gu + r * 2 * I + I + i * VEC, Vec16<T>::pack(du));
        }
}

// ---- GEGLU backward: out = v * gelu(g), gelu(g) = g Phi(g) (exact erf form)  ->  dv = d * gelu(g),
// dg = d * v * (Phi(g) + g phi(g)), Phi / phi the standard normal CDF / density.  fp32, one rounding at the store.  The
// index space is the (rows, I) grid flattened; kVec: I % VEC == 0 and 16-byte aligned tensors, so every 16-byte vector
// lies inside one row; otherwise one element per step.
__device__ __forceinline__ void geglu_grad(float v, float g, float d, float &dv, float &dg) {
    const float cdf = 0.5f * (1.f + erff(g * 0.70710678118654752f));
    const float pdf = 0.39894228040143268f * expf(-0.5f * g * g);
    dv = d * g * cdf;
    dg = d * v * fmaf(g, pdf, cdf);
}

template <typename T, bool kVec>
__global__ void __launch_bounds__(256) geglu_bwd_kernel(const T *__restrict__ vg, const T *__restrict__ d_out,
                                                        T *__restrict__ d_vg, long rows, int I) {
    constexpr int VEC = kVec ? 16 / (int)sizeof(T) : 1;
    const long per_row = I / VEC, n = rows * per_row;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
        const long r = t / per_row, i = (t - r * per_row) * VEC;
        const long v_at = r * 2 * I + i, g_at = v_at + I;
        float v[VEC], g[VEC], d[VEC], dv[VEC], dg[VEC];
        if constexpr (kVec) {
            Vec16<T>::unpack(ldg_nc_v4(vg + v_at), v);
            Vec16<T>::unpack(ldg_nc_v4(vg + g_at), g);
            Vec16<T>::unpack(ldg_nc_v4(d_out + r * I + i), d);
        } else {
            v[0] = to_op(vg[v_at]);
            g[0] = to_op(vg[g_at]);
            d[0] = to_op(d_out[r * I + i]);
        }
#pragma unroll
        for (int k = 0; k < VEC; ++k) geglu_grad(v[k], g[k], d[k], dv[k], dg[k]);
        if constexpr (kVec) {
            stg_v4(d_vg + v_at, Vec16<T>::pack(dv));
            stg_v4(d_vg + g_at, Vec16<T>::pack(dg));
        } else {
            d_vg[v_at] = from_op<T>(dv[0]);
            d_vg[g_at] = from_op<T>(dg[0]);
        }
    }
}

template <typename T>
static int launch_geglu_bwd(const void *vg, const void *d_out, void *d_vg, long rows, int inter, bool vec, cudaStream_t st) {
    const long items = rows * (vec ? inter / (16 / (int)sizeof(T)) : inter);
    const int grid = capped_grid((items + 255) / 256, 8);
    if (vec)
        geglu_bwd_kernel<T, true><<<grid, 256, 0, st>>>((const T *)vg, (const T *)d_out, (T *)d_vg, rows, inter);
    else
        geglu_bwd_kernel<T, false><<<grid, 256, 0, st>>>((const T *)vg, (const T *)d_out, (T *)d_vg, rows, inter);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_rmsnorm_bwd(const void *x, const void *w, const void *dy, void *dx, void *dw, float *partials, long rows,
                              int cols, float eps, cudaStream_t st) {
    const int parts = (int)(rows < kRmsBwdParts ? rows : kRmsBwdParts);
    rmsnorm_bwd_kernel<T><<<parts, 256, dw ? cols * sizeof(float) : 0, st>>>(
        (const T *)x, (const T *)w, (const T *)dy, (T *)dx, dw ? partials : nullptr, rows, cols, eps);
    MMFS_CUDA(cudaGetLastError());
    if (dw) {
        rmsnorm_dw_reduce_kernel<T><<<(cols + 255) / 256, 256, 0, st>>>(partials, (T *)dw, parts, cols);
        MMFS_CUDA(cudaGetLastError());
    }
    return MMFS_OK;
}

template <typename T>
static int launch_layernorm_bwd(const void *x, const void *w, const void *dy, void *dx, void *dw, void *db, float *partials,
                                long rows, int cols, float eps, cudaStream_t st) {
    const int parts = (int)(rows < kRmsBwdParts ? rows : kRmsBwdParts);
    const int nvec = cols / (16 / (int)sizeof(T));
    const int threads = nvec >= 256 ? 256 : (nvec + 31) / 32 * 32;
    const bool red = dw != nullptr || db != nullptr;
    const size_t smem = red ? 2 * (size_t)cols * sizeof(float) : 0;
    const int rc = ensure_dynamic_smem<layernorm_bwd_kernel<T>>(smem);
    if (rc != MMFS_OK) return rc;
    layernorm_bwd_kernel<T><<<parts, threads, smem, st>>>((const T *)x, (const T *)w, (const T *)dy, (T *)dx,
                                                           red ? partials : nullptr, rows, cols, eps);
    MMFS_CUDA(cudaGetLastError());
    if (red) {
        layernorm_dwdb_reduce_kernel<T><<<(cols + 255) / 256, 256, 0, st>>>(partials, (T *)dw, (T *)db, parts, cols);
        MMFS_CUDA(cudaGetLastError());
    }
    return MMFS_OK;
}

template <typename T>
static int launch_swiglu_bwd(const void *gu, const void *d_out, void *d_gu, long rows, int inter, cudaStream_t st) {
    swiglu_bwd_kernel<T><<<capped_grid(rows, 8), 256, 0, st>>>((const T *)gu, (const T *)d_out, (T *)d_gu, rows, inter);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_rmsnorm(const void *x, const void *weight, void *y, long rows, int cols, float eps, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && cols > 0, "rmsnorm: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && weight && y, "rmsnorm: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)x | (uintptr_t)weight | (uintptr_t)y) % 16 == 0 && (cols * dtype_size(dtype)) % 16 == 0,
                   "rmsnorm: rows must be 16-byte aligned");
    return dispatch_dtype<kF32Types>(dtype, "rmsnorm", [&](auto tag) {
        return launch_rmsnorm<typename decltype(tag)::type>(x, weight, y, rows, cols, eps, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_layernorm(const void *x, const void *weight, const void *bias, void *y, long rows, int cols, float eps,
                              int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && cols > 0, "layernorm: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && y, "layernorm: null pointer argument");
    return dispatch_dtype<kF32Types>(dtype, "layernorm", [&](auto tag) {
        return launch_layernorm<typename decltype(tag)::type>(x, weight, bias, y, rows, cols, eps, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_rope_qk(void *q, void *k, const float *cos_table, const float *sin_table, const int64_t *position_ids,
                            long n_tokens, int T_len, int H, int hd, int q_stride, int k_stride, int pos_per_batch,
                            int dtype, void *stream) {
    MMFS_CHECK_ARG(n_tokens >= 0 && H > 0 && hd > 0 && hd % 2 == 0 && T_len > 0, "rope_qk: bad shape");
    if (n_tokens == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && cos_table && sin_table && position_ids, "rope_qk: null pointer argument");
    MMFS_CHECK_ARG((hd / 2) % (16 / (int)dtype_size(dtype)) == 0 && ((uintptr_t)q | (uintptr_t)k) % 16 == 0 &&
                   (q_stride * dtype_size(dtype)) % 16 == 0 && (k_stride * dtype_size(dtype)) % 16 == 0,
                   "rope_qk: head_dim/2 must be a multiple of the 16-byte vector and rows 16-byte aligned");
    return dispatch_dtype<kF32Types>(dtype, "rope_qk", [&](auto tag) {
        return launch_rope<typename decltype(tag)::type>(q, k, cos_table, sin_table, position_ids, n_tokens, T_len, H, hd, q_stride,
                                                         k_stride, pos_per_batch, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_rope_qk_append(void *q, const void *k, const void *v, const float *cos_table, const float *sin_table,
                                   const int64_t *position_ids, void *k_cache, void *v_cache, const int64_t *slot_dev,
                                   long slot_host, long n_tokens, int T_len, int H, int hd, int q_stride, int k_stride,
                                   int v_stride, long cache_bs, long cache_ts, int pos_per_batch, int dtype, void *stream) {
    MMFS_CHECK_ARG(n_tokens >= 0 && H > 0 && hd > 0 && hd % 2 == 0 && T_len > 0 && slot_host >= 0, "rope_qk_append: bad shape");
    if (n_tokens == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && cos_table && sin_table && position_ids && k_cache && v_cache, "rope_qk_append: null pointer argument");
    const size_t es = dtype_size(dtype);
    MMFS_CHECK_ARG(es == 2 || es == 4, "rope_qk_append: f32 / f16 / bf16");
    MMFS_CHECK_ARG((hd / 2) % (16 / (int)es) == 0 &&
                       ((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)k_cache | (uintptr_t)v_cache) % 16 == 0 &&
                       (q_stride * es) % 16 == 0 && (k_stride * es) % 16 == 0 && (v_stride * es) % 16 == 0 &&
                       (cache_bs * es) % 16 == 0 && (cache_ts * es) % 16 == 0,
                   "rope_qk_append: head_dim/2 must be a multiple of the 16-byte vector and all rows 16-byte aligned");
    return dispatch_dtype<kF32Types>(dtype, "rope_qk_append", [&](auto tag) {
        return launch_rope_append<typename decltype(tag)::type>(q, k, v, cos_table, sin_table, position_ids, k_cache, v_cache,
                                                                slot_dev, slot_host, n_tokens, T_len, H, hd, q_stride, k_stride,
                                                                v_stride, cache_bs, cache_ts, pos_per_batch, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_swiglu(const void *gate_up, void *out, long rows, int inter, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && inter > 0, "swiglu: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(gate_up && out, "swiglu: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)gate_up | (uintptr_t)out) % 16 == 0 && (inter * dtype_size(dtype)) % 16 == 0,
                   "swiglu: rows must be 16-byte aligned");
    return dispatch_dtype<kF32Types>(dtype, "swiglu", [&](auto tag) {
        return launch_glu<typename decltype(tag)::type>(gate_up, out, rows, inter, false, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_geglu(const void *value_gate, void *out, long rows, int inter, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && inter > 0, "geglu: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value_gate && out, "geglu: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)value_gate | (uintptr_t)out) % 16 == 0 && (inter * dtype_size(dtype)) % 16 == 0,
                   "geglu: rows must be 16-byte aligned");
    return dispatch_dtype<kF32Types>(dtype, "geglu", [&](auto tag) {
        return launch_glu<typename decltype(tag)::type>(value_gate, out, rows, inter, true, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_rmsnorm_backward(const void *x, const void *weight, const void *dy, void *dx, void *dweight,
                                     float *partials, long rows, int cols, float eps, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && cols > 0, "rmsnorm_backward: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && weight && dy && dx && (!dweight || partials), "rmsnorm_backward: null pointer argument");
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16) || cols % 8 != 0 || cols > kRmsBwdMaxCols ||
        ((uintptr_t)x | (uintptr_t)weight | (uintptr_t)dy | (uintptr_t)dx) % 16 != 0) {
        set_error("rmsnorm_backward: needs bf16 / f16, cols %% 8 == 0, cols <= %d, 16-byte aligned rows (got cols=%d dtype=%d)",
                  kRmsBwdMaxCols, cols, dtype);
        return MMFS_EUNSUPPORTED;
    }
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "rmsnorm_backward", [&](auto tag) {
        return launch_rmsnorm_bwd<typename decltype(tag)::type>(x, weight, dy, dx, dweight, partials, rows, cols, eps,
                                                                (cudaStream_t)stream);
    });
}

extern "C" int mmfs_swiglu_backward(const void *gate_up, const void *d_out, void *d_gate_up, long rows, int inter, int dtype,
                                    void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && inter > 0, "swiglu_backward: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(gate_up && d_out && d_gate_up, "swiglu_backward: null pointer argument");
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16) || inter % 8 != 0 ||
        ((uintptr_t)gate_up | (uintptr_t)d_out | (uintptr_t)d_gate_up) % 16 != 0) {
        set_error("swiglu_backward: needs bf16 / f16, inter %% 8 == 0 and 16-byte aligned rows (got inter=%d dtype=%d)", inter, dtype);
        return MMFS_EUNSUPPORTED;
    }
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "swiglu_backward", [&](auto tag) {
        return launch_swiglu_bwd<typename decltype(tag)::type>(gate_up, d_out, d_gate_up, rows, inter, (cudaStream_t)stream);
    });
}

extern "C" int mmfs_geglu_backward(const void *value_gate, const void *d_out, void *d_value_gate, long rows, int inter,
                                   int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && inter > 0, "geglu_backward: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value_gate && d_out && d_value_gate, "geglu_backward: null pointer argument");
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16)) {
        set_error("geglu_backward: needs bf16 / f16 (got dtype=%d)", dtype);
        return MMFS_EUNSUPPORTED;
    }
    const bool vec = inter % 8 == 0 && ((uintptr_t)value_gate | (uintptr_t)d_out | (uintptr_t)d_value_gate) % 16 == 0;
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "geglu_backward", [&](auto tag) {
        return launch_geglu_bwd<typename decltype(tag)::type>(value_gate, d_out, d_value_gate, rows, inter, vec,
                                                              (cudaStream_t)stream);
    });
}

extern "C" int mmfs_layernorm_backward(const void *x, const void *weight, const void *dy, void *dx, void *dweight, void *dbias,
                                       float *partials, long rows, int cols, float eps, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && cols > 0, "layernorm_backward: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && weight && dy && dx && (!(dweight || dbias) || partials), "layernorm_backward: null pointer argument");
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16) || cols % 8 != 0 || cols > kRmsBwdMaxCols ||
        ((uintptr_t)x | (uintptr_t)weight | (uintptr_t)dy | (uintptr_t)dx) % 16 != 0) {
        set_error("layernorm_backward: needs bf16 / f16, cols %% 8 == 0, cols <= %d, 16-byte aligned rows (got cols=%d dtype=%d)",
                  kRmsBwdMaxCols, cols, dtype);
        return MMFS_EUNSUPPORTED;
    }
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "layernorm_backward", [&](auto tag) {
        return launch_layernorm_bwd<typename decltype(tag)::type>(x, weight, dy, dx, dweight, dbias, partials, rows, cols, eps,
                                                                  (cudaStream_t)stream);
    });
}
