// llama_ops_sm100.cu -- HBM-bound element-wise / row-wise kernels of the Llama-MMFS decoder layer.
//
//   mmfs_rmsnorm      LlamaRMSNorm.forward               decoders/modeling_llama_mmfs.py:53-70
//   mmfs_rope_qk      apply_rotary_pos_emb / rotate_half decoders/modeling_llama_mmfs.py:158-172
//   mmfs_swiglu       LlamaMLP: act_fn(gate) * up        decoders/modeling_llama_mmfs.py:188-189
//   mmfs_layernorm    nn.LayerNorm (CLIP / Q-Former / MMFSBlock norms)
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
static int launch_all(int which, const void *a, const void *b, const void *c, void *d, const void *e, const void *f,
                      long n0, int i0, int i1, int i2, int i3, int i4, int i5, float eps, cudaStream_t st) {
    (void)i5;
    switch (which) {
        case 0:   // rmsnorm: a=x b=w d=y n0=rows i0=cols
            if (i0 % (16 / (int)sizeof(T)) == 0 && i0 / (16 / (int)sizeof(T)) <= kRmsThreads * kRmsChunks)
                rmsnorm_reg_kernel<T><<<(unsigned)n0, kRmsThreads, 0, st>>>((const T *)a, (const T *)b, (T *)d, i0, eps);
            else
                rmsnorm_kernel<T><<<(unsigned)n0, 256, 0, st>>>((const T *)a, (const T *)b, (T *)d, i0, eps);
            break;
        case 1: { // layernorm: a=x b=w c=bias d=y
            constexpr int VEC = 16 / (int)sizeof(T);
            const bool vec_ok = (i0 % VEC == 0) && (i0 / VEC <= 32 * kLnChunks) &&
                                (((uintptr_t)a | (uintptr_t)d | (uintptr_t)b | (uintptr_t)c) % 16 == 0);
            if (vec_ok) {
                const int nvec = i0 / VEC;
                const unsigned grid = (unsigned)((n0 + 7) / 8);
#define MMFS_LN(CH) layernorm_warp_kernel<T, CH><<<grid, 256, 0, st>>>((const T *)a, (const T *)b, (const T *)c, (T *)d, n0, i0, eps)
                if (nvec <= 32) MMFS_LN(1); else if (nvec <= 64) MMFS_LN(2); else if (nvec <= 128) MMFS_LN(4); else MMFS_LN(8);
#undef MMFS_LN
            } else
                layernorm_kernel<T><<<(unsigned)n0, 256, 0, st>>>((const T *)a, (const T *)b, (const T *)c, (T *)d, i0, eps);
            break;
        }
        case 2: { // rope: d=q (in place), a=k (in place, cast away const), e=cos f=sin c=pos; n0=tokens i0=H i1=hd i2=q_stride i3=k_stride i4=pos_per_batch i5=T
            const int per_tok = i0 * 2 * ((i1 / 2) / (16 / (int)sizeof(T)));
            const int threads = per_tok >= 256 ? 256 : ((per_tok + 31) / 32) * 32;
            const int grid = (int)(n0 < (long)num_sms() * 32 ? n0 : (long)num_sms() * 32);
            rope_qk_kernel<T><<<grid, threads, 0, st>>>((T *)d, (T *)const_cast<void *>(a), (const float *)e, (const float *)f,
                                                     (const int64_t *)c, n0, i0, i1, i2, i3, i4, i5);
            break;
        }
        case 3: { // swiglu / geglu: a=gate_up d=out n0=rows i0=I i1=variant (0 silu [gate|up], 1 gelu [value|gate])
            const int nvec = i0 / (16 / (int)sizeof(T));
            const int threads = nvec >= 512 ? 256 : (nvec >= 64 ? 64 : 32);
            const int gx = (int)(n0 < (long)num_sms() * 64 ? n0 : (long)num_sms() * 64);
            int gy = 1;                                   // fewer CTAs than SMs: slice the columns (two vectors per thread)
            if (gx < num_sms()) { gy = (nvec + 2 * threads - 1) / (2 * threads); if (gy > 64) gy = 64; if (gy < 1) gy = 1; }
            const dim3 grid(gx, gy);
            if (i1 == 1)
                swiglu_kernel<T, 1, true><<<grid, threads, 0, st>>>((const T *)a, (T *)d, n0, i0);
            else
                swiglu_kernel<T, 0, false><<<grid, threads, 0, st>>>((const T *)a, (T *)d, n0, i0);
            break;
        }
    }
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

static int dispatch(int dtype, int which, const void *a, const void *b, const void *c, void *d, const void *e, const void *f,
                    long n0, int i0, int i1, int i2, int i3, int i4, int i5, float eps, void *stream) {
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case MMFS_F32: return launch_all<float>(which, a, b, c, d, e, f, n0, i0, i1, i2, i3, i4, i5, eps, st);
        case MMFS_F16: return launch_all<__half>(which, a, b, c, d, e, f, n0, i0, i1, i2, i3, i4, i5, eps, st);
        case MMFS_BF16: return launch_all<__nv_bfloat16>(which, a, b, c, d, e, f, n0, i0, i1, i2, i3, i4, i5, eps, st);
        default: set_error("dtype %d not supported by this kernel", dtype); return MMFS_EINVAL;
    }
}

}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_rmsnorm(const void *x, const void *weight, void *y, long rows, int cols, float eps, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && cols > 0, "rmsnorm: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && weight && y, "rmsnorm: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)x | (uintptr_t)weight | (uintptr_t)y) % 16 == 0 && (cols * dtype_size(dtype)) % 16 == 0,
                   "rmsnorm: rows must be 16-byte aligned");
    return dispatch(dtype, 0, x, weight, nullptr, y, nullptr, nullptr, rows, cols, 0, 0, 0, 0, 0, eps, stream);
}

extern "C" int mmfs_layernorm(const void *x, const void *weight, const void *bias, void *y, long rows, int cols, float eps,
                              int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && cols > 0, "layernorm: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && y, "layernorm: null pointer argument");
    return dispatch(dtype, 1, x, weight, bias, y, nullptr, nullptr, rows, cols, 0, 0, 0, 0, 0, eps, stream);
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
    return dispatch(dtype, 2, k, nullptr, position_ids, q, cos_table, sin_table, n_tokens, H, hd, q_stride, k_stride,
                    pos_per_batch, T_len, 0.f, stream);
}

template <typename T>
static int launch_rope_append(void *q, const void *k, const void *v, const float *cos_t, const float *sin_t, const int64_t *pos,
                              void *kc, void *vc, const int64_t *slot_dev, long slot_host, long n_tok, int T_len, int H, int hd,
                              int qs, int ks, int vs, long cbs, long cts, int ppb, cudaStream_t st) {
    const int items = H * ((hd / 2) / (16 / (int)sizeof(T))) * 2 + H * hd / (16 / (int)sizeof(T));
    const int threads = items >= 256 ? 256 : ((items + 31) / 32) * 32;
    const int grid = (int)(n_tok < (long)num_sms() * 32 ? n_tok : (long)num_sms() * 32);
    rope_append_kernel<T><<<grid, threads, 0, st>>>((T *)q, (const T *)k, (const T *)v, cos_t, sin_t, pos, (T *)kc, (T *)vc, slot_dev,
                                                 slot_host, n_tok, H, hd, qs, ks, vs, cbs, cts, ppb, T_len);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
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
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case MMFS_F32: return launch_rope_append<float>(q, k, v, cos_table, sin_table, position_ids, k_cache, v_cache, slot_dev, slot_host, n_tokens, T_len, H, hd, q_stride, k_stride, v_stride, cache_bs, cache_ts, pos_per_batch, st);
        case MMFS_F16: return launch_rope_append<__half>(q, k, v, cos_table, sin_table, position_ids, k_cache, v_cache, slot_dev, slot_host, n_tokens, T_len, H, hd, q_stride, k_stride, v_stride, cache_bs, cache_ts, pos_per_batch, st);
        case MMFS_BF16: return launch_rope_append<__nv_bfloat16>(q, k, v, cos_table, sin_table, position_ids, k_cache, v_cache, slot_dev, slot_host, n_tokens, T_len, H, hd, q_stride, k_stride, v_stride, cache_bs, cache_ts, pos_per_batch, st);
        default: set_error("rope_qk_append: dtype %d unsupported", dtype); return MMFS_EINVAL;
    }
}

extern "C" int mmfs_swiglu(const void *gate_up, void *out, long rows, int inter, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && inter > 0, "swiglu: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(gate_up && out, "swiglu: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)gate_up | (uintptr_t)out) % 16 == 0 && (inter * dtype_size(dtype)) % 16 == 0,
                   "swiglu: rows must be 16-byte aligned");
    return dispatch(dtype, 3, gate_up, nullptr, nullptr, out, nullptr, nullptr, rows, inter, 0, 0, 0, 0, 0, 0.f, stream);
}

extern "C" int mmfs_geglu(const void *value_gate, void *out, long rows, int inter, int dtype, void *stream) {
    MMFS_CHECK_ARG(rows >= 0 && inter > 0, "geglu: bad shape");
    if (rows == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value_gate && out, "geglu: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)value_gate | (uintptr_t)out) % 16 == 0 && (inter * dtype_size(dtype)) % 16 == 0,
                   "geglu: rows must be 16-byte aligned");
    return dispatch(dtype, 3, value_gate, nullptr, nullptr, out, nullptr, nullptr, rows, inter, 1, 0, 0, 0, 0, 0.f, stream);
}
