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
// read consecutive 16-byte vectors of a pixel row (coalesced).  Statistics are fp32 (count, mean, M2) -- M2 the sum of
// squared deviations from the mean -- merged in a fixed order (no atomics: results are reproducible run to run); the
// bf16 pipeline's rounding points (norm -> T, silu -> T) are kept so a bf16 run tracks diffusers' bf16 run.
//
// Why (count, mean, M2) and not sum / sum of squares: var = E[x^2] - mean^2 loses ~(mean/std)^2 ulps to cancellation,
// and a group whose mean is large next to its spread (flat image regions, outlier channels) is common: with that
// formula an fp32 group at mean/std = 16 came out 3e-4 off, at 4096 entirely wrong.  Each thread accumulates its pixels
// shifted by its first value (a sample of the group, so the shifted sums stay small), and the partial statistics are
// combined with Chan et al.'s pairwise update (GnMerge), whose error grows only linearly with mean/std -- the floor set
// by rounding the mean itself to fp32.
#include "common.cuh"

namespace mmfs {

template <typename T> __device__ __forceinline__ float gn_rnd(float x) { return to_op(from_op<T>(x)); }
template <> __device__ __forceinline__ float gn_rnd<float>(float x) { return x; }

constexpr int kGnMaxChunks = 64;     // pixel chunks per image: the partial-statistics scratch is (B, kGnMaxChunks, G, 2) floats

__device__ __forceinline__ float gn_warp_sum(float v) {   // butterfly: every lane ends with the same, fixed-order sum
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Parts i = 0..k-1 with (n_i, mean_i, M2_i) are merged in one pass, shifted by the first part's mean m_0 (Chan, Golub
// & LeVeque's pairwise update applied to k parts at once): with d_i = mean_i - m_0, S1 = sum n_i d_i, S2 = sum n_i d_i^2,
// mean = m_0 + S1 / n and M2 = sum M2_i + (S2 - S1^2 / n).  The d_i are of the order of the group's spread, so nothing
// cancels, and the loop has the shape of a plain sum: independent loads, one FMA chain per term, no division.
struct GnMerge {
    float m0 = 0.f, s1 = 0.f, s2 = 0.f, q = 0.f;
    __device__ __forceinline__ void add(float n, float mean, float m2) {
        const float d = mean - m0;
        s1 = fmaf(n, d, s1);
        s2 = fmaf(n * d, d, s2);
        q += m2;
    }
    __device__ __forceinline__ void finish(float n, float &mean, float &m2) const {
        const float d = s1 / n;
        mean = m0 + d;
        m2 = q + fmaxf(fmaf(-s1, d, s2), 0.f);
    }
};

// Pass 1: per (image, pixel chunk) mean and M2 of every group, written (not accumulated) to partial[b][chunk][g][0..1];
// the counts follow from (HW, ppb, C / G).  All merges run in a fixed order -- registers over a thread's pixels, shared
// memory over the pixel lanes of a channel, then over the channels of a group -- so the result is bit-reproducible run
// to run (the first version used shared + global float atomics, whose order is not).
template <typename T>
__global__ void __launch_bounds__(1024) gn_stats_kernel(const T *__restrict__ x, float *__restrict__ partial, int HW, int C,
                                                         int G, int ppb, int cvecs, int lanes) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dyn[];                     // [lanes][C][2] thread (mean, M2), then [C][2] channel stats in place of lane 0
    const int b = blockIdx.y, p0 = blockIdx.x * ppb, p1 = min(HW, p0 + ppb);
    const int cv = threadIdx.x % cvecs, pl = threadIdx.x / cvecs;
    const int np = p1 - p0;                              // pixels of this chunk; lane l takes pixels p0 + l, p0 + l + lanes, ...
    auto lane_count = [&](int l) { return l < np ? (np - l + lanes - 1) / lanes : 0; };
    float piv[VEC], s[VEC], ss[VEC];                     // sums of (x - piv) and (x - piv)^2, piv = the thread's first value
#pragma unroll
    for (int k = 0; k < VEC; ++k) piv[k] = s[k] = ss[k] = 0.f;
    const T *base = x + ((size_t)b * HW) * C + (size_t)cv * VEC;
    if (pl < lanes) {
        int p = p0 + pl;
        bool first = true;                               // the pivot is taken from the first batch (its own term is 0)
        for (; p + 3 * lanes < p1; p += 4 * lanes) {     // four independent 16-byte loads in flight
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = ldg_nc_v4(base + (size_t)(p + u * lanes) * C);
            if (first) { Vec16<T>::unpack(v[0], piv); first = false; }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                float f[VEC];
                Vec16<T>::unpack(v[u], f);
#pragma unroll
                for (int k = 0; k < VEC; ++k) { const float d = f[k] - piv[k]; s[k] += d; ss[k] = fmaf(d, d, ss[k]); }
            }
        }
        for (; p < p1; p += lanes) {
            float f[VEC];
            Vec16<T>::unpack(ldg_nc_v4(base + (size_t)p * C), f);
            if (first) {
#pragma unroll
                for (int k = 0; k < VEC; ++k) piv[k] = f[k];
                first = false;
            }
#pragma unroll
            for (int k = 0; k < VEC; ++k) { const float d = f[k] - piv[k]; s[k] += d; ss[k] = fmaf(d, d, ss[k]); }
        }
        const int n = lane_count(pl);
        const float inv = n > 0 ? 1.f / (float)n : 0.f;
#pragma unroll
        for (int k = 0; k < VEC; ++k) {                  // shifted sums -> (mean, M2) of the thread's pixels
            const float ds = s[k] * inv;                 // mean - piv
            ss[k] = fmaxf(fmaf(-s[k], ds, ss[k]), 0.f);  // sum (x - piv)^2 - n (mean - piv)^2
            s[k] = piv[k] + ds;
        }
        float *mine = s_dyn + ((size_t)pl * C + (size_t)cv * VEC) * 2;
#pragma unroll
        for (int k = 0; k < VEC; ++k) { mine[2 * k] = s[k]; mine[2 * k + 1] = ss[k]; }
    }
    __syncthreads();
    if (pl == 0) {                                       // channel statistics over the pixel lanes, lane order
        GnMerge m[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) { m[k].m0 = s[k]; m[k].q = ss[k]; }   // lane 0 = this thread: d_0 = 0
        for (int l = 1; l < lanes; ++l) {
            const float *o = s_dyn + ((size_t)l * C + (size_t)cv * VEC) * 2;
            const float nl = (float)lane_count(l);
#pragma unroll
            for (int k = 0; k < VEC; ++k) m[k].add(nl, o[2 * k], o[2 * k + 1]);
        }
        float *mine = s_dyn + (size_t)cv * VEC * 2;      // only this thread reads or writes these columns here
#pragma unroll
        for (int k = 0; k < VEC; ++k) m[k].finish((float)np, mine[2 * k], mine[2 * k + 1]);
    }
    __syncthreads();
    const int cg = C / G;
    for (int g = threadIdx.x; g < G; g += blockDim.x) {  // group statistics over the group's channels (np pixels each), channel order
        const float *cs = s_dyn + (size_t)g * cg * 2;
        GnMerge m;
        m.m0 = cs[0];
        for (int c = 0; c < cg; ++c) m.add((float)np, cs[2 * c], cs[2 * c + 1]);
        float *out = partial + (((size_t)b * kGnMaxChunks + blockIdx.x) * G + g) * 2;
        m.finish((float)np * (float)cg, out[0], out[1]);
    }
}

// Image b's group statistics from pass 1's per-chunk partials: stats[2g] = mean, stats[2g + 1] = variance.  A warp per
// group, lane l taking chunks l and l + 32 (blockDim.x is a multiple of 32): one batch of loads, then fixed-order
// butterfly sums, so every lane -- and every run -- gets the same result.  The forward's apply kernel and the backward
// kernels share it, so the backward normalises with the forward's mean and variance bit for bit.
__device__ __forceinline__ void gn_image_stats(const float *__restrict__ partial, float *stats, int b, int HW, int G, int cg,
                                               int ppb, int chunks) {
    static_assert(kGnMaxChunks <= 64, "two chunks per lane");
    const int lane = threadIdx.x & 31;
    auto count = [&](int ch) { return (float)(min(HW, (ch + 1) * ppb) - ch * ppb) * (float)cg; };
    for (int g = threadIdx.x >> 5; g < G; g += blockDim.x >> 5) {
        const float *pg = partial + ((size_t)b * kGnMaxChunks * G + g) * 2;   // chunk ch at pg[ch * 2G]
        const int c0 = lane, c1 = lane + 32;
        const float ma = c0 < chunks ? pg[(size_t)c0 * 2 * G] : 0.f, qa = c0 < chunks ? pg[(size_t)c0 * 2 * G + 1] : 0.f;
        const float mb = c1 < chunks ? pg[(size_t)c1 * 2 * G] : 0.f, qb = c1 < chunks ? pg[(size_t)c1 * 2 * G + 1] : 0.f;
        GnMerge m;
        m.m0 = __shfl_sync(0xffffffffu, ma, 0);
        if (c0 < chunks) m.add(count(c0), ma, qa);
        if (c1 < chunks) m.add(count(c1), mb, qb);
        m.s1 = gn_warp_sum(m.s1);
        m.s2 = gn_warp_sum(m.s2);
        m.q = gn_warp_sum(m.q);
        if (lane == 0) {
            const float n = (float)HW * (float)cg;
            float mean, m2;
            m.finish(n, mean, m2);
            stats[2 * g] = mean;
            stats[2 * g + 1] = m2 / n;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(1024) gn_apply_kernel(const T *__restrict__ x, const T *__restrict__ gamma,
                                                         const T *__restrict__ beta, const float *__restrict__ partial,
                                                         T *__restrict__ y, int HW, int C, int G, int ppb, int cvecs, int lanes,
                                                         float eps, int silu, int chunks) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float stats[];                     // [G][2] mean, variance of this image (chunk order: reproducible)
    const int b = blockIdx.y, p0 = blockIdx.x * ppb, p1 = min(HW, p0 + ppb);
    const int cv = threadIdx.x % cvecs, pl = threadIdx.x / cvecs;
    const int cg = C / G;
    gn_image_stats(partial, stats, b, HW, G, cg, ppb, chunks);
    __syncthreads();
    if (pl >= lanes) return;
    float sc[VEC], sh[VEC];                              // y = x * (r * gamma) + (beta - mean * r * gamma)
    {
        float gm[VEC], bt[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) { gm[k] = 1.f; bt[k] = 0.f; }
        if (gamma) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(gamma + cv * VEC), gm);
        if (beta) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(beta + cv * VEC), bt);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const int g = (cv * VEC + k) / cg;
            sc[k] = rsqrtf(stats[2 * g + 1] + eps) * gm[k];
            sh[k] = fmaf(-stats[2 * g], sc[k], bt[k]);
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

// ---- backward (dx only): z = gamma xhat + beta, xhat = (x - mean) r, r = 1 / sqrt(var + eps);
// dz = dy, or with the SiLU dz = dy s (1 + z (1 - s)), s = sigmoid(z) at the z the forward rounded to T (what autograd of
// the 16-bit pipeline differentiates); g = dz gamma; dx = r (g - mean(g) - xhat mean(g xhat)) per (image, group).
// Pass 1 is the forward's statistics kernel with the forward's geometry, and both kernels below merge its partials with
// gn_image_stats, so mean and r are the forward's.  xhat is formed from x - mean, i.e. centred on the group's own mean:
// sum(g xhat) does not cancel however large mean / std is.  Per-thread sums are reduced over pixel lanes, then channels,
// then chunks, each in a fixed order -- no atomics, so dx is bit-reproducible run to run.

// Per-channel constants of one thread's 16-byte channel vector.
template <typename T>
struct GnBwdChannels {
    static constexpr int VEC = 16 / (int)sizeof(T);
    float mean[VEC], r[VEC], gm[VEC], sc[VEC], sh[VEC];
    __device__ __forceinline__ void load(const T *gamma, const T *beta, const float *stats, int cv, int cg, float eps) {
        float bt[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) { gm[k] = 1.f; bt[k] = 0.f; }
        if (gamma) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(gamma + cv * VEC), gm);
        if (beta) Vec16<T>::unpack(*reinterpret_cast<const uint4 *>(beta + cv * VEC), bt);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const int g = (cv * VEC + k) / cg;
            mean[k] = stats[2 * g];
            r[k] = rsqrtf(stats[2 * g + 1] + eps);
            sc[k] = r[k] * gm[k];                        // the forward's scale and shift: z below is its z bit for bit
            sh[k] = fmaf(-mean[k], sc[k], bt[k]);
        }
    }
    // g = dz gamma and xhat of element k with input f and incoming gradient d
    __device__ __forceinline__ void grad(int k, float f, float d, int silu, float &g, float &xh) const {
        float dz = d;
        if (silu) {
            const float z = gn_rnd<T>(fmaf(f, sc[k], sh[k]));
            const float s = 1.f / (1.f + expf(-z));
            dz = d * s * fmaf(z, 1.f - s, 1.f);
        }
        g = dz * gm[k];
        xh = (f - mean[k]) * r[k];
    }
};

// Pass 2: per (image, chunk, group) sum(g) and sum(g xhat), written to dpart[b][chunk][g][0..1].
template <typename T>
__global__ void __launch_bounds__(512) gn_bwd_reduce_kernel(const T *__restrict__ x, const T *__restrict__ dy,
                                                              const T *__restrict__ gamma, const T *__restrict__ beta,
                                                              const float *__restrict__ partial, float *__restrict__ dpart,
                                                              int HW, int C, int G, int ppb, int cvecs, int lanes, float eps,
                                                              int silu, int chunks) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dyn[];                     // [G][2] statistics, then [lanes][C][2] thread sums
    float *stats = s_dyn, *sums = s_dyn + 2 * G;
    const int b = blockIdx.y, p0 = blockIdx.x * ppb, p1 = min(HW, p0 + ppb);
    const int cv = threadIdx.x % cvecs, pl = threadIdx.x / cvecs;
    const int cg = C / G;
    gn_image_stats(partial, stats, b, HW, G, cg, ppb, chunks);
    __syncthreads();
    if (pl < lanes) {
        GnBwdChannels<T> ch;
        ch.load(gamma, beta, stats, cv, cg, eps);
        float sg[VEC], sgx[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) sg[k] = sgx[k] = 0.f;
        const size_t off = ((size_t)b * HW) * C + (size_t)cv * VEC;
        for (int p = p0 + pl; p < p1; p += lanes) {
            float f[VEC], d[VEC];
            Vec16<T>::unpack(ldg_nc_v4(x + off + (size_t)p * C), f);
            Vec16<T>::unpack(ldg_nc_v4(dy + off + (size_t)p * C), d);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
                float g, xh;
                ch.grad(k, f[k], d[k], silu, g, xh);
                sg[k] += g;
                sgx[k] = fmaf(g, xh, sgx[k]);
            }
        }
        float *mine = sums + ((size_t)pl * C + (size_t)cv * VEC) * 2;
#pragma unroll
        for (int k = 0; k < VEC; ++k) { mine[2 * k] = sg[k]; mine[2 * k + 1] = sgx[k]; }
    }
    __syncthreads();
    if (pl == 0) {                                       // channel sums over the pixel lanes, lane order
        float *mine = sums + (size_t)cv * VEC * 2;
        for (int l = 1; l < lanes; ++l) {
            const float *o = sums + ((size_t)l * C + (size_t)cv * VEC) * 2;
#pragma unroll
            for (int k = 0; k < 2 * VEC; ++k) mine[k] += o[k];
        }
    }
    __syncthreads();
    for (int g = threadIdx.x; g < G; g += blockDim.x) {  // group sums over the group's channels, channel order
        const float *cs = sums + (size_t)g * cg * 2;
        float a = 0.f, q = 0.f;
        for (int c = 0; c < cg; ++c) { a += cs[2 * c]; q += cs[2 * c + 1]; }
        float *out = dpart + (((size_t)b * kGnMaxChunks + blockIdx.x) * G + g) * 2;
        out[0] = a;
        out[1] = q;
    }
}

// Pass 3: merge pass 2's chunk sums per group (a warp per group, as gn_image_stats), then dx.
template <typename T>
__global__ void __launch_bounds__(512) gn_bwd_apply_kernel(const T *__restrict__ x, const T *__restrict__ dy,
                                                             const T *__restrict__ gamma, const T *__restrict__ beta,
                                                             const float *__restrict__ partial, const float *__restrict__ dpart,
                                                             T *__restrict__ dx, int HW, int C, int G, int ppb, int cvecs,
                                                             int lanes, float eps, int silu, int chunks) {
    constexpr int VEC = 16 / (int)sizeof(T);
    extern __shared__ float s_dyn[];                     // [G][2] statistics, [G][2] mean(g), mean(g xhat)
    float *stats = s_dyn, *gmeans = s_dyn + 2 * G;
    const int b = blockIdx.y, p0 = blockIdx.x * ppb, p1 = min(HW, p0 + ppb);
    const int cv = threadIdx.x % cvecs, pl = threadIdx.x / cvecs;
    const int cg = C / G;
    gn_image_stats(partial, stats, b, HW, G, cg, ppb, chunks);
    const int lane = threadIdx.x & 31;
    for (int g = threadIdx.x >> 5; g < G; g += blockDim.x >> 5) {
        const float *pg = dpart + ((size_t)b * kGnMaxChunks * G + g) * 2;
        float a = 0.f, q = 0.f;
        if (lane < chunks) { a = pg[(size_t)lane * 2 * G]; q = pg[(size_t)lane * 2 * G + 1]; }
        if (lane + 32 < chunks) { a += pg[(size_t)(lane + 32) * 2 * G]; q += pg[(size_t)(lane + 32) * 2 * G + 1]; }
        a = gn_warp_sum(a);
        q = gn_warp_sum(q);
        if (lane == 0) {
            const float inv_n = 1.f / ((float)HW * (float)cg);
            gmeans[2 * g] = a * inv_n;
            gmeans[2 * g + 1] = q * inv_n;
        }
    }
    __syncthreads();
    if (pl >= lanes) return;
    GnBwdChannels<T> ch;
    ch.load(gamma, beta, stats, cv, cg, eps);
    float mg[VEC], mgx[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
        const int g = (cv * VEC + k) / cg;
        mg[k] = gmeans[2 * g];
        mgx[k] = gmeans[2 * g + 1];
    }
    const size_t off = ((size_t)b * HW) * C + (size_t)cv * VEC;
    for (int p = p0 + pl; p < p1; p += lanes) {
        float f[VEC], d[VEC], o[VEC];
        Vec16<T>::unpack(ldg_nc_v4(x + off + (size_t)p * C), f);
        Vec16<T>::unpack(ldg_nc_v4(dy + off + (size_t)p * C), d);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            float g, xh;
            ch.grad(k, f[k], d[k], silu, g, xh);
            o[k] = ch.r[k] * fmaf(-xh, mgx[k], g - mg[k]);
        }
        stg_v4(dx + off + (size_t)p * C, Vec16<T>::pack(o));
    }
}

// Launch geometry shared by the forward and the backward (the backward's pass 1 must see the forward's chunks): thread
// t owns channel vector t % cvecs of pixels p0 + t / cvecs, + lanes, ...; `chunks` CTAs of ppb pixels per image.
struct GnGeometry {
    int cvecs, lanes, threads, ppb, chunks;
};

template <typename T>
static GnGeometry gn_geometry(int B, int HW, int C) {
    constexpr int VEC = 16 / (int)sizeof(T);
    GnGeometry g;
    g.cvecs = C / VEC;
    g.lanes = max(1, min(HW, 512 / g.cvecs));
    g.threads = g.cvecs * g.lanes;
    const int target_blocks = max(1, (num_sms() * 8) / B);               // ~8 CTAs' worth of work per SM over the batch
    int ppb = max(g.lanes * 4, (HW + target_blocks - 1) / target_blocks);
    ppb = max(ppb, (HW + kGnMaxChunks - 1) / kGnMaxChunks);
    g.ppb = min(ppb, HW);
    g.chunks = (HW + g.ppb - 1) / g.ppb;                 // <= kGnMaxChunks
    return g;
}

template <typename T>
static int gn_stats_launch(const void *x, float *stats, int B, int HW, int C, int G, const GnGeometry &g, cudaStream_t st) {
    const size_t smem_stats = (size_t)g.lanes * C * 2 * sizeof(float);
    constexpr auto kern = gn_stats_kernel<T>;
    const int rc = ensure_dynamic_smem<kern>(smem_stats);
    if (rc != MMFS_OK) return rc;
    kern<<<dim3(g.chunks, B), g.threads, smem_stats, st>>>((const T *)x, stats, HW, C, G, g.ppb, g.cvecs, g.lanes);
    return MMFS_OK;
}

template <typename T>
static int gn_launch(const void *x, const void *gamma, const void *beta, void *y, float *stats, int B, int HW, int C, int G,
                     float eps, int silu, cudaStream_t st) {
    const GnGeometry g = gn_geometry<T>(B, HW, C);
    const int rc = gn_stats_launch<T>(x, stats, B, HW, C, G, g, st);
    if (rc != MMFS_OK) return rc;
    // whole warps for the chunk merge; the padding threads (pl >= lanes) leave after it
    gn_apply_kernel<T><<<dim3(g.chunks, B), (g.threads + 31) / 32 * 32, 2 * G * sizeof(float), st>>>(
        (const T *)x, (const T *)gamma, (const T *)beta, stats, (T *)y, HW, C, G, g.ppb, g.cvecs, g.lanes, eps, silu, g.chunks);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int gn_bwd_launch(const void *x, const void *gamma, const void *beta, const void *dy, void *dx, float *scratch, int B,
                         int HW, int C, int G, float eps, int silu, cudaStream_t st) {
    const GnGeometry g = gn_geometry<T>(B, HW, C);
    float *stats = scratch, *dpart = scratch + (size_t)B * kGnMaxChunks * G * 2;
    int rc = gn_stats_launch<T>(x, stats, B, HW, C, G, g, st);
    if (rc != MMFS_OK) return rc;
    const dim3 grid(g.chunks, B);
    const int threads = (g.threads + 31) / 32 * 32;
    const size_t smem_reduce = (2 * (size_t)G + (size_t)g.lanes * C * 2) * sizeof(float);
    constexpr auto reduce = gn_bwd_reduce_kernel<T>;
    rc = ensure_dynamic_smem<reduce>(smem_reduce);
    if (rc != MMFS_OK) return rc;
    reduce<<<grid, threads, smem_reduce, st>>>((const T *)x, (const T *)dy, (const T *)gamma, (const T *)beta, stats, dpart,
                                               HW, C, G, g.ppb, g.cvecs, g.lanes, eps, silu, g.chunks);
    gn_bwd_apply_kernel<T><<<grid, threads, 4 * G * sizeof(float), st>>>(
        (const T *)x, (const T *)dy, (const T *)gamma, (const T *)beta, stats, dpart, (T *)dx, HW, C, G, g.ppb, g.cvecs,
        g.lanes, eps, silu, g.chunks);
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

extern "C" int mmfs_groupnorm_nhwc_backward(const void *x, const void *gamma, const void *beta, const void *dy, void *dx,
                                            float *scratch, int B, int HW, int C, int G, float eps, int silu, int dtype,
                                            void *stream) {
    using namespace mmfs;
    MMFS_CHECK_ARG(x && dy && dx && scratch, "groupnorm_backward: null pointer");
    MMFS_CHECK_ARG(B > 0 && HW > 0 && C > 0 && G > 0 && C % G == 0 && B <= 65535,
                   "groupnorm_backward: bad sizes B=%d HW=%d C=%d G=%d", B, HW, C, G);
    const size_t es = dtype_size(dtype);
    if (dtype == MMFS_F64 || es == 0 || C % (16 / (int)es) != 0 || C / (16 / (int)es) > 512) {
        set_error("groupnorm_backward: unsupported dtype %d / channel count %d (need C %% (16/sizeof) == 0, C*sizeof <= 8 KiB)",
                  dtype, C);
        return MMFS_EUNSUPPORTED;
    }
    if (((uintptr_t)x | (uintptr_t)dy | (uintptr_t)dx | (uintptr_t)gamma | (uintptr_t)beta) % 16 != 0) {
        set_error("groupnorm_backward: x, dy, dx, gamma and beta must be 16-byte aligned");
        return MMFS_EUNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kF32Types>(dtype, "groupnorm_backward", [&](auto tag) {
        return gn_bwd_launch<typename decltype(tag)::type>(x, gamma, beta, dy, dx, scratch, B, HW, C, G, eps, silu, st);
    });
}
