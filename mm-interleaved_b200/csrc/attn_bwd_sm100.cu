// attn_bwd_sm100.cu -- gradient of O = softmax(Q K^T * scale + mask) V (head dim 64 or 128, causal or not, key padding)
// on the tensor cores.
//
// The training path of LlamaAttention (decoders/modeling_llama_mmfs.py:246-264 under autograd: causal, hd 128, Tq = Tkv)
// and of the Q-Former's self- and cross-attention (non-causal, hd 64, Tq = 64 queries over Tkv = 64 queries or 257
// image tokens).  Flash-attention backward with P recomputed from the row log-sum-exp that mmfs_attn_forward_lse saved,
// in three launches:
//   1. delta:  D[b,h,i] = rowsum(dO * O) in fp32;
//   2. dK, dV: one CTA per 64-key tile walks the query tiles that can see it (q >= k0 under causality),
//              S^T = K Q^T, P^T = exp2(S^T * scale*log2e - LSE*log2e), dV += P^T dO, dP^T = V dO^T,
//              dS^T = P^T * (dP^T - D), dK += dS^T Q;
//   3. dQ:     one CTA per 64-query tile walks the key tiles it sees: S, P, dP = dO V^T, dS, dQ += dS K.
// Every output element is owned by one thread and accumulated in a fixed order: no atomics, so two runs give
// bit-identical gradients (the project's rule for its backward kernels, cf. msda_bwd_sm100.cu).  P is recomputed once
// per pass instead of accumulating dQ with atomics in pass 2.  Q and K / V may have different lengths and strides
// (cross-attention); causality assumes Tq = Tkv.
//
// MMA: mma.sync m16n8k16 (fp32 accumulators) fed by ldmatrix from padded shared-memory tiles.  The five products need
// Q, K, V and dO both K-major and MN-major; ldmatrix(.trans) gives either from one row-major tile, and the 16-bit
// register fragments of P^T / dS^T feed the next MMA as its A operand directly.  4 warps x 16 rows per CTA.
// Tiles stay 64 rows at hd 64: the pass-2 accumulators (dK, dV) halve to 64 floats per thread and the four tiles to
// 36 KB of shared memory, so several CTAs share an SM (DESIGN.md section 4.7 lists registers and occupancy).
#include "attn_common.cuh"

namespace mmfs {

namespace {

constexpr int kBwdBlk = 64;              // rows of every tile (queries or keys)
constexpr int kBwdThreads = 128;
// shared-memory row pitch in elements: 272 B (hd 128) / 144 B (hd 64), ldmatrix without bank conflicts
template <int HD> constexpr int kBwdLd = HD + 8;
template <int HD> constexpr int kBwdTile = kBwdBlk * kBwdLd<HD>;
template <int HD> constexpr size_t kBwdSmem = 4 * kBwdTile<HD> * 2 + 2 * kBwdBlk * sizeof(float) + kBwdBlk;

struct AttnBwdParams {
    const void *q, *k, *v, *dout;
    const float *lse, *delta;            // (B, H, T)
    void *dq, *dk, *dv;
    const uint8_t *key_mask;             // (B, Tkv) or null
    int H, Tq;
    long q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, do_bs, do_ts, dq_bs, dq_ts, dk_bs, dk_ts, dv_bs, dv_ts;
    float scale, scale_log2e;
    int Tkv;                             // read by the non-causal kernels only (causal: Tkv = Tq)
};

// keys of the problem: Tq under causality (read where used, as the causal kernels always did)
template <bool CAUSAL> __host__ __device__ __forceinline__ int kv_len(const AttnBwdParams &p) { return CAUSAL ? p.Tq : p.Tkv; }

__device__ __forceinline__ void cp_async16(void *dst, const void *src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s_addr(dst)), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void *p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s_addr(p)));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void *p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s_addr(p)));
}

// D(16x8) += A(16x16, row) * B(16x8, col); fragments as in the PTX ISA (g = lane / 4, t = lane % 4):
//   a = {(g, 2t..), (g+8, 2t..), (g, 2t+8..), (g+8, 2t+8..)}, b = {(k 2t.., n g), (k 2t+8.., n g)},
//   d = {(g, 2t), (g, 2t+1), (g+8, 2t), (g+8, 2t+1)}.
template <typename T> __device__ __forceinline__ void mma16816(float *d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mma16816<__nv_bfloat16>(float *d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void mma16816<__half>(float *d, const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// 64 rows x HD columns starting at row `row0` of a (T, ., hd) view into a padded tile; rows >= T are zero-filled
template <int HD, typename T>
__device__ __forceinline__ void load_tile(T *s, const T *g, long ts, int row0, int rows_total) {
    for (int i = threadIdx.x; i < kBwdBlk * (HD / 8); i += kBwdThreads) {
        constexpr int SH = HD == 128 ? 4 : 3;                 // log2 of the 16-byte chunks per row
        const int r = i >> SH, c = (i & ((1 << SH) - 1)) * 8;
        const bool ok = row0 + r < rows_total;
        cp_async16(s + r * kBwdLd<HD> + c, g + (ok ? (long)(row0 + r) * ts + c : 0), ok);
    }
}

// acc(16 x 64) = rows [16 warp, +16) of A-tile times the 64 rows of B-tile transposed, over the HD columns of both
// (A K-major, B "N rows of K": S = Q K^T, S^T = K Q^T, dP = dO V^T, dP^T = V dO^T)
template <int HD, typename T>
__device__ __forceinline__ void mma_abt(float (&acc)[32], const T *sA, const T *sB, int warp, int lane) {
    constexpr int LD = kBwdLd<HD>;
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
#pragma unroll
    for (int kk = 0; kk < HD / 16; ++kk) {
        uint32_t a[4];
        ldsm_x4(a, sA + (warp * 16 + (lane & 15)) * LD + kk * 16 + (lane >> 4) * 8);
#pragma unroll
        for (int np = 0; np < kBwdBlk / 16; ++np) {
            uint32_t b[4];
            ldsm_x4(b, sB + (np * 16 + (lane & 7) + ((lane >> 4) << 3)) * LD + kk * 16 + ((lane >> 3) & 1) * 8);
            mma16816<T>(acc + (2 * np) * 4, a, b[0], b[1]);
            mma16816<T>(acc + (2 * np + 1) * 4, a, b[2], b[3]);
        }
    }
}

// acc(16 x HD) += P(16 x 64, register fragments of an accumulator) times the 64 x HD B-tile (row-major: dV += P^T dO,
// dK += dS^T Q, dQ += dS K)
template <int HD, typename T>
__device__ __forceinline__ void mma_pb(float (&acc)[HD / 2], const float (&pf)[32], const T *sB, int lane) {
#pragma unroll
    for (int kk = 0; kk < kBwdBlk / 16; ++kk) {
        const uint32_t a[4] = {pack2<T>(pf[8 * kk + 0], pf[8 * kk + 1]), pack2<T>(pf[8 * kk + 2], pf[8 * kk + 3]),
                               pack2<T>(pf[8 * kk + 4], pf[8 * kk + 5]), pack2<T>(pf[8 * kk + 6], pf[8 * kk + 7])};
#pragma unroll
        for (int np = 0; np < HD / 16; ++np) {
            uint32_t b[4];
            ldsm_x4_t(b, sB + (kk * 16 + (lane & 15)) * kBwdLd<HD> + np * 16 + (lane >> 4) * 8);
            mma16816<T>(acc + (2 * np) * 4, a, b[0], b[1]);
            mma16816<T>(acc + (2 * np + 1) * 4, a, b[2], b[3]);
        }
    }
}

// rows [16 warp, +16) of a 16 x HD accumulator * mul -> (rows_total, ., hd) view at row row0
template <int HD, typename T>
__device__ __forceinline__ void store_rows(T *g, long ts, int row0, int rows_total, const float (&acc)[HD / 2], float mul,
                                           int warp, int lane) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = row0 + warp * 16 + (lane >> 2) + 8 * i;
        if (r >= rows_total) continue;
        T *dst = g + (long)r * ts + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < HD / 8; ++j)
            *reinterpret_cast<uint32_t *>(dst + 8 * j) = pack2<T>(acc[4 * j + 2 * i] * mul, acc[4 * j + 2 * i + 1] * mul);
    }
}

template <typename T, int HD>
__global__ void __launch_bounds__(256) attn_bwd_delta_kernel(const T *__restrict__ o, const T *__restrict__ dout,
                                                             float *__restrict__ delta, int H, int T_len, long rows,
                                                             long o_bs, long o_ts, long do_bs, long do_ts) {
    const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);       // (b, t, h), heads fastest
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const int h = (int)(row % H);
    const long bt = row / H;
    const int t = (int)(bt % T_len), b = (int)(bt / T_len);
    constexpr int PER = HD / 32;                                       // elements per lane
    const T *op = o + b * o_bs + t * o_ts + h * HD + PER * lane, *dp = dout + b * do_bs + t * do_ts + h * HD + PER * lane;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < PER; ++i) s = fmaf(to_op(op[i]), to_op(dp[i]), s);
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    if (lane == 0) delta[((long)b * H + h) * T_len + t] = s;
}

template <typename T, int HD, bool CAUSAL>
__global__ void __launch_bounds__(kBwdThreads) attn_bwd_dkdv_kernel(const AttnBwdParams p) {
    constexpr int TILE = kBwdTile<HD>;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    T *sK = reinterpret_cast<T *>(smem_raw), *sV = sK + TILE, *sQ = sV + TILE, *sdO = sQ + TILE;
    float *sL = reinterpret_cast<float *>(sdO + TILE), *sD = sL + kBwdBlk;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k0 = blockIdx.x * kBwdBlk, h = blockIdx.y, b = blockIdx.z;
    const T *q = static_cast<const T *>(p.q) + b * p.q_bs + h * HD;
    const T *dout = static_cast<const T *>(p.dout) + b * p.do_bs + h * HD;
    load_tile<HD>(sK, static_cast<const T *>(p.k) + b * p.k_bs + h * HD, p.k_ts, k0, kv_len<CAUSAL>(p));
    load_tile<HD>(sV, static_cast<const T *>(p.v) + b * p.v_bs + h * HD, p.v_ts, k0, kv_len<CAUSAL>(p));
    int key[2];
    bool kvis[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        key[i] = k0 + warp * 16 + (lane >> 2) + 8 * i;
        kvis[i] = key[i] < kv_len<CAUSAL>(p) && (p.key_mask == nullptr || p.key_mask[(long)b * kv_len<CAUSAL>(p) + key[i]] != 0);
    }
    const long lrow = ((long)b * p.H + h) * p.Tq;
    float dk[HD / 2], dv[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dk[i] = dv[i] = 0.f;

    for (int q0 = CAUSAL ? k0 : 0; q0 < p.Tq; q0 += kBwdBlk) {   // causal: queries below k0 see none of these keys
        __syncthreads();                                    // the previous tile's readers are done
        load_tile<HD>(sQ, q, p.q_ts, q0, p.Tq);
        load_tile<HD>(sdO, dout, p.do_ts, q0, p.Tq);
        if (threadIdx.x < kBwdBlk) {
            const int qi = q0 + threadIdx.x;                // rows past Tq: P = exp2(-inf) = 0
            sL[threadIdx.x] = qi < p.Tq ? p.lse[lrow + qi] * 1.4426950408889634f : INFINITY;
            sD[threadIdx.x] = qi < p.Tq ? p.delta[lrow + qi] : 0.f;
        }
        cp_async_wait_all();
        __syncthreads();

        float pt[32], dpt[32];
        mma_abt<HD>(pt, sK, sQ, warp, lane);                // S^T: rows = keys, columns = queries
#pragma unroll
        for (int j = 0; j < kBwdBlk / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int ql = 8 * j + 2 * (lane & 3) + c;
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const bool ok = kvis[i] && (!CAUSAL || key[i] <= q0 + ql);
                    float &e = pt[4 * j + 2 * i + c];
                    e = ok ? fast_exp2(fmaf(e, p.scale_log2e, -sL[ql])) : 0.f;   // fully masked row: LSE = +inf -> 0
                }
            }
        mma_pb<HD>(dv, pt, sdO, lane);                      // dV += P^T dO
        mma_abt<HD>(dpt, sV, sdO, warp, lane);              // dP^T = V dO^T
#pragma unroll
        for (int j = 0; j < kBwdBlk / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const float d = sD[8 * j + 2 * (lane & 3) + c];
#pragma unroll
                for (int i = 0; i < 2; ++i) dpt[4 * j + 2 * i + c] = pt[4 * j + 2 * i + c] * (dpt[4 * j + 2 * i + c] - d);
            }
        mma_pb<HD>(dk, dpt, sQ, lane);                      // dK += dS^T Q
    }
    store_rows<HD>(static_cast<T *>(p.dk) + b * p.dk_bs + h * HD, p.dk_ts, k0, kv_len<CAUSAL>(p), dk, p.scale, warp, lane);
    store_rows<HD>(static_cast<T *>(p.dv) + b * p.dv_bs + h * HD, p.dv_ts, k0, kv_len<CAUSAL>(p), dv, 1.f, warp, lane);
}

template <typename T, int HD, bool CAUSAL>
__global__ void __launch_bounds__(kBwdThreads) attn_bwd_dq_kernel(const AttnBwdParams p) {
    constexpr int TILE = kBwdTile<HD>;
    extern __shared__ __align__(16) uint8_t smem_raw[];
    T *sQ = reinterpret_cast<T *>(smem_raw), *sdO = sQ + TILE, *sK = sdO + TILE, *sV = sK + TILE;
    uint8_t *sKm = reinterpret_cast<uint8_t *>(sV + TILE) + 2 * kBwdBlk * sizeof(float);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * kBwdBlk, h = blockIdx.y, b = blockIdx.z;
    const T *k = static_cast<const T *>(p.k) + b * p.k_bs + h * HD;
    const T *v = static_cast<const T *>(p.v) + b * p.v_bs + h * HD;
    load_tile<HD>(sQ, static_cast<const T *>(p.q) + b * p.q_bs + h * HD, p.q_ts, q0, p.Tq);
    load_tile<HD>(sdO, static_cast<const T *>(p.dout) + b * p.do_bs + h * HD, p.do_ts, q0, p.Tq);
    const long lrow = ((long)b * p.H + h) * p.Tq;
    int row[2];
    float lse2[2], dl[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        row[i] = q0 + warp * 16 + (lane >> 2) + 8 * i;
        lse2[i] = row[i] < p.Tq ? p.lse[lrow + row[i]] * 1.4426950408889634f : INFINITY;
        dl[i] = row[i] < p.Tq ? p.delta[lrow + row[i]] : 0.f;
    }
    float dq[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) dq[i] = 0.f;
    // causal: keys past the tile's last query are never seen
    const int k_end = CAUSAL ? min(p.Tq, q0 + kBwdBlk) : kv_len<CAUSAL>(p);

    for (int k0 = 0; k0 < k_end; k0 += kBwdBlk) {
        __syncthreads();
        load_tile<HD>(sK, k, p.k_ts, k0, kv_len<CAUSAL>(p));
        load_tile<HD>(sV, v, p.v_ts, k0, kv_len<CAUSAL>(p));
        if (threadIdx.x < kBwdBlk) {
            const int kj = k0 + threadIdx.x;
            sKm[threadIdx.x] = kj < kv_len<CAUSAL>(p) && (p.key_mask == nullptr || p.key_mask[(long)b * kv_len<CAUSAL>(p) + kj] != 0);
        }
        cp_async_wait_all();
        __syncthreads();

        float s[32], dp[32];
        mma_abt<HD>(s, sQ, sK, warp, lane);                 // S = Q K^T
#pragma unroll
        for (int j = 0; j < kBwdBlk / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int kl = 8 * j + 2 * (lane & 3) + c;
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const bool ok = sKm[kl] && (!CAUSAL || k0 + kl <= row[i]);
                    float &e = s[4 * j + 2 * i + c];
                    e = ok ? fast_exp2(fmaf(e, p.scale_log2e, -lse2[i])) : 0.f;
                }
            }
        mma_abt<HD>(dp, sdO, sV, warp, lane);               // dP = dO V^T
#pragma unroll
        for (int j = 0; j < 32; ++j) dp[j] = s[j] * (dp[j] - dl[(j >> 1) & 1]);
        mma_pb<HD>(dq, dp, sK, lane);                       // dQ += dS K
    }
    store_rows<HD>(static_cast<T *>(p.dq) + b * p.dq_bs + h * HD, p.dq_ts, q0, p.Tq, dq, p.scale, warp, lane);
}

template <typename T, int HD, bool CAUSAL>
int launch_attn_bwd(const AttnBwdParams &p, const void *o, long o_bs, long o_ts, float *delta, int B, cudaStream_t st) {
    const long rows = (long)B * p.Tq * p.H;
    attn_bwd_delta_kernel<T, HD><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(
        static_cast<const T *>(o), static_cast<const T *>(p.dout), delta, p.H, p.Tq, rows, o_bs, o_ts, p.do_bs, p.do_ts);
    MMFS_CUDA(cudaGetLastError());
    constexpr size_t smem = kBwdSmem<HD>;
    int rc = ensure_dynamic_smem<attn_bwd_dkdv_kernel<T, HD, CAUSAL>>(smem);
    if (rc != MMFS_OK) return rc;
    if ((rc = ensure_dynamic_smem<attn_bwd_dq_kernel<T, HD, CAUSAL>>(smem)) != MMFS_OK) return rc;
    const int Tkv = kv_len<CAUSAL>(p);
    attn_bwd_dkdv_kernel<T, HD, CAUSAL><<<dim3((Tkv + kBwdBlk - 1) / kBwdBlk, p.H, B), kBwdThreads, smem, st>>>(p);
    MMFS_CUDA(cudaGetLastError());
    attn_bwd_dq_kernel<T, HD, CAUSAL><<<dim3((p.Tq + kBwdBlk - 1) / kBwdBlk, p.H, B), kBwdThreads, smem, st>>>(p);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

}  // namespace

// Checks shared by both entry points (after their shape checks), then the launch for (hd, causal).
static int attn_backward(const char *what, const void *q, const void *k, const void *v, const void *o, const void *d_out,
                         const float *lse, void *dq, void *dk, void *dv, float *delta, const uint8_t *key_mask, int B, int H,
                         int Tq, int Tkv, int hd, long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs,
                         long o_ts, long do_bs, long do_ts, long dq_bs, long dq_ts, long dk_bs, long dk_ts, long dv_bs,
                         long dv_ts, float scale, bool causal, int dtype, void *stream) {
    MMFS_CHECK_ARG(q && k && v && o && d_out && lse && dq && dk && dv && delta, "%s: null pointer argument", what);
    if (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)d_out | (uintptr_t)dq | (uintptr_t)dk | (uintptr_t)dv) % 16 != 0 ||
        (q_ts | k_ts | v_ts | do_ts | dq_ts | dk_ts | dv_ts | q_bs | k_bs | v_bs | do_bs | dq_bs | dk_bs | dv_bs) % 8 != 0 ||
        B > 65535 || H > 65535) {
        set_error("%s: q/k/v/dO/dQ/dK/dV pointers and strides must be 16-byte aligned; B, H <= 65535", what);
        return MMFS_EUNSUPPORTED;
    }
    AttnBwdParams p;
    p.q = q; p.k = k; p.v = v; p.dout = d_out; p.lse = lse; p.delta = delta; p.dq = dq; p.dk = dk; p.dv = dv;
    p.key_mask = key_mask; p.H = H; p.Tq = Tq; p.Tkv = Tkv;
    p.q_bs = q_bs; p.q_ts = q_ts; p.k_bs = k_bs; p.k_ts = k_ts; p.v_bs = v_bs; p.v_ts = v_ts; p.do_bs = do_bs; p.do_ts = do_ts;
    p.dq_bs = dq_bs; p.dq_ts = dq_ts; p.dk_bs = dk_bs; p.dk_ts = dk_ts; p.dv_bs = dv_bs; p.dv_ts = dv_ts;
    p.scale = scale; p.scale_log2e = scale * 1.4426950408889634f;
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, what, [&](auto tag) {
        using T = typename decltype(tag)::type;
        cudaStream_t st = (cudaStream_t)stream;
        if (hd == 64)
            return causal ? launch_attn_bwd<T, 64, true>(p, o, o_bs, o_ts, delta, B, st)
                          : launch_attn_bwd<T, 64, false>(p, o, o_bs, o_ts, delta, B, st);
        return causal ? launch_attn_bwd<T, 128, true>(p, o, o_bs, o_ts, delta, B, st)
                      : launch_attn_bwd<T, 128, false>(p, o, o_bs, o_ts, delta, B, st);
    });
}

}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_attn_backward(const void *q, const void *k, const void *v, const void *o, const void *d_out,
                                  const float *lse, void *dq, void *dk, void *dv, float *delta, const uint8_t *key_mask,
                                  int B, int H, int T, int hd, long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts,
                                  long o_bs, long o_ts, long do_bs, long do_ts, long dq_bs, long dq_ts, long dk_bs, long dk_ts,
                                  long dv_bs, long dv_ts, float scale, int dtype, void *stream) {
    MMFS_CHECK_ARG(B >= 0 && H > 0 && T >= 0 && hd > 0, "attn_backward: bad shape");
    if (B == 0 || T == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && o && d_out && lse && dq && dk && dv && delta, "attn_backward: null pointer argument");
    if (hd != 128 || !(dtype == MMFS_BF16 || dtype == MMFS_F16)) {
        set_error("attn_backward: needs hd = 128 and bf16 / f16 (got hd=%d dtype=%d)", hd, dtype);
        return MMFS_EUNSUPPORTED;
    }
    return attn_backward("attn_backward", q, k, v, o, d_out, lse, dq, dk, dv, delta, key_mask, B, H, T, T, hd, q_bs, q_ts,
                         k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, do_bs, do_ts, dq_bs, dq_ts, dk_bs, dk_ts, dv_bs, dv_ts, scale,
                         true, dtype, stream);
}

extern "C" int mmfs_attn_backward_general(const void *q, const void *k, const void *v, const void *o, const void *d_out,
                                          const float *lse, void *dq, void *dk, void *dv, float *delta,
                                          const uint8_t *key_mask, int B, int H, int Tq, int Tkv, int hd, long q_bs,
                                          long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                                          long do_bs, long do_ts, long dq_bs, long dq_ts, long dk_bs, long dk_ts, long dv_bs,
                                          long dv_ts, float scale, int causal, int dtype, void *stream) {
    MMFS_CHECK_ARG(B >= 0 && H > 0 && Tq > 0 && Tkv > 0 && hd > 0, "attn_backward_general: bad shape");
    MMFS_CHECK_ARG(!causal || Tq == Tkv, "attn_backward_general: causal attention needs Tq == Tkv (got %d, %d)", Tq, Tkv);
    if (B == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && o && d_out && lse && dq && dk && dv && delta, "attn_backward_general: null pointer argument");
    if (!(hd == 64 || hd == 128) || !(dtype == MMFS_BF16 || dtype == MMFS_F16)) {
        set_error("attn_backward_general: needs hd in {64, 128} and bf16 / f16 (got hd=%d dtype=%d)", hd, dtype);
        return MMFS_EUNSUPPORTED;
    }
    return attn_backward("attn_backward_general", q, k, v, o, d_out, lse, dq, dk, dv, delta, key_mask, B, H, Tq, Tkv, hd,
                         q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, do_bs, do_ts, dq_bs, dq_ts, dk_bs, dk_ts, dv_bs,
                         dv_ts, scale, causal != 0, dtype, stream);
}
