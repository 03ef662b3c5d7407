// attn_fwd_sm100.cu -- softmax(Q K^T * scale + mask) V on the Hopper tensor cores (wgmma).
//
// Replaces, for prefill-sized problems,
//   LlamaAttention.forward's eager path      decoders/modeling_llama_mmfs.py:246-264
//       (matmul -> +mask -> max(finfo.min) -> fp32 softmax -> matmul, (B,40,T,T) scores materialised)
//   CLIPXAttention.forward                   encoders/vit_adapter/xattn.py:47-141 (xformers
//       memory_efficient_attention, non-causal, T = 257, 16 x 64)
//   the SD-UNet self-/cross-attention        decoders/sd.py:64-65 (xformers)
//
// Design (hand-written PTX, no CUTLASS):
//   * one work item = (128 query rows, head, batch entry); Q / K / V tiles arrive by TMA (cp.async.bulk.tensor.4d,
//     SWIZZLE_128B) straight from the projection GEMM's (B, T, H, hd) layout -- no transposes, K and V double-buffered;
//   * warps 0-3 and 4-7 are two consumer warpgroups of 64 query rows each, warp 8 is the TMA producer;
//   * S = Q K^T is wgmma m64n64k16 with both operands in shared memory; the online softmax runs on the fp32
//     accumulator fragment in registers (row max / sum over the 4 lanes of a quad), P is packed to 16 bit in
//     registers and fed to O += P V as the register A operand (wgmma m64n{hd}k16, V MN-major exactly as TMA
//     delivers it); O stays in registers for the whole item;
//   * causal tiles above the diagonal are never loaded; causal / key-padding / tail masks are applied on the
//     scores in registers; the (B,1,T,T) additive mask is never built.
// One CTA per SM at hd 128 (139 registers per thread), two at hd 64.  With more items than resident CTAs the kernel
// is persistent: the producer hands out items through an atomic counter (longest causal query tile first, heads
// fastest inside a batch entry, so that the resident CTAs share one batch entry's K / V in L2), and every
// barrier phase runs on a global tile counter, so the K / V ring continues across items without a drain.
#include "attn_common.cuh"

namespace mmfs {

constexpr int kBM = 128, kBN = 64;
constexpr int kAttnThreads = 288;   // warpgroups 0, 1: softmax + MMA; warp 8: TMA producer
constexpr int kConsumers = 256;

// Shared memory (dynamic, 1024-byte aligned):
//   Q [HD/64 boxes][128 rows][128 B] | K [2 stages][HD/64][64][128 B] | V [2][HD/64][64][128 B] | barriers | items [2]
template <int HD> constexpr int attn_ctas_per_sm() { return HD == 64 ? 2 : 1; }

template <typename T, int HD>
__global__ void __launch_bounds__(kAttnThreads, attn_ctas_per_sm<HD>())
attn_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                const __grid_constant__ CUtensorMap map_v, const AttnParams p, unsigned *__restrict__ sched, int n_work) {
    constexpr int NBOX = HD / 64;
    constexpr uint32_t QBOX_BYTES = kBM * 128, KBOX_BYTES = kBN * 128;
    constexpr uint32_t Q_BYTES = NBOX * QBOX_BYTES, KV_BYTES = NBOX * KBOX_BYTES;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // SWIZZLE_128B tiles need 1024-byte alignment; the dynamic window starts at offset 0 of the CTA's shared memory
    // (no static __shared__ in this kernel), which the __align__ above requests.
    if ((s_addr(smem_raw) & 1023u) != 0u) { asm volatile("trap;"); }
    uint8_t *sQ = smem_raw;
    uint8_t *sK = sQ + Q_BYTES;
    uint8_t *sV = sK + 2 * KV_BYTES;
    uint64_t *bars = reinterpret_cast<uint64_t *>(sV + 2 * KV_BYTES);
    uint64_t *q_full = bars + 0, *q_empty = bars + 1, *k_full = bars + 2 /*[2]*/, *k_empty = bars + 4 /*[2]*/,
             *v_full = bars + 6 /*[2]*/, *v_empty = bars + 8 /*[2]*/, *item_full = bars + 10 /*[2]*/, *item_empty = bars + 12 /*[2]*/;
    int *s_item = reinterpret_cast<int *>(bars + 14);            // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_q = (p.Tq + kBM - 1) / kBM;
    // item w -> (batch, query tile, head): batch-major, longest tile first inside a batch entry, heads fastest
    auto decode = [&](int w, int &h, int &b, int &q0, int &n_tiles) {
        b = w / (n_q * p.H);
        const int r = w - b * (n_q * p.H);
        const int mi = r / p.H;
        h = r - mi * p.H;
        q0 = (p.causal ? n_q - 1 - mi : mi) * kBM;
        int kv_end = p.Tkv;
        if (p.causal) kv_end = min(p.Tkv, p.past + min(q0 + kBM, p.Tq));
        n_tiles = (kv_end + kBN - 1) / kBN;
    };

    if (threadIdx.x == 0) {
        bar_init(q_full, 1);
        bar_init(q_empty, kConsumers);
        for (int i = 0; i < 2; ++i) {
            bar_init(k_full + i, 1); bar_init(v_full + i, 1); bar_init(k_empty + i, kConsumers); bar_init(v_empty + i, kConsumers);
            bar_init(item_full + i, 1); bar_init(item_empty + i, kConsumers);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        // ============================== scheduler + TMA producer ==============================
        if (lane == 0) {
            int w = blockIdx.x;
            int g = 0;                                               // global tile counter
            for (int qn = 0;; ++qn) {
                const int slot = qn & 1;
                if (qn >= 2) bar_wait(item_empty + slot, ((qn >> 1) - 1) & 1);
                s_item[slot] = w < n_work ? w : -1;
                bar_arrive(item_full + slot);
                if (w >= n_work) break;
                // non-persistent launch: one item per CTA.  Persistent: fetched early, the latency hides under this item
                const int w_next = sched ? (int)gridDim.x + (int)atomicAdd(sched, 1u) : n_work;
                int h, b, q0, n_tiles;
                decode(w, h, b, q0, n_tiles);
                if (qn > 0) bar_wait(q_empty, (qn - 1) & 1);        // the previous item's S MMAs no longer read Q
                bar_expect_tx(q_full, Q_BYTES);
#pragma unroll
                for (int bx = 0; bx < NBOX; ++bx) tma_load_4d(sQ + bx * QBOX_BYTES, &map_q, q_full, bx * 64, h, q0, b);
                for (int j = 0; j < n_tiles; ++j, ++g) {
                    const int s = g & 1;
                    const uint32_t ph = (g >> 1) & 1;
                    bar_wait(k_empty + s, ph ^ 1);
                    bar_expect_tx(k_full + s, KV_BYTES);
#pragma unroll
                    for (int bx = 0; bx < NBOX; ++bx)
                        tma_load_4d(sK + s * KV_BYTES + bx * KBOX_BYTES, &map_k, k_full + s, bx * 64, h, j * kBN, b);
                    bar_wait(v_empty + s, ph ^ 1);
                    bar_expect_tx(v_full + s, KV_BYTES);
#pragma unroll
                    for (int bx = 0; bx < NBOX; ++bx)
                        tma_load_4d(sV + s * KV_BYTES + bx * KBOX_BYTES, &map_v, v_full + s, bx * 64, h, j * kBN, b);
                }
                w = w_next;
            }
        }
        return;
    }

    // ============================== consumer warpgroups: S, softmax, O ==============================
    const int wg = warp >> 2;                        // 64-row half of the query tile
    const int quad = lane >> 2, tq = lane & 3;
    const int row_in_tile = wg * 64 + (warp & 3) * 16 + quad;   // + 8 for the second row of the fragment
    const uint32_t q_base = s_addr(sQ) + wg * 64 * 128;
    int g = 0;
    for (int qn = 0;; ++qn) {
        const int slot = qn & 1;
        bar_wait(item_full + slot, (qn >> 1) & 1);
        const int w = s_item[slot];
        bar_arrive(item_empty + slot);
        if (w < 0) break;
        int h, b, q0, n_tiles;
        decode(w, h, b, q0, n_tiles);
        const int r0 = q0 + row_in_tile;             // rows r0 and r0 + 8
        float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l: this thread's columns only
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        bar_wait(q_full, qn & 1);
        if (n_tiles == 0) bar_arrive(q_empty);

        for (int j = 0; j < n_tiles; ++j, ++g) {
            const int s = g & 1;
            const int k0 = j * kBN;
            float sc[kBN / 2];
            bar_wait(k_full + s, (g >> 1) & 1);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < HD / 16; ++kk)     // 64-element box along hd, then 32 B inside the 128-byte swizzle atom
                Wgmma<T>::ss_n64(sc, smem_desc(q_base + (kk >> 2) * QBOX_BYTES + (kk & 3) * 32, 16, 1024),
                                 smem_desc(s_addr(sK) + s * KV_BYTES + (kk >> 2) * KBOX_BYTES + (kk & 3) * 32, 16, 1024), kk > 0);
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(sc);
            bar_arrive(k_empty + s);
            if (j + 1 == n_tiles) bar_arrive(q_empty);

            // masks: key padding, ragged tail, causality (key index <= past + query index)
            const bool need_mask = (k0 + kBN > p.Tkv) || (p.key_mask != nullptr) ||
                                   (p.causal && k0 + kBN - 1 > p.past + q0 + wg * 64);
            if (need_mask) {
#pragma unroll
                for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int key = k0 + jj * 8 + 2 * tq + c;
                        bool vis = key < p.Tkv;
                        if (vis && p.key_mask != nullptr) vis = p.key_mask[(long)b * p.Tkv + key] != 0;
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const bool ok = vis && (!p.causal || key <= p.past + r0 + 8 * i);
                            if (!ok) sc[jj * 4 + 2 * i + c] = -INFINITY;
                        }
                    }
            }
            float alpha[2], neg_m[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float mx = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < kBN / 8; ++jj) mx = fmaxf(mx, fmaxf(sc[jj * 4 + 2 * i], sc[jj * 4 + 2 * i + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[i], mx);
                alpha[i] = (m_new == -INFINITY) ? 1.f : fast_exp2((m_run[i] - m_new) * p.scale_log2e);   // exp2(-inf) = 0
                m_run[i] = m_new;
                neg_m[i] = (m_new == -INFINITY) ? 0.f : -m_new * p.scale_log2e;
            }
            // P = exp2(S * scale_log2e - m), packed to 16 bit as the A fragments of the four k16 steps of P V
            uint32_t pa[kBN / 16][4];
            float ls[2] = {0.f, 0.f};
#pragma unroll
            for (int jj = 0; jj < kBN / 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const float e0 = fast_exp2(fmaf(sc[jj * 4 + 2 * i], p.scale_log2e, neg_m[i]));   // masked: exp2(-inf) = 0
                    const float e1 = fast_exp2(fmaf(sc[jj * 4 + 2 * i + 1], p.scale_log2e, neg_m[i]));
                    ls[i] += e0 + e1;
                    pa[jj >> 1][(jj & 1) * 2 + i] = pack2<T>(e0, e1);
                }
#pragma unroll
            for (int i = 0; i < 2; ++i) l_run[i] = l_run[i] * alpha[i] + ls[i];
#pragma unroll
            for (int jj = 0; jj < HD / 8; ++jj) {
                o[jj * 4 + 0] *= alpha[0]; o[jj * 4 + 1] *= alpha[0];
                o[jj * 4 + 2] *= alpha[1]; o[jj * 4 + 3] *= alpha[1];
            }

            bar_wait(v_full + s, (g >> 1) & 1);
            reg_fence(o);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < kBN / 16; ++kk) {  // V: MN-major, 16 key rows of 128 B per k-step, hd boxes KBOX_BYTES apart
                const uint64_t dv = smem_desc(s_addr(sV) + s * KV_BYTES + kk * 16 * 128, KBOX_BYTES, 1024);
                if constexpr (HD == 64) Wgmma<T>::rs_n64(o, pa[kk], dv, 1);
                else Wgmma<T>::rs_n128(o, pa[kk], dv, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            reg_fence(o);
            bar_arrive(v_empty + s);
        }

        // epilogue: O / l -> global
        T *out = static_cast<T *>(p.out) + (long)b * p.o_bs + (long)h * HD;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float l = l_run[i];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = (l > 0.f) ? 1.f / l : 0.f;     // fully masked row -> zeros
            const int q = r0 + 8 * i;
            if (q < p.Tq) {
                T *op = out + (long)q * p.o_ts + 2 * tq;
#pragma unroll
                for (int jj = 0; jj < HD / 8; ++jj)
                    *reinterpret_cast<uint32_t *>(op + jj * 8) = pack2<T>(o[jj * 4 + 2 * i] * inv, o[jj * 4 + 2 * i + 1] * inv);
            }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------------
// (B, T, H, hd) tensor with element strides bs / ts (heads dense): dims innermost-first {hd, H, T, B}
// Encoding a tensor map costs a driver call on the host (three per launch); the decoder calls this op
// with the same few (pointer, shape, strides) combinations layer after layer, so the last encodings are kept per
// host thread.  A map depends only on its arguments (it holds no device state), so a hit is always valid.
struct MapKey {
    const void *ptr; int dtype, B, T, H, hd, box_rows; long bs, ts;
    bool operator==(const MapKey &o) const {
        return ptr == o.ptr && dtype == o.dtype && B == o.B && T == o.T && H == o.H && hd == o.hd && box_rows == o.box_rows &&
               bs == o.bs && ts == o.ts;
    }
};
constexpr int kMapCache = 32;
static thread_local MapKey g_map_keys[kMapCache];
static thread_local CUtensorMap g_map_vals[kMapCache];
static thread_local int g_map_n = 0, g_map_next = 0;

static int make_map_uncached(CUtensorMap *map, const void *ptr, int dtype, int B, int T, int H, int hd, long bs, long ts, int box_rows);

static int make_map(CUtensorMap *map, const void *ptr, int dtype, int B, int T, int H, int hd, long bs, long ts, int box_rows) {
    const MapKey key{ptr, dtype, B, T, H, hd, box_rows, bs, ts};
    for (int i = 0; i < g_map_n; ++i)
        if (g_map_keys[i] == key) { *map = g_map_vals[i]; return MMFS_OK; }
    const int rc = make_map_uncached(map, ptr, dtype, B, T, H, hd, bs, ts, box_rows);
    if (rc != MMFS_OK) return rc;
    g_map_keys[g_map_next] = key;
    g_map_vals[g_map_next] = *map;
    g_map_next = (g_map_next + 1) % kMapCache;
    if (g_map_n < kMapCache) ++g_map_n;
    return MMFS_OK;
}

static int make_map_uncached(CUtensorMap *map, const void *ptr, int dtype, int B, int T, int H, int hd, long bs, long ts, int box_rows) {
    EncodeTiledFn fn = tensor_map_encoder();
    if (!fn) { set_error("attn: cuTensorMapEncodeTiled is not available from this driver"); return MMFS_ECUDA; }
    const cuuint64_t dims[4] = {(cuuint64_t)hd, (cuuint64_t)H, (cuuint64_t)T, (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)hd * 2, (cuuint64_t)ts * 2, (cuuint64_t)bs * 2};
    const cuuint32_t box[4] = {64, 1, (cuuint32_t)box_rows, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(map, dtype == MMFS_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                    const_cast<void *>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("attn: cuTensorMapEncodeTiled failed (%d)", (int)r); return MMFS_ECUDA; }
    return MMFS_OK;
}

template <typename T, int HD>
static int launch_attn(const CUtensorMap &mq, const CUtensorMap &mk, const CUtensorMap &mv, const AttnParams &p, unsigned *sched,
                       cudaStream_t st) {
    const int dev = current_device();
    const int n_q = (p.Tq + kBM - 1) / kBM;
    const long n_work = (long)n_q * p.H * p.B;
    if (n_work >= (1L << 30)) { set_error("attn_forward: %ld work items", n_work); return MMFS_EUNSUPPORTED; }
    constexpr size_t smem = (size_t)(HD / 64) * (kBM * 128 + 4 * kBN * 128) + 14 * 8 + 2 * sizeof(int);
    auto kern = attn_fwd_kernel<T, HD>;
    static bool attr_set[kMaxDevices] = {};          // the attribute is per device
    if (dev < 0 || dev >= kMaxDevices || !attr_set[dev]) {
        MMFS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (dev >= 0 && dev < kMaxDevices) attr_set[dev] = true;
    }
    // more items than resident CTAs: persistent, otherwise one item per CTA
    const int resident = attn_ctas_per_sm<HD>() * num_sms();
    const bool persistent = sched != nullptr && n_work > resident;
    const int grid = persistent ? resident : (int)n_work;
    kern<<<grid, kAttnThreads, smem, st>>>(mq, mk, mv, p, persistent ? sched : nullptr, (int)n_work);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

}  // namespace mmfs

using namespace mmfs;

static int attn_forward_impl(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                             int B, int H, int Tq, int Tkv, int hd,
                             long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                             float scale, int causal, int past, int dtype, unsigned *sched, void *stream) {
    MMFS_CHECK_ARG(B >= 0 && H > 0 && Tq >= 0 && Tkv > 0, "attn_forward: bad shape");
    if (B == 0 || Tq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(q && k && v && out, "attn_forward: null pointer argument");
    if (!(hd == 64 || hd == 128) || !(dtype == MMFS_BF16 || dtype == MMFS_F16)) {
        set_error("attn_forward: tensor-core path needs hd in {64,128} and bf16/f16 (got hd=%d dtype=%d)", hd, dtype);
        return MMFS_EUNSUPPORTED;
    }
    if (((uintptr_t)q | (uintptr_t)k | (uintptr_t)v | (uintptr_t)out) % 16 != 0 ||
        (q_bs | q_ts | k_bs | k_ts | v_bs | v_ts | o_bs | o_ts) % 8 != 0 || B > 65535 || H > 65535) {
        set_error("attn_forward: pointers / strides must be 16-byte aligned; B, H <= 65535");
        return MMFS_EUNSUPPORTED;
    }
    CUtensorMap mq, mk, mv;
    int rc;
    if ((rc = make_map(&mq, q, dtype, B, Tq, H, hd, q_bs, q_ts, kBM)) != MMFS_OK) return rc;
    if ((rc = make_map(&mk, k, dtype, B, Tkv, H, hd, k_bs, k_ts, kBN)) != MMFS_OK) return rc;
    if ((rc = make_map(&mv, v, dtype, B, Tkv, H, hd, v_bs, v_ts, kBN)) != MMFS_OK) return rc;
    AttnParams p;
    p.out = out; p.key_mask = key_mask; p.B = B; p.H = H; p.Tq = Tq; p.Tkv = Tkv; p.causal = causal; p.past = past;
    p.o_bs = o_bs; p.o_ts = o_ts; p.scale_log2e = scale * 1.4426950408889634f;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == MMFS_BF16)
        return hd == 64 ? launch_attn<__nv_bfloat16, 64>(mq, mk, mv, p, sched, st) : launch_attn<__nv_bfloat16, 128>(mq, mk, mv, p, sched, st);
    return hd == 64 ? launch_attn<__half, 64>(mq, mk, mv, p, sched, st) : launch_attn<__half, 128>(mq, mk, mv, p, sched, st);
}

extern "C" int mmfs_attn_forward(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                                 int B, int H, int Tq, int Tkv, int hd,
                                 long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                                 float scale, int causal, int past, int dtype, void *stream) {
    return attn_forward_impl(q, k, v, out, key_mask, B, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, scale, causal,
                             past, dtype, nullptr, stream);
}

extern "C" int mmfs_attn_forward_persistent(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                                            int B, int H, int Tq, int Tkv, int hd,
                                            long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                                            float scale, int causal, int past, int dtype, unsigned *work_counter, void *stream) {
    MMFS_CHECK_ARG(work_counter != nullptr && (uintptr_t)work_counter % 4 == 0, "attn_forward_persistent: work_counter must be a zeroed device uint32");
    return attn_forward_impl(q, k, v, out, key_mask, B, H, Tq, Tkv, hd, q_bs, q_ts, k_bs, k_ts, v_bs, v_ts, o_bs, o_ts, scale, causal,
                             past, dtype, work_counter, stream);
}
