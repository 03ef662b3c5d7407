// linear_skinny_sm100.cu -- y[M, N] = prologue(x)[M, K] . W[N, K]^T (+ residual) for M <= 8 rows: the dense linears of
// a DECODE step (LlamaAttention q/k/v and o_proj, LlamaMLP gate/up and down, decoders/modeling_llama_mmfs.py:175-189,
// 217-280, with the RMSNorm in front of them, :53-70, and the SwiGLU between them, :188-189, folded in).
//
// At M = batch (4 at cfg 5) every weight byte is used once per token: the op is a stream of W out of HBM (27 GB per
// token for the 13 B decoder), not a tensor-core problem.  cuBLAS needs a separate RMSNorm / SwiGLU kernel in front
// of each pair, and its N = 5120 projections launch fewer CTAs than there are SMs.  This kernel:
//   * persistent, one CTA of 16 warps per SM.  The work is numbered in STEPS: step (block b, J) = the 32 weight rows of
//     block b x the 512 columns J*512 .. J*512+511, block-major; the steps are cut into equal contiguous ranges, one
//     per CTA ("stream-K" at 32 KB granularity): every SM streams the same number of bytes whatever N is;
//   * in a step warp w owns columns J*512 + w*32 .. +31: lane (g = lane / 4, t = lane % 4) owns, in each of the block's
//     four 8-row groups r, the 16 bytes W[32b + 8r + g][.. + 8t .. 8t+7] (per warp and group: 8 rows x 64 contiguous
//     bytes, every sector fully used) and feeds them, as they are, to two mma.sync.m16n8k16: the k index of a dot product
//     may be permuted freely as long as both operands use the same permutation, so the lane's four registers serve as
//     the B fragments of two MMAs whose A fragments are the matching 16 bytes of x row g.  No shuffles, no unpacking,
//     no shared-memory staging of W.  Rows 8-15 of the m16 tile are unused.  (The math is ~2 % of
//     the tensor pipe; the legacy mma path is used because the output tile is 8 x 8 and the operand arrives in
//     registers -- wgmma's 64-row warpgroup tile and shared-memory operands buy nothing for an HBM-bound stream.)
//   * memory-level parallelism: every lane keeps 3-4 steps x 4 cp.async (16-byte, L2-only) copies of ITS OWN future
//     operands in flight into private 16-byte slots of a shared-memory ring and reads them back itself (no barrier: a
//     thread sees its own completed copies after cp.async.wait_group) -- 96-128 KB in flight per SM, across block
//     boundaries and across the reduction barriers.  Plain loads into a register ring do not get there: a warp has six
//     scoreboards, so twelve individually tracked loads serialise; cp.async at 8-row blocks is issue-bound (33
//     instructions per 512 bytes) -- hence four row groups per step: one x fragment, one cursor update, one commit per
//     2 KB.  (The first version of this kernel staged W through a shared-memory ring filled by cp.async.bulk row pieces
//     and ldmatrix; every 1-D bulk copy pays a fixed cost on the SM's copy engine, which caps that design.)
//   * x is staged ONCE per CTA in shared memory by the consumer warps while the producer already streams W, through
//     the prologue: plain copy | RMSNorm(x) * weight (LlamaRMSNorm's rounding points: T(x * rstd), then * weight in T) |
//     SwiGLU of a [gate | up] row pair (T(silu(gate)) * up in T) -- the same arithmetic as the stand-alone kernels in
//     llama_ops_sm100.cu;
//   * a block that lies inside one CTA's range is finished there (sum over the 16 column-slice warps in fixed order,
//     + residual, one rounding to T); a block cut by a range boundary leaves fp32 partials in scratch and the LAST
//     CTA to arrive (a ticket per block) adds them in slot order: results do not depend on timing.  The tickets live
//     in caller-provided scratch that must be ZERO before the first call and is left zero by every call (no memset
//     node per linear in the decode graph); calls sharing a scratch buffer must be ordered (one stream).
// Roofline: HBM, N * K * sizeof(T) bytes per call.
#include "tc_common.cuh"

namespace mmfs {

constexpr int kSkRG = 4;                                  // 8-row groups per block: the x fragment of a step serves all four
constexpr int kSkRows = 8 * kSkRG;                        // weight rows per block
constexpr int kSkWarps = 16;
constexpr int kSkThreads = kSkWarps * 32;
constexpr int kSkStepCols = kSkWarps * 32;                // 512 columns per step
constexpr int kSkPlane = kSkThreads * 16;                 // one row group of a ring slot: 16 bytes per lane
constexpr int kSkSlotBytes = kSkRG * kSkPlane;            // 32 KB per step
constexpr int kSkMaxM = 8;
constexpr int kSkMaxSmem = 227 * 1024;
constexpr int kSkTile = kSkRows * 8;                      // fp32 outputs of a block (32 weight rows x 8 x rows)
constexpr int kSkXPad = 64;                               // x rows K * 2 + 64 bytes apart: two rows per LDS.128 phase, no conflict
constexpr int kSkMaxBlocks = 1 << 16;                     // tickets [kSkMaxBlocks] sit at the head of scratch for every N

struct SkinnyArgs {
    const void *x, *w, *residual, *norm_w;
    void *y;
    float *part;                                          // [n_blocks][2][256] fp32 partial tiles
    unsigned *tickets;                                    // [n_blocks], zero on entry; the last arriver re-zeroes its ticket
    int M, N, K, prologue;
    float eps;
    int spb, total, q, rm;                                // steps per block (K / 512), total steps, steps per CTA (q, +1 for c < rm)
    int xp;                                               // bytes between x rows in shared memory
    unsigned long long *dbg;                              // timing probe (tools/skinny_timeline.py): 4 globaltimer stamps per CTA, or null
};

template <typename T> struct SkMma;
template <> struct SkMma<__nv_bfloat16> {
    __device__ __forceinline__ static void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
};
template <> struct SkMma<__half> {
    __device__ __forceinline__ static void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
};

// 16-byte asynchronous copy global -> shared through L2 only (SASS LDGSTS.E.BYPASS.128): completion is tracked by
// commit groups, not by the warp's six scoreboards, so the depth of the prefetch is a free parameter.
__device__ __forceinline__ void sk_cp_async16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void sk_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void sk_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void finisher_sync() { asm volatile("bar.sync 2, 256;" ::: "memory"); }

template <typename T> __device__ __forceinline__ float sk_rnd(float x) { return to_op(from_op<T>(x)); }
__device__ __forceinline__ float sk_silu(float g) { return __fdividef(g, 1.f + __expf(-g)); }

__device__ __forceinline__ int sk_range_start(int c, int q, int rm) { return c * q + (c < rm ? c : rm); }
__device__ __forceinline__ int sk_cta_of(int f, int q, int rm) {          // the CTA whose range holds stage f
    const int cut = rm * (q + 1);
    return f < cut ? f / (q + 1) : rm + (f - cut) / q;
}

// The lane's 16 bytes of x are stored as words (0, 2, 1, 3): one LDS.128 = (X0, X2, X1, X3) is then, as it is, the A
// fragment of the first MMA (a0 = X0, a2 = X1; a1 / a3 feed the unused rows 8-15) against B = (W0, W1), and X2, X3 move
// into slots 0 / 2 of a second fragment against B = (W2, W3): two register moves per 512 bytes of W per warp.
__device__ __forceinline__ uint4 sk_perm(const uint4 &v) { return make_uint4(v.x, v.z, v.y, v.w); }

// ---- x -> shared memory through the prologue (all 512 threads) ----------------------------------------------------------
// All global loads of a pass are issued in batches of kSkXBatch independent vectors per thread BEFORE anything is done
// with them: walking the rows with load -> use -> load pays one dependent L2 round trip per vector (up to 32 of them
// for the 13824-wide SwiGLU operand).
constexpr int kSkXBatch = 8;

template <typename T, int NT, bool PERM>
__device__ __forceinline__ void sk_stage_x(const SkinnyArgs &a, uint8_t *xs, float *s_red, int tid) {
    constexpr int VEC = 8;
    auto put = [&](uint8_t *dst, const uint4 &v) { *reinterpret_cast<uint4 *>(dst) = PERM ? sk_perm(v) : v; };
    auto sync_all = [&]() {
        if (NT == kSkThreads) __syncthreads();
        else asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
    };
    const int nvec = a.K / VEC;                                          // 16-byte vectors per operand row
    const int total = a.M * nvec;
    const T *x = static_cast<const T *>(a.x);
    if (a.prologue == 0) {                                               // x is [M][K] contiguous: vector i sits at x + 8 i
        for (int i0 = tid; i0 < total; i0 += NT * kSkXBatch) {
            uint4 v[kSkXBatch];
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u)
                if (i0 + u * NT < total) v[u] = ldg_nc_v4(x + (size_t)(i0 + u * NT) * VEC);
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u) {
                const int i = i0 + u * NT;
                if (i < total) { const int m = i / nvec; put(xs + (size_t)m * a.xp + (i - m * nvec) * 16, v[u]); }
            }
        }
    } else if (a.prologue == 1) {                                        // RMSNorm
        float ss[kSkMaxM];
#pragma unroll
        for (int m = 0; m < kSkMaxM; ++m) ss[m] = 0.f;
        for (int i0 = tid; i0 < total; i0 += NT * kSkXBatch) {
            uint4 v[kSkXBatch];
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u)
                if (i0 + u * NT < total) v[u] = ldg_nc_v4(x + (size_t)(i0 + u * NT) * VEC);
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u) {
                const int i = i0 + u * NT;
                if (i < total) {
                    float f[VEC], sq = 0.f;
                    Vec16<T>::unpack(v[u], f);
#pragma unroll
                    for (int k = 0; k < VEC; ++k) sq = fmaf(f[k], f[k], sq);
                    const int m = i / nvec;
#pragma unroll
                    for (int mm = 0; mm < kSkMaxM; ++mm) ss[mm] += (m == mm) ? sq : 0.f;
                }
            }
        }
#pragma unroll
        for (int m = 0; m < kSkMaxM; ++m) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) ss[m] += __shfl_xor_sync(0xffffffffu, ss[m], o);
            if ((tid & 31) == 0) s_red[(tid >> 5) * kSkMaxM + m] = ss[m];
        }
        sync_all();
        float rstd[kSkMaxM];
#pragma unroll
        for (int m = 0; m < kSkMaxM; ++m) {
            float tot = 0.f;
            for (int w = 0; w < NT / 32; ++w) tot += s_red[w * kSkMaxM + m];
            rstd[m] = rsqrtf(tot / (float)a.K + a.eps);
        }
        const T *nw = static_cast<const T *>(a.norm_w);
        for (int i0 = tid; i0 < total; i0 += NT * kSkXBatch) {          // second pass: x again (L2) + the norm weights
            uint4 v[kSkXBatch], wv[kSkXBatch];
            int mi[kSkXBatch];
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u) {
                const int i = i0 + u * NT;
                if (i < total) {
                    mi[u] = i / nvec;
                    v[u] = ldg_nc_v4(x + (size_t)i * VEC);
                    wv[u] = ldg_nc_v4(nw + (size_t)(i - mi[u] * nvec) * VEC);
                }
            }
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u) {
                const int i = i0 + u * NT;
                if (i < total) {
                    float r = 0.f;
#pragma unroll
                    for (int mm = 0; mm < kSkMaxM; ++mm) r = (mi[u] == mm) ? rstd[mm] : r;
                    float f[VEC], g[VEC], o[VEC];
                    Vec16<T>::unpack(v[u], f);
                    Vec16<T>::unpack(wv[u], g);
#pragma unroll
                    for (int k = 0; k < VEC; ++k) o[k] = g[k] * sk_rnd<T>(f[k] * r);
                    put(xs + (size_t)mi[u] * a.xp + (i - mi[u] * nvec) * 16, Vec16<T>::pack(o));
                }
            }
        }
    } else {                                                             // SwiGLU of [gate | up] rows of 2K columns
        for (int i0 = tid; i0 < total; i0 += NT * kSkXBatch) {
            uint4 gv[kSkXBatch], uv[kSkXBatch];
            int mi[kSkXBatch];
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u) {
                const int i = i0 + u * NT;
                if (i < total) {
                    mi[u] = i / nvec;
                    const T *row = x + (size_t)mi[u] * 2 * a.K + (size_t)(i - mi[u] * nvec) * VEC;
                    gv[u] = ldg_nc_v4(row);
                    uv[u] = ldg_nc_v4(row + a.K);
                }
            }
#pragma unroll
            for (int u = 0; u < kSkXBatch; ++u) {
                const int i = i0 + u * NT;
                if (i < total) {
                    float g[VEC], up[VEC], o[VEC];
                    Vec16<T>::unpack(gv[u], g);
                    Vec16<T>::unpack(uv[u], up);
#pragma unroll
                    for (int k = 0; k < VEC; ++k) o[k] = sk_rnd<T>(sk_silu(g[k])) * up[k];
                    put(xs + (size_t)mi[u] * a.xp + (i - mi[u] * nvec) * 16, Vec16<T>::pack(o));
                }
            }
        }
    }
}

// One block's share is complete in this CTA: reduce the 16 column slices, then finish the block or leave a partial.
template <typename T>
__device__ __noinline__ void sk_block_end(const SkinnyArgs &a, float *red, int *s_flag, const float (&v)[kSkRG][2], int blk) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    __syncthreads();                                                          // the previous block's tile has been read
#pragma unroll
    for (int r = 0; r < kSkRG; ++r) {                                         // tile[weight row][x row]
        red[warp * kSkTile + (r * 8 + 2 * t) * 8 + g] = v[r][0];
        red[warp * kSkTile + (r * 8 + 2 * t + 1) * 8 + g] = v[r][1];
    }
    __syncthreads();
    if (tid >= kSkTile) return;
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < kSkWarps; ++w) acc += red[w * kSkTile + tid];
    const int row = tid >> 3, m = tid & 7, c = blockIdx.x;
    const int first = blk * a.spb, last = first + a.spb - 1;                  // the block's step range
    const int c_first = sk_cta_of(first, a.q, a.rm), c_last = sk_cta_of(last, a.q, a.rm);
    bool finish = true;
    if (c_first != c_last) {                                                  // cut by a range boundary: partials + ticket
        const int n_part = c_last - c_first + 1;                              // == 2 (host: every range holds >= spb steps)
        float *pp = a.part + ((size_t)blk * 2) * kSkTile;
        pp[(c - c_first) * kSkTile + tid] = acc;
        __threadfence();
        finisher_sync();
        if (tid == 0) *s_flag = atomicAdd(a.tickets + blk, 1u) == (unsigned)(n_part - 1);
        finisher_sync();
        finish = *s_flag != 0;
        if (finish) {
            __threadfence();
            acc = 0.f;
            for (int p = 0; p < n_part; ++p) acc += __ldcg(pp + p * kSkTile + tid);   // slot order: timing-independent
            if (tid == 0) a.tickets[blk] = 0u;                                // zero on entry, zero on exit
        }
        finisher_sync();                                                      // s_flag may be rewritten by the next block
    }
    if (finish && m < a.M) {
        const size_t o = (size_t)m * a.N + (size_t)blk * kSkRows + row;
        if (a.residual != nullptr) acc += to_op(static_cast<const T *>(a.residual)[o]);
        static_cast<T *>(a.y)[o] = from_op<T>(acc);
    }
}

template <typename T, int DEPTH>
__global__ void __launch_bounds__(kSkThreads, 1) linear_skinny_kernel(const __grid_constant__ SkinnyArgs a) {
    extern __shared__ __align__(128) uint8_t s_dyn[];
    // layout: W ring [DEPTH][4 row groups][512 lanes][16 B] | x rows | reduction tile [16][256] fp32 | rmsnorm scratch | flag
    uint8_t *ring = s_dyn;
    uint8_t *xs = ring + DEPTH * kSkSlotBytes;
    float *red = reinterpret_cast<float *>(xs + (size_t)a.M * a.xp);
    float *s_red = red + kSkWarps * kSkTile;
    int *s_flag = reinterpret_cast<int *>(s_red + kSkWarps * kSkMaxM);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int c = blockIdx.x;
    const int f0 = sk_range_start(c, a.q, a.rm), n_my = sk_range_start(c + 1, a.q, a.rm) - f0;

    // ---- load cursor: the lane's 16 bytes of step (blk, J), row group r: W[32 blk + 8 r + g][J*512 + warp*32 + 8t ..]
    const size_t row_bytes = (size_t)a.K * 2, group_bytes = 8 * row_bytes;
    int l_j = f0 % a.spb, l_left = n_my;                                      // steps still to request
    const uint8_t *lp = static_cast<const uint8_t *>(a.w) + ((size_t)(f0 / a.spb) * kSkRows + g) * row_bytes +
                        ((size_t)l_j * kSkStepCols + warp * 32 + t * 8) * 2;
    const uint32_t ring_addr = (uint32_t)__cvta_generic_to_shared(ring) + tid * 16;
    uint32_t l_slot = ring_addr;
    auto request = [&]() {                                                    // one commit group per step, empty past the end
        if (l_left > 0) {
#pragma unroll
            for (int r = 0; r < kSkRG; ++r) sk_cp_async16(l_slot + r * kSkPlane, lp + r * group_bytes);
            --l_left;
            lp += kSkStepCols * 2;
            if (++l_j == a.spb) { l_j = 0; lp += (kSkRows - 1) * row_bytes; }   // same row of the next block
        }
        sk_commit();
        l_slot += kSkSlotBytes;
        if (l_slot == ring_addr + DEPTH * kSkSlotBytes) l_slot = ring_addr;
    };
#pragma unroll
    for (int i = 0; i < DEPTH; ++i) request();

    sk_stage_x<T, kSkThreads, true>(a, xs, s_red, tid);   // overlaps the first DEPTH steps of copies
    __syncthreads();

    // ---- compute cursor ------------------------------------------------------------------------------------------------
    // Operand roles: the x rows are the M side (row g of the tile = x row g; rows >= M repeat row 0 and rows 8-15 are
    // whatever the unused registers hold -- an output row depends on its own operand row only, and those outputs are
    // never stored), the 8 weight rows of a group are the N side: the lane's 16 bytes (W0, W1, W2, W3) are the B
    // fragments of two MMAs as they are.
    int blk = f0 / a.spb, j = f0 - blk * a.spb;
    const uint8_t *xq = xs + (size_t)(g < a.M ? g : 0) * a.xp + (warp * 32 + t * 8) * 2 + (size_t)j * (kSkStepCols * 2);
    const uint8_t *wq = ring + tid * 16, *wq_end = wq + DEPTH * kSkSlotBytes;
    const uint8_t *wc = wq;
    float d[kSkRG][2][4];                                                     // [group][chain]: d[.][.][0..1] = x row g x weight rows 2t, 2t+1
#pragma unroll
    for (int r = 0; r < kSkRG; ++r)
#pragma unroll
        for (int k = 0; k < 4; ++k) d[r][0][k] = d[r][1][k] = 0.f;
    uint32_t a1[4] = {0u, 0u, 0u, 0u};                                        // slots 1, 3 stay as they are
    int it = 0;
    while (it < n_my) {
        const int seg = min(n_my - it, a.spb - j);                            // steps of this block in my range
        for (int s = 0; s < seg; ++s) {
            sk_wait_group<DEPTH - 1>();                                       // the copies of this step have landed
            const uint4 xv = *reinterpret_cast<const uint4 *>(xq);            // (X0, X2, X1, X3)
            const uint32_t a0[4] = {xv.x, xv.y, xv.z, xv.w};
            a1[0] = xv.y;
            a1[2] = xv.w;
#pragma unroll
            for (int r = 0; r < kSkRG; ++r) {
                const uint4 wv = *reinterpret_cast<const uint4 *>(wc + r * kSkPlane);
                SkMma<T>::mma(d[r][0], a0, wv.x, wv.y);
                SkMma<T>::mma(d[r][1], a1, wv.z, wv.w);
            }
            request();                                                        // refills the slot just read (issued after its readers)
            xq += kSkStepCols * 2;
            wc += kSkSlotBytes;
            if (wc == wq_end) wc = wq;
        }
        it += seg;
        j += seg;
        float v[kSkRG][2];
#pragma unroll
        for (int r = 0; r < kSkRG; ++r) {
            v[r][0] = d[r][0][0] + d[r][1][0];
            v[r][1] = d[r][0][1] + d[r][1][1];
#pragma unroll
            for (int k = 0; k < 4; ++k) d[r][0][k] = d[r][1][k] = 0.f;
        }
        sk_block_end<T>(a, red, s_flag, v, blk);
        if (j == a.spb) { j = 0; ++blk; xq -= (size_t)a.spb * (kSkStepCols * 2); }
    }
}

// ------------------------------------------------------------------------------------------------------------
// The same op fed by tensor-map TMA (what the library's own skinny kernels do): one cp.async.bulk.tensor.2d per
// (128 rows x 64 columns) = 16 KB box of W, SWIZZLE_128B, into a ring of up to 11 stages (176 KB in flight per SM, no
// per-lane copy instructions, no L1 involvement).  Stream-K over (128-row block, 64-column step) units; warp w of the 8
// consumer warps owns rows 16w .. 16w+15 of the block for ALL its K steps (ldmatrix.x4 from the swizzled stage as the A
// fragment, x from shared memory as the B fragment, fp32 accumulators in registers), so a block needs no cross-warp
// reduction.  A block cut by range boundaries leaves per-CTA partial tiles (at most two per CTA: its first and its last
// block) and the last CTA to arrive adds them in CTA order.
constexpr int kTmRows = 128, kTmCols = 64, kTmStage = kTmRows * kTmCols * 2, kTmWarps = 8, kTmThreads = (kTmWarps + 1) * 32;
constexpr int kTmTile = kTmRows * 8;                      // fp32 outputs of a block
constexpr int kTmMaxStages = 12, kTmMaxCtas = 256;

static __device__ unsigned long long g_sk_dbg[4 * 256];
__device__ __forceinline__ unsigned long long sk_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ void tm_consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void tm_ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

template <typename T>
__global__ void __launch_bounds__(kTmThreads, 1)
linear_skinny_tma_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ SkinnyArgs a, int n_stages) {
    extern __shared__ __align__(1024) uint8_t s_tm[];
    // layout: W ring [n_stages][16 KB] (1024-byte aligned for the swizzle) | x rows | rmsnorm scratch | barriers | flag
    uint8_t *ring = s_tm;
    uint8_t *xs = ring + (size_t)n_stages * kTmStage;
    float *s_red = reinterpret_cast<float *>(xs + (size_t)a.M * a.xp);
    uint64_t *full = reinterpret_cast<uint64_t *>(s_red + kTmWarps * kSkMaxM);
    uint64_t *empty = full + kTmMaxStages;
    int *s_flag = reinterpret_cast<int *>(empty + kTmMaxStages);
    if ((s_addr(s_tm) & 1023u) != 0u) { asm volatile("trap;"); }

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int c = blockIdx.x;
    const int f0 = sk_range_start(c, a.q, a.rm), n_my = sk_range_start(c + 1, a.q, a.rm) - f0;
    if (a.dbg != nullptr && tid == 0) a.dbg[c * 4 + 0] = sk_now();

    if (tid == 0) {
        for (int s = 0; s < n_stages; ++s) { bar_init(full + s, 1); bar_init(empty + s, kTmWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kTmWarps) {
        // ======================================= producer =======================================
        if (lane == 0) {
            int s = 0, round = 0, blk = f0 / a.spb, kc = f0 - blk * a.spb;
            for (int it = 0; it < n_my; ++it) {
                if (round > 0) bar_wait(empty + s, (round - 1) & 1);
                bar_expect_tx(full + s, kTmStage);
                tma_load_2d(ring + (size_t)s * kTmStage, &map_w, full + s, kc * kTmCols, blk * kTmRows);
                if (++s == n_stages) { s = 0; ++round; }
                if (++kc == a.spb) { kc = 0; ++blk; }
            }
        }
        return;
    }

    // ========================================= consumers =========================================
    sk_stage_x<T, 256, false>(a, xs, s_red, tid);          // while the producer already streams W
    tm_consumer_sync();

    const int g = lane >> 2, t = lane & 3;
    // ldmatrix.x4 lane -> (row, k half) of the 16 x 16 tile: lanes 0-7 rows 0-7 / k 0-7, 8-15 rows 8-15 / k 0-7,
    // 16-23 rows 0-7 / k 8-15, 24-31 rows 8-15 / k 8-15; a 16-byte chunk c of row r sits at chunk c ^ (r & 7) (SWIZZLE_128B)
    const int lr = (lane & 7) + ((lane >> 3) & 1) * 8, lhi = lane >> 4;
    const uint32_t row_off = (uint32_t)((warp * 16 + lr) * 128);
    const uint32_t ring_addr = s_addr(ring);
    const uint8_t *xb = xs + (size_t)(g < a.M ? g : 0) * a.xp + 2 * t * 2;      // x[g][k + 2t], x[g][k + 2t + 8]
    T *y = static_cast<T *>(a.y);
    const T *res = static_cast<const T *>(a.residual);

    float d[4] = {0.f, 0.f, 0.f, 0.f};
    int s = 0, round = 0, blk = f0 / a.spb, kc = f0 - blk * a.spb;
    const int my_first_blk = blk;
    for (int it = 0; it < n_my; ++it) {
        bar_wait(full + s, round & 1);
        if (a.dbg != nullptr && tid == 0 && (it == 0 || it == n_my - 1)) a.dbg[c * 4 + (it == 0 ? 1 : 2)] = sk_now();
        const uint32_t st = ring_addr + (uint32_t)s * kTmStage + row_off;
        const uint8_t *xk = xb + (size_t)kc * (kTmCols * 2);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            uint32_t af[4];
            tm_ldmatrix_x4(af, st + (uint32_t)(((kk * 2 + lhi) ^ (lr & 7)) << 4));
            const uint32_t b0 = *reinterpret_cast<const uint32_t *>(xk + kk * 32);
            const uint32_t b1 = *reinterpret_cast<const uint32_t *>(xk + kk * 32 + 16);
            SkMma<T>::mma(d, af, b0, b1);
        }
        __syncwarp();
        if (lane == 0) bar_arrive(empty + s);
        if (++s == n_stages) { s = 0; ++round; }

        const bool block_ends = (kc == a.spb - 1) || (it == n_my - 1);
        const int this_blk = blk;
        if (++kc == a.spb) { kc = 0; ++blk; }
        if (!block_ends) continue;
        // ---- this CTA's share of block `this_blk`: the lane holds (row g / g + 8 of the warp's 16, x rows 2t, 2t + 1) ------
        const int first = this_blk * a.spb, last = first + a.spb - 1;
        const int c_first = sk_cta_of(first, a.q, a.rm), c_last = sk_cta_of(last, a.q, a.rm);
        const int r0 = warp * 16 + g;
        float v[4] = {d[0], d[1], d[2], d[3]};
        d[0] = d[1] = d[2] = d[3] = 0.f;
        bool finish = true;
        if (c_first != c_last) {                                              // cut: per-CTA partial tiles + a ticket
            float *mine = a.part + ((size_t)c * 2 + (this_blk == my_first_blk ? 0 : 1)) * kTmTile;
            mine[r0 * 8 + 2 * t] = v[0];
            mine[r0 * 8 + 2 * t + 1] = v[1];
            mine[(r0 + 8) * 8 + 2 * t] = v[2];
            mine[(r0 + 8) * 8 + 2 * t + 1] = v[3];
            __threadfence();
            tm_consumer_sync();
            if (tid == 0) *s_flag = atomicAdd(a.tickets + this_blk, 1u) == (unsigned)(c_last - c_first);
            tm_consumer_sync();
            finish = *s_flag != 0;
            if (finish) {
                __threadfence();
                v[0] = v[1] = v[2] = v[3] = 0.f;
                for (int cc = c_first; cc <= c_last; ++cc) {                  // CTA order: timing-independent
                    const int cc_first_blk = sk_range_start(cc, a.q, a.rm) / a.spb;
                    const float *pp = a.part + ((size_t)cc * 2 + (this_blk == cc_first_blk ? 0 : 1)) * kTmTile;
                    v[0] += __ldcg(pp + r0 * 8 + 2 * t);
                    v[1] += __ldcg(pp + r0 * 8 + 2 * t + 1);
                    v[2] += __ldcg(pp + (r0 + 8) * 8 + 2 * t);
                    v[3] += __ldcg(pp + (r0 + 8) * 8 + 2 * t + 1);
                }
                if (tid == 0) a.tickets[this_blk] = 0u;                       // zero on entry, zero on exit
            }
            tm_consumer_sync();                                               // s_flag may be rewritten by the next block
        }
        if (finish) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = 2 * t + (e & 1), row = r0 + (e >> 1) * 8;
                if (m < a.M) {
                    const size_t o = (size_t)m * a.N + (size_t)this_blk * kTmRows + row;
                    float out = v[e];
                    if (res != nullptr) out += to_op(res[o]);
                    y[o] = from_op<T>(out);
                }
            }
        }
    }
    if (a.dbg != nullptr && tid == 0) a.dbg[c * 4 + 3] = sk_now();
}

static inline size_t skinny_tma_smem(int stages, int M, int K) {
    return (size_t)stages * kTmStage + (size_t)M * (K * 2 + 16) + kTmWarps * kSkMaxM * sizeof(float) + 2 * kTmMaxStages * sizeof(uint64_t) + 16;
}

struct SkMapKey { const void *ptr; int dtype, N, K; };
static thread_local SkMapKey g_sk_keys[16];
static thread_local CUtensorMap g_sk_maps[16];
static thread_local int g_sk_n = 0, g_sk_next = 0;

static int skinny_weight_map(CUtensorMap *map, const void *w, int dtype, int N, int K) {
    for (int i = 0; i < g_sk_n; ++i)
        if (g_sk_keys[i].ptr == w && g_sk_keys[i].dtype == dtype && g_sk_keys[i].N == N && g_sk_keys[i].K == K) { *map = g_sk_maps[i]; return MMFS_OK; }
    EncodeTiledFn fn = tensor_map_encoder();
    if (!fn) { set_error("linear_skinny: cuTensorMapEncodeTiled is not available from this driver"); return MMFS_ECUDA; }
    const cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)N};
    const cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    const cuuint32_t box[2] = {kTmCols, kTmRows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, dtype == MMFS_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                    const_cast<void *>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("linear_skinny: cuTensorMapEncodeTiled failed (%d)", (int)r); return MMFS_ECUDA; }
    g_sk_keys[g_sk_next] = SkMapKey{w, dtype, N, K};
    g_sk_maps[g_sk_next] = *map;
    g_sk_next = (g_sk_next + 1) % 16;
    if (g_sk_n < 16) ++g_sk_n;
    return MMFS_OK;
}

template <typename T>
static int launch_skinny_tma(SkinnyArgs a, int dtype, cudaStream_t st) {
    CUtensorMap map;
    int rc = skinny_weight_map(&map, a.w, dtype, a.N, a.K);
    if (rc != MMFS_OK) return rc;
    const int n_blocks = a.N / kTmRows;
    a.xp = a.K * 2 + 16;
    a.spb = a.K / kTmCols;
    a.total = n_blocks * a.spb;
    int grid = num_sms();
    if (grid > kTmMaxCtas) grid = kTmMaxCtas;
    if (grid > a.total) grid = a.total;
    a.q = a.total / grid;
    a.rm = a.total % grid;
    int stages = kTmMaxStages;
    while (stages > 3 && skinny_tma_smem(stages, a.M, a.K) + 1024 > (size_t)kSkMaxSmem) --stages;
    if (skinny_tma_smem(stages, a.M, a.K) + 1024 > (size_t)kSkMaxSmem) {
        set_error("linear_skinny: M = %d rows of K = %d do not fit shared memory next to a 3-stage weight ring", a.M, a.K);
        return MMFS_EUNSUPPORTED;
    }
    if (stages > a.q + 1) stages = a.q + 1;
    auto kern = linear_skinny_tma_kernel<T>;
    static bool attr_set[kMaxDevices] = {};
    const int dev = current_device();
    if (dev < 0 || dev >= kMaxDevices || !attr_set[dev]) {
        MMFS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkMaxSmem));
        if (dev >= 0 && dev < kMaxDevices) attr_set[dev] = true;
    }
    kern<<<grid, kTmThreads, skinny_tma_smem(stages, a.M, a.K), st>>>(map, a, stages);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

static bool g_sk_probe = false;
static int g_sk_mode = 0;   // 0 / 2: tensor-map TMA kernel when the shape allows; 1: per-lane cp.async kernel

static inline size_t skinny_smem(int depth, int M, int K) {
    return (size_t)depth * kSkSlotBytes + (size_t)M * (K * 2 + kSkXPad) + (kSkWarps * kSkTile + kSkWarps * kSkMaxM) * sizeof(float) + 16;
}

template <typename T, int DEPTH>
static int launch_skinny_depth(const SkinnyArgs &a, int grid, cudaStream_t st) {
    auto kern = linear_skinny_kernel<T, DEPTH>;
    static bool attr_set[kMaxDevices] = {};
    const int dev = current_device();
    if (dev < 0 || dev >= kMaxDevices || !attr_set[dev]) {
        MMFS_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSkMaxSmem));
        if (dev >= 0 && dev < kMaxDevices) attr_set[dev] = true;
    }
    kern<<<grid, kSkThreads, skinny_smem(DEPTH, a.M, a.K), st>>>(a);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int launch_skinny(SkinnyArgs a, cudaStream_t st) {
    const int n_blocks = a.N / kSkRows;
    a.xp = a.K * 2 + kSkXPad;
    a.spb = a.K / kSkStepCols;
    a.total = n_blocks * a.spb;
    // at most one CTA per block: every range then holds >= spb steps, so a block is cut by at most ONE range boundary
    // (two partial tiles per block in scratch)
    int grid = num_sms();
    if (grid > n_blocks) grid = n_blocks;
    a.q = a.total / grid;
    a.rm = a.total % grid;
    if (skinny_smem(4, a.M, a.K) <= (size_t)kSkMaxSmem) return launch_skinny_depth<T, 4>(a, grid, st);
    if (skinny_smem(3, a.M, a.K) <= (size_t)kSkMaxSmem) return launch_skinny_depth<T, 3>(a, grid, st);
    if (skinny_smem(2, a.M, a.K) <= (size_t)kSkMaxSmem) return launch_skinny_depth<T, 2>(a, grid, st);
    set_error("linear_skinny: M = %d rows of K = %d do not fit shared memory next to the copy ring", a.M, a.K);
    return MMFS_EUNSUPPORTED;
}

}  // namespace mmfs

using namespace mmfs;

extern "C" long mmfs_linear_skinny_scratch_floats(int N) {
    const long n_blocks = (N + kSkRows - 1) / kSkRows;
    // tickets at a FIXED place (the head) whatever N is -- a buffer shared between calls of different N must never see
    // one call's partial tiles where another call expects zero tickets -- then two partial tiles per block
    const long lanes = kSkMaxBlocks + n_blocks * 2 * kSkTile;                // per-lane cp.async kernel: two tiles per 32-row block
    const long boxes = kSkMaxBlocks + (long)kTmMaxCtas * 2 * kTmTile;        // tensor-map kernel: two tiles per CTA
    return lanes > boxes ? lanes : boxes;
}

extern "C" int mmfs_linear_skinny_set_tuning(int mode) {
    MMFS_CHECK_ARG((mode & 3) <= 2 && mode >= 0 && mode < 8, "linear_skinny_set_tuning: 0 default, 1 per-lane cp.async kernel, 2 tensor-map TMA kernel, +4 timing probe");
    g_sk_mode = mode & 3;
    g_sk_probe = (mode & 4) != 0;
    return MMFS_OK;
}

/* timing probe (mode + 4, tensor-map kernel): per CTA {entry, first stage landed, last stage landed, exit} in globaltimer ns */
extern "C" int mmfs_linear_skinny_probe(unsigned long long *host_out, int n_ctas) {
    MMFS_CHECK_ARG(host_out != nullptr && n_ctas > 0 && n_ctas <= 256, "linear_skinny_probe: bad arguments");
    MMFS_CUDA(cudaDeviceSynchronize());
    MMFS_CUDA(cudaMemcpyFromSymbol(host_out, g_sk_dbg, sizeof(unsigned long long) * 4 * n_ctas));
    return MMFS_OK;
}

extern "C" int mmfs_linear_skinny(const void *x, const void *w, void *y, const void *residual, const void *norm_weight,
                                  float *scratch, int M, int N, int K, int prologue, float eps, int dtype, void *stream) {
    MMFS_CHECK_ARG(M >= 0 && N > 0 && K > 0, "linear_skinny: bad shape");
    if (M == 0) return MMFS_OK;
    MMFS_CHECK_ARG(x && w && y && scratch, "linear_skinny: null pointer argument");
    MMFS_CHECK_ARG(prologue >= 0 && prologue <= 2 && (prologue != 1 || norm_weight != nullptr),
                   "linear_skinny: prologue 0 (none) / 1 (rmsnorm, needs norm_weight) / 2 (swiglu)");
    if (M > kSkMaxM || (dtype != MMFS_F16 && dtype != MMFS_BF16) || N % kSkRows != 0 || N / kSkRows > kSkMaxBlocks || K % kSkStepCols != 0 ||
        ((uintptr_t)x | (uintptr_t)w | (uintptr_t)y | (uintptr_t)scratch | (uintptr_t)norm_weight) % 16 != 0) {
        set_error("linear_skinny: needs M <= %d, f16 / bf16, N %% %d == 0, K %% %d == 0, 16-byte aligned pointers", kSkMaxM, kSkRows, kSkStepCols);
        return MMFS_EUNSUPPORTED;
    }
    SkinnyArgs a{};
    a.x = x; a.w = w; a.y = y; a.residual = residual; a.norm_w = norm_weight;
    a.tickets = reinterpret_cast<unsigned *>(scratch);
    a.part = scratch + kSkMaxBlocks;
    a.M = M; a.N = N; a.K = K; a.prologue = prologue; a.eps = eps;
    a.dbg = nullptr;
    if (g_sk_probe) MMFS_CUDA(cudaGetSymbolAddress((void **)&a.dbg, g_sk_dbg));
    cudaStream_t st = (cudaStream_t)stream;
    if (g_sk_mode != 1 && N % kTmRows == 0 && K % kTmCols == 0 && N / kTmRows <= kSkMaxBlocks &&
        skinny_tma_smem(3, M, K) + 1024 <= (size_t)kSkMaxSmem)
        return dtype == MMFS_F16 ? launch_skinny_tma<__half>(a, dtype, st) : launch_skinny_tma<__nv_bfloat16>(a, dtype, st);
    return dtype == MMFS_F16 ? launch_skinny<__half>(a, st) : launch_skinny<__nv_bfloat16>(a, st);
}
