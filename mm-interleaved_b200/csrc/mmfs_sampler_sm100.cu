// mmfs_sampler_sm100.cu -- fused MMFS sampler for sm_90a.
//
// Replaces the un-fused middle of the reference's MMFS.forward
//   ops/modules/mmfs.py:178-273  (relpos embedding add, offset / weight views and rearranges,
//                                 image mask add, null-slot softmax, sampling-location arithmetic,
//                                 MSDeformAttnFunction.apply)
// with ONE kernel that reads the two small GEMM outputs directly and never materialises the
// (N,Lq,M,L,P,2) location tensor or the (N,Lq,M,L,P) weight tensor:
//
//   qproj   (N, Lq, C)   [sampling_offsets | attention_weights](dynamic_offset_mask(query)) + bias,
//                        C = M*P*2 + M*n_lvl*(P+1), computed ONCE per token (the reference repeats
//                        the query n_img times, mmfs.py:174-175)
//   rtable  (R, C)       the same two linears applied to query_relpos.weight (no bias): by linearity
//                        Linear(q1 + e_r) = Linear(q1) + W e_r, so the per-image conditioning
//                        (mmfs.py:178-179) becomes a table lookup
//   relpos  (N, n_img, Lq_r) uint8 relative image index, 0 = image not visible (mmfs.py:154-163)
//
// Per output row (b, q, m) a warp: finds the visible images, forms their logits, does the
// null-slot softmax (every level -- visible or not -- owns a null slot with logit -log(L),
// mmfs.py:225; masked images get -1e4 and vanish exactly), derives the sampling locations
//   loc = ref + (off * scale_ratio[l]) / (W_l, H_l)                       (mmfs.py:194-198, 243-250)
// with the SAME intermediate roundings to the storage type the reference's tensor pipeline
// performs, and feeds the shared gather machinery (sampler_common.cuh).  Masked images cost
// nothing: no loads, no index math, no fetches.
//
// The EMIT instantiation writes the location / weight tensors instead of gathering: it is the
// parity instrumentation (tests compare them with the reference's intermediates and push them
// through the index-stream check) and the route for head sizes without a fast gather path.
#include "sampler_common.cuh"

namespace mmfs {

// Shared memory of one CTA: int4 lvl[L] | float scale[n_lvl] (padded to 16 B) | per warp:
//   Tap taps[kTapsPerWarp] | float xs[n_img*n_lvl*P] (logits of the row) | int vis[32]
template <typename T, int D, bool EMIT>
__global__ void __launch_bounds__(32 * kWarpsPerCta, 3) mmfs_sampler_kernel(const SamplerArgs a) {
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int LPR = D / VEC;
    const int M = a.M, n_img = a.n_img, n_lvl = a.n_lvl, Lq = a.Lq, P = a.P;
    const int L = n_img * n_lvl;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    extern __shared__ int4 s_dyn[];
    int4 *s_lvl = s_dyn;
    float *s_scale = reinterpret_cast<float *>(s_dyn + L);
    const int scale_slots = (n_lvl + 3) / 4;  // int4 units
    const int xs_elems = n_img * ((n_lvl * P + 31) / 32) * 32;
    const int q_elems = P * 2 + n_lvl * (P + 1);              // this head's slice of a qproj row: offsets | logits
    const int qs_elems = ((q_elems + 3) / 4) * 4;
    const int per_warp_bytes = kTapsPerWarp * (int)sizeof(Tap) + (xs_elems + qs_elems) * 4 + 256;   // + s_vis[64]
    char *wbase = reinterpret_cast<char *>(s_dyn + L + scale_slots) + warp * per_warp_bytes;
    Tap *taps = reinterpret_cast<Tap *>(wbase);
    float *xs = reinterpret_cast<float *>(wbase + kTapsPerWarp * sizeof(Tap));
    float *qs = xs + xs_elems;                                // [P*2 offsets | n_lvl*(P+1) logits] of the current row, fp32
    int *s_vis = reinterpret_cast<int *>(wbase + kTapsPerWarp * sizeof(Tap) + (xs_elems + qs_elems) * 4);

    for (int l = threadIdx.x; l < L; l += blockDim.x)
        s_lvl[l] = make_int4((int)a.shapes[2 * l], (int)a.shapes[2 * l + 1], (int)a.starts[l], 0);
    for (int l = threadIdx.x; l < n_lvl; l += blockDim.x) s_scale[l] = a.scale_ratios[l];
    __syncthreads();

    const T *value = static_cast<const T *>(a.value);
    const T *qproj = static_cast<const T *>(a.qproj);
    const T *rtable = static_cast<const T *>(a.rtable);
    const int C = M * P * 2 + M * n_lvl * (P + 1);
    const long long row_bytes = (long long)M * D * (int)sizeof(T);
    const bool strict = a.flags & MMFS_MSDA_STRICT;
    const int slot = lane / LPR;
    const float nullv = round_to<T>(a.null_logit);
    const int per_img = n_lvl * P;                            // sampling items of one image
    const int img_passes = (per_img + 31) / 32;               // 1 for every shipped configuration (24 or 32 items)
    const int l_lane = lane / P, p_lane = lane - l_lane * P;  // (level, point) of this lane's item in pass 0

    RowWalk walk;
    walk.itiles = (int)a.ntiles; walk.igrid = (int)gridDim.x; walk.qtiles = a.qtiles; walk.M = M; walk.Lq = Lq;
    walk.rows_per_warp = a.rows_per_warp; walk.warp = warp;

    // Everything a row needs from HBM -- its relpos bytes and its head's slice of the qproj row -- is
    // fetched one row AHEAD into registers, so a row's critical path only sees shared memory, the
    // L1-resident relpos table and the gathers.
    constexpr int kQPre = 4;                                  // supports slices of up to 128 elements
    if (q_elems > 32 * kQPre) { asm volatile("trap;"); }
    const int q_loads = (q_elems + 31) / 32;
    float pre_q[kQPre];
    int pre_r = 0;
    auto prefetch = [&](const RowCursor &c) {
        const T *qp = qproj + ((size_t)c.b * Lq + c.q) * C;
        const int ob = c.m * P * 2, ab = M * P * 2 + c.m * n_lvl * (P + 1);
#pragma unroll
        for (int t = 0; t < kQPre; ++t) {
            const int e = lane + 32 * t;
            pre_q[t] = 0.f;
            if (t < q_loads && e < q_elems) pre_q[t] = to_op(qp[e < P * 2 ? ob + e : ab + (e - P * 2)]);
        }
        pre_r = 0;
        if (lane < n_img) pre_r = a.relpos[((size_t)c.b * n_img + lane) * a.Lq_r + (a.Lq_r == 1 ? 0 : c.q)];
    };
    RowCursor cur = walk.first(a.ctas_per_sm, a.nsm);
    if (cur.ok) prefetch(cur);

    while (cur.ok) {
        const int b = cur.b, m = cur.m, q = cur.q;
        const size_t qm = ((size_t)b * Lq + q) * M + m;
        const int off_base = m * P * 2, att_base = M * P * 2 + m * n_lvl * (P + 1);
        __syncwarp();                                         // previous row done with qs / xs / s_vis
#pragma unroll
        for (int t = 0; t < kQPre; ++t)
            if (t < q_loads && lane + 32 * t < q_elems) qs[lane + 32 * t] = pre_q[t];
        const int r_mine = pre_r;
        int r_mine1 = 0;                                      // images 32..63 (second ballot chunk, rare)
        if (n_img > 32 && lane + 32 < n_img)
            r_mine1 = a.relpos[((size_t)b * n_img + lane + 32) * a.Lq_r + (a.Lq_r == 1 ? 0 : q)];
        const RowCursor nxt = walk.next(cur);
        if (nxt.ok) prefetch(nxt);                            // loads for the next row are now in flight

        // ---- visible images of this token (mask row; last row if the mask is shorter) ---------
        const unsigned vis = __ballot_sync(0xffffffffu, r_mine != 0);
        const unsigned vis1 = n_img > 32 ? __ballot_sync(0xffffffffu, r_mine1 != 0) : 0u;
        const int nvis = __popc(vis) + __popc(vis1);
        // list of images to walk: the visible ones (EMIT: all, masked ones flagged by bit 30)
        if (EMIT) {
            if (lane < n_img) s_vis[lane] = lane | (r_mine << 8) | (r_mine == 0 ? (1 << 30) : 0);
            if (lane + 32 < n_img) s_vis[lane + 32] = (lane + 32) | (r_mine1 << 8) | (r_mine1 == 0 ? (1 << 30) : 0);
        } else {
            if (r_mine != 0) s_vis[__popc(vis & ((1u << lane) - 1u))] = lane | (r_mine << 8);
            if (r_mine1 != 0) s_vis[__popc(vis) + __popc(vis1 & ((1u << lane) - 1u))] = (lane + 32) | (r_mine1 << 8);
        }
        __syncwarp();
        const int nlist = EMIT ? n_img : nvis;

        // ---- pass A: logits of the listed images -> xs[], softmax statistics ------------------
        // one pass per (image, chunk of 32 items): lane = item = (level, point) of that image
        float lmax = nullv;
        for (int vi = 0; vi < nlist; ++vi) {
            const int e = s_vis[vi];
            const T *rt = rtable + (size_t)((e >> 8) & 0xff) * C + att_base;
            for (int c0 = 0; c0 < img_passes; ++c0) {
                const int it = c0 * 32 + lane;
                if (it < per_img) {
                    const int l = c0 == 0 ? l_lane : it / P, pp = c0 == 0 ? p_lane : it - (it / P) * P;
                    float x = round_to<T>(qs[P * 2 + l * (P + 1) + pp] + to_op(rt[l * (P + 1) + pp]));
                    if (e & (1 << 30)) x = -INFINITY;   // EMIT only: masked image -> weight exactly 0
                    xs[(vi * img_passes + c0) * 32 + lane] = x;
                    lmax = fmaxf(lmax, x);
                }
            }
        }
        lmax = warp_max(lmax);
        float lsum = 0.f;
        for (int vi = 0; vi < nlist * img_passes; ++vi)
            if ((vi % img_passes) * 32 + lane < per_img) lsum += expf(xs[vi * 32 + lane] - lmax);
        const float e_null = expf(nullv - lmax);
        const float denom = warp_sum(lsum) + (float)L * e_null;   // one null slot per level, mmfs.py:225
        if (a.null_mass != nullptr && lane == 0)
            a.null_mass[qm] = (float)L * round_to<T>(__fdiv_rn(e_null, denom));

        if (!EMIT && nvis == 0) {   // no visible image: the sampled row is exactly zero
            float zero[VEC];
#pragma unroll
            for (int k = 0; k < VEC; ++k) zero[k] = 0.f;
            if (lane < LPR) stg_v4(static_cast<T *>(a.out) + qm * D + lane * VEC, Vec16<T>::pack(zero));
            cur = nxt;
            continue;
        }

        const char *slab = reinterpret_cast<const char *>(value + ((size_t)b * a.S * M + m) * D);
        const char *vbase = slab + (lane % LPR) * 16;
        const long long zero_off = reinterpret_cast<const char *>(g_zero_row) - slab;
        float acc[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[k] = 0.f;

        // ---- pass B: weights, sampling locations, taps, gather (one pass per image chunk) ------
        for (int vi = 0; vi < nlist; ++vi) {
            const int e = s_vis[vi];
            const int img = e & 0xff;
            const T *rt = rtable + (size_t)((e >> 8) & 0xff) * C + off_base;
            for (int c0 = 0; c0 < img_passes; ++c0) {
                const int it = c0 * 32 + lane;
                bool live = false;
                PointGeom<float> g;
                g.in_range = false; g.h_low = g.w_low = 0; g.lh = g.lw = 0.f;
                float aw = 0.f;
                int4 lv = make_int4(1, 1, 0, 0);
                if (it < per_img) {
                    const int l = c0 == 0 ? l_lane : it / P, pp = c0 == 0 ? p_lane : it - (it / P) * P;
                    const int gl = img * n_lvl + l;                   // global level index (n l), mmfs.py:198
                    aw = round_to<T>(__fdiv_rn(expf(xs[(vi * img_passes + c0) * 32 + lane] - lmax), denom));
                    if (EMIT || strict || aw != 0.f) {
                        lv = s_lvl[gl];
                        const float ox = round_to<T>(qs[pp * 2] + to_op(rt[pp * 2]));
                        const float oy = round_to<T>(qs[pp * 2 + 1] + to_op(rt[pp * 2 + 1]));
                        const float sc = s_scale[l];
                        // off * scale_ratio (mmfs.py:194-195), / (W, H) (mmfs.py:248-249): each a tensor op in
                        // the storage type in the reference, hence the intermediate roundings
                        const float tx = round_to<T>(__fdiv_rn(round_to<T>(__fmul_rn(ox, sc)), (float)lv.y));
                        const float ty = round_to<T>(__fdiv_rn(round_to<T>(__fmul_rn(oy, sc)), (float)lv.x));
                        const float *rp = a.refpts + ((((size_t)(a.Nr == 1 ? 0 : b) * Lq + q) * a.Lr) + (a.Lr == 1 ? 0 : gl)) * 2;
                        const float x = round_to<T>(__fadd_rn(rp[0], tx));   // fp32 ref + offset, cast to value dtype (mmfs.py:265)
                        const float y = round_to<T>(__fadd_rn(rp[1], ty));
                        if (EMIT) {
                            const size_t o = (qm * L + gl) * P + pp;
                            static_cast<T *>(a.loc_out)[2 * o] = from_op<T>(x);
                            static_cast<T *>(a.loc_out)[2 * o + 1] = from_op<T>(y);
                            static_cast<T *>(a.attn_out)[o] = from_op<T>(aw);
                        } else {
                            g = point_geom(x, y, lv.x, lv.y);
                            live = g.in_range;
                        }
                    }
                }
                if (EMIT) continue;
                const unsigned livemask = __ballot_sync(0xffffffffu, live);
                if (livemask == 0u) continue;
                __syncwarp();
                emit_taps(taps, lane, live, g, aw, lv.x, lv.y, lv.z, row_bytes, zero_off);
                __syncwarp();
                gather_pass<T, D>(taps, livemask, vbase, slot, acc);
            }
        }
        if (!EMIT) store_row<T, D>(acc, static_cast<T *>(a.out) + qm * D, lane);
        cur = nxt;
    }
}

template <typename T, int D, bool EMIT>
static int launch_sampler(SamplerArgs a, int N, cudaStream_t st) {
    const int L = a.n_img * a.n_lvl;
    const int xs_elems = a.n_img * ((a.n_lvl * a.P + 31) / 32) * 32;
    const int qs_elems = ((a.P * 2 + a.n_lvl * (a.P + 1) + 3) / 4) * 4;
    if (a.P * 2 + a.n_lvl * (a.P + 1) > 128) { set_error("mmfs_sampler: P*2 + n_lvl*(P+1) > 128 unsupported"); return MMFS_EUNSUPPORTED; }
    const size_t smem = (size_t)(L + (a.n_lvl + 3) / 4) * sizeof(int4) +
                        (size_t)kWarpsPerCta * (kTapsPerWarp * sizeof(Tap) + (size_t)(xs_elems + qs_elems) * 4 + 256);
    if (smem > 200 * 1024) { set_error("mmfs_sampler: n_img*n_lvl*P = %d too large", L * a.P); return MMFS_EUNSUPPORTED; }
    constexpr auto kern = mmfs_sampler_kernel<T, D, EMIT>;
    int rc = ensure_dynamic_smem<kern>(smem);
    if (rc != MMFS_OK) return rc;
    RowWalkPlan w;
    if ((rc = plan_row_walk(kern, smem, (long)N * a.M, a.Lq, 8, "mmfs_sampler", w)) != MMFS_OK) return rc;
    a.rows_per_warp = w.rows_per_warp; a.qtiles = w.qtiles; a.ntiles = w.ntiles; a.ctas_per_sm = w.ctas_per_sm; a.nsm = w.nsm;
    kern<<<w.grid, 32 * kWarpsPerCta, smem, st>>>(a);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

template <typename T>
static int dispatch_sampler(const SamplerArgs &a, int N, int D, bool emit, cudaStream_t st) {
    if (emit) return launch_sampler<T, 64, true>(a, N, st);   // D is irrelevant when nothing is gathered
    switch (D) {
        case 32: return launch_sampler<T, 32, false>(a, N, st);
        case 64: return launch_sampler<T, 64, false>(a, N, st);
        case 128: return launch_sampler<T, 128, false>(a, N, st);
        default:
            set_error("mmfs_sampler: head size %d has no fused gather path (use the emit + msda route)", D);
            return MMFS_EUNSUPPORTED;
    }
}

}  // namespace mmfs

using namespace mmfs;

static int sampler_entry(const void *value, const int64_t *shapes, const int64_t *starts, const void *qproj,
                         const void *rtable, const uint8_t *relpos, const float *refpts, const float *scale_ratios,
                         void *out, float *null_mass, void *loc_out, void *attn_out,
                         int N, int S, int M, int D, int n_img, int n_lvl, int Lq, int P,
                         int Lq_r, int Nr, int Lr, int R, int dtype, unsigned flags, void *stream, bool emit) {
    MMFS_CHECK_ARG(N >= 0 && Lq >= 0, "mmfs_sampler: negative batch or query count");
    MMFS_CHECK_ARG(S > 0 && M > 0 && D > 0 && n_img > 0 && n_lvl > 0 && P > 0 && R > 0,
                   "mmfs_sampler: non-positive dimension");
    MMFS_CHECK_ARG(n_img <= 64, "mmfs_sampler: at most 64 images per sequence (got %d)", n_img);
    MMFS_CHECK_ARG(R <= 256, "mmfs_sampler: relpos table too long (%d)", R);
    MMFS_CHECK_ARG(n_img < R, "mmfs_sampler: relative image indices reach n_img = %d but the table has only %d rows "
                   "(mmfs.py:177 asserts relpos < max_num_image_per_seq)", n_img, R);
    MMFS_CHECK_ARG((Lq_r == 1 || Lq_r == Lq) && (Nr == 1 || Nr == N) && (Lr == 1 || Lr == n_img * n_lvl),
                   "mmfs_sampler: broadcast dims must be 1 or full (Lq_r=%d Nr=%d Lr=%d)", Lq_r, Nr, Lr);
    MMFS_CHECK_ARG(dtype == MMFS_F32 || dtype == MMFS_F16 || dtype == MMFS_BF16, "mmfs_sampler: dtype %d unsupported", dtype);
    if (N == 0 || Lq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(shapes && starts && qproj && rtable && relpos && refpts && scale_ratios, "mmfs_sampler: null pointer argument");
    if (emit) MMFS_CHECK_ARG(loc_out && attn_out, "mmfs_sampler_locw: null output pointer");
    else MMFS_CHECK_ARG(value && out, "mmfs_sampler: null value/out pointer");
    if (!emit && ((uintptr_t)value % 16 != 0 || (uintptr_t)out % 16 != 0)) {
        set_error("mmfs_sampler: value/out must be 16-byte aligned");
        return MMFS_EUNSUPPORTED;
    }
    SamplerArgs a;
    a.value = value; a.shapes = shapes; a.starts = starts; a.qproj = qproj; a.rtable = rtable; a.relpos = relpos;
    a.refpts = refpts; a.scale_ratios = scale_ratios; a.out = out; a.null_mass = null_mass;
    a.loc_out = loc_out; a.attn_out = attn_out;
    a.S = S; a.M = M; a.n_img = n_img; a.n_lvl = n_lvl; a.Lq = Lq; a.P = P; a.Lq_r = Lq_r; a.Nr = Nr; a.Lr = Lr; a.R = R;
    a.null_logit = -logf((float)(n_img * n_lvl));
    a.flags = flags;
    cudaStream_t st = (cudaStream_t)stream;
    if (!emit && !(flags & MMFS_SAMPLER_GENERIC)) {   // the specialised kernel where its domain applies
        const int rc = launch_sampler_v2(a, N, D, dtype, st);
        if (rc != MMFS_EUNSUPPORTED) return rc;
    }
    return dispatch_dtype<kF32Types>(dtype, "mmfs_sampler", [&](auto tag) {
        return dispatch_sampler<typename decltype(tag)::type>(a, N, D, emit, st);
    });
}

extern "C" int mmfs_sampler_forward(const void *value, const int64_t *shapes, const int64_t *starts,
                                    const void *qproj, const void *rtable, const uint8_t *relpos,
                                    const float *refpts, const float *scale_ratios, void *out, float *null_mass,
                                    int N, int S, int M, int D, int n_img, int n_lvl, int Lq, int P,
                                    int Lq_r, int Nr, int Lr, int R, int dtype, unsigned flags, void *stream) {
    return sampler_entry(value, shapes, starts, qproj, rtable, relpos, refpts, scale_ratios, out, null_mass,
                         nullptr, nullptr, N, S, M, D, n_img, n_lvl, Lq, P, Lq_r, Nr, Lr, R, dtype, flags, stream, false);
}

extern "C" int mmfs_sampler_locw(const int64_t *shapes, const int64_t *starts, const void *qproj, const void *rtable,
                                 const uint8_t *relpos, const float *refpts, const float *scale_ratios,
                                 void *loc_out, void *attn_out, float *null_mass,
                                 int N, int M, int n_img, int n_lvl, int Lq, int P,
                                 int Lq_r, int Nr, int Lr, int R, int dtype, void *stream) {
    return sampler_entry(nullptr, shapes, starts, qproj, rtable, relpos, refpts, scale_ratios, nullptr, null_mass,
                         loc_out, attn_out, N, 1, M, 64, n_img, n_lvl, Lq, P, Lq_r, Nr, Lr, R, dtype, 0u, stream, true);
}
