// linear_fp8_sm100.cu -- weight-only FP8 linear for the decode step: y = x * (w8 * scale)^T [+ bias] [+ residual]
// with x (M, K) bf16 / fp16, M <= 64, and w8 (N, K) e4m3 with one fp32 scale per output channel.
//
// The kernel streams the weights: every byte of w8 is read from HBM once per call.  A CTA owns kBN = 64 output
// channels and one K slice; each of its four warps owns 16 channels and streams their rows through its own ring of
// kStages shared-memory stages (one cp.async.bulk per row and stage, completing on the stage's mbarrier), so the warps
// never wait for one another inside the main loop.  x is staged in shared memory once per CTA (in windows of at most
// kXBudget bytes when M * K_slice is large).  The MMA is mma.sync m16n8k16 with the weights as the A operand (16
// channels) and x^T as B (8 rows of x per n8 tile); the e4m3 pairs are converted in registers with
// cvt.rn.f16x2.e4m3x2, and for bf16 x moved to bf16 exactly (bit shift into bf16 scaled by 2^-112, then a bf16x2
// multiply by 2^112).  A lane reads 16 contiguous weight bytes per row and 64-wide k step; the four MMAs of the step
// take them in an order of k that the B fragments (x read as 16 contiguous elements) follow too -- a dot product is
// indifferent to the order of its k.
//
// Split-K: the K slices of one channel tile form a thread-block cluster (gridDim.y = S <= 8 CTAs).  Each CTA leaves its
// fp32 partial tile in shared memory; after a cluster barrier each CTA reduces a share of the tile's outputs over the
// S partials in rank order through distributed shared memory, applies scale, bias and residual and rounds once.  No
// workspace, no atomics: two runs are bit-identical.  One launch, no host synchronisation: graph-capturable.
#include <cooperative_groups.h>

#include "common.cuh"

namespace mmfs {
namespace lfp8 {

namespace cg = cooperative_groups;

constexpr int kThreads = 128;                    // four warps
constexpr int kBN = 64;                          // output channels per CTA (16 per warp)
constexpr int kBK = 512;                         // k (= weight bytes per row) per ring stage
constexpr int kStages = 2;                       // 2 x 512: two CTAs per SM (3 x 256, 4 x 256, 3 x 512 and 2 x 1024
                                                 // measured slower on an H100 80GB HBM3 at 700 W)
constexpr int kRowPitch = kBK + 64;              // a row's stride in a stage: conflict-free 16-byte reads
constexpr int kWarpRing = kStages * 16 * kRowPitch;
constexpr int kRingBytes = 4 * kWarpRing;
constexpr int kXBudget = 32 * 1024;              // bytes of staged x per window
constexpr int kMaxSplits = 8;                    // portable cluster size
constexpr int kMaxM = 64;

struct Params {
    const void *x;
    const uint8_t *w;
    const float *scale;
    const void *bias;
    const void *residual;
    void *out;
    int M, N, K;
    int kc;       // K per split (multiple of kBK)
    int xk;       // k per staged x window (multiple of kBK)
};

__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t v16) {
    uint32_t r;
    asm("{\n\t.reg .b16 t;\n\tcvt.u16.u32 t, %1;\n\tcvt.rn.f16x2.e4m3x2 %0, t;\n\t}" : "=r"(r) : "r"(v16));
    return r;
}
// two e4m3 (low 16 bits of v16) -> the 16-bit MMA operand pair of T; both steps are exact
template <typename T> __device__ __forceinline__ uint32_t e4m3x2_to(uint32_t v16);
template <> __device__ __forceinline__ uint32_t e4m3x2_to<__half>(uint32_t v16) { return e4m3x2_to_f16x2(v16); }
template <> __device__ __forceinline__ uint32_t e4m3x2_to<__nv_bfloat16>(uint32_t v16) {
    const uint32_t h = e4m3x2_to_f16x2(v16);
    // an f16 made from e4m3 is zero or normal with its low 7 mantissa bits clear: exponent and top mantissa bits,
    // shifted into bf16's fields, give the same value times 2^(15 - 127) (never subnormal: e4m3's least is 2^-9)
    const uint32_t t = ((h >> 3) & 0x0fff0fffu) | (h & 0x80008000u);
    uint32_t r;
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(t), "r"(0x77807780u));   // * 2^112 in both halves
    return r;
}

template <typename T> struct Mma;
#define MMFS_LFP8_MMA(T, TY)                                                                                          \
    template <> struct Mma<T> {                                                                                       \
        __device__ __forceinline__ static void run(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, \
                                                   uint32_t b0, uint32_t b1) {                                        \
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." TY "." TY ".f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "     \
                         "{%8,%9}, {%0,%1,%2,%3};"                                                                     \
                         : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])                                              \
                         : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));                                     \
        }                                                                                                             \
    };
MMFS_LFP8_MMA(__nv_bfloat16, "bf16")
MMFS_LFP8_MMA(__half, "f16")
#undef MMFS_LFP8_MMA

__device__ __forceinline__ uint4 lds128(const void *p) {
    uint4 r;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(s_addr(p)));
    return r;
}

// MT: n8 tiles of x rows (M <= 8 * MT)
template <typename T, int MT>
__global__ void __launch_bounds__(kThreads) linear_fp8_kernel(const Params p) {
    extern __shared__ __align__(128) unsigned char smem[];
    constexpr int Mp = 8 * MT;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gid = lane >> 2, q = lane & 3;
    const int xpitch = 2 * p.xk + 16;                        // bytes per staged x row
    unsigned char *ring = smem + warp * kWarpRing;
    unsigned char *xs = smem + kRingBytes;
    float *part = reinterpret_cast<float *>(xs + Mp * xpitch);          // (Mp, kBN) fp32 partial of this CTA
    uint64_t *bars = reinterpret_cast<uint64_t *>(part + Mp * kBN) + warp * kStages;

    const int n0 = blockIdx.x * kBN, wrow0 = n0 + 16 * warp;
    const int kbeg = blockIdx.y * p.kc, kend = min(p.K, kbeg + p.kc);
    const int n_stages = (kend - kbeg + kBK - 1) / kBK;
    const int rows_valid = max(0, min(16, p.N - wrow0));

    // zero the ring: a short last stage leaves bytes past its k range untouched, and they meet x = 0 there (a stale
    // byte could be an e4m3 NaN pattern only before the first copy)
    for (int i = tid; i < kRingBytes / 16; i += kThreads) reinterpret_cast<uint4 *>(smem)[i] = make_uint4(0, 0, 0, 0);
    if (lane == 0)
        for (int s = 0; s < kStages; ++s) bar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    auto issue = [&](int s) {                                 // stage s of this warp's rows into ring slot s % kStages
        const int slot = s % kStages, k0 = kbeg + s * kBK;
        const int bytes = min(kBK, kend - k0);
        if (lane == 0) bar_expect_tx(&bars[slot], (uint32_t)(bytes * rows_valid));
        __syncwarp();
        if (lane < rows_valid)
            bulk_g2s(ring + slot * 16 * kRowPitch + lane * kRowPitch, p.w + (size_t)(wrow0 + lane) * p.K + k0,
                     (uint32_t)bytes, &bars[slot]);
    };
    for (int s = 0; s < kStages && s < n_stages; ++s) issue(s);

    float acc[MT][4];
#pragma unroll
    for (int t = 0; t < MT; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;

    const int stages_per_window = p.xk / kBK;
    const T *x = static_cast<const T *>(p.x);
    int wk0 = kbeg;
    for (int s = 0; s < n_stages; ++s) {
        if (s % stages_per_window == 0) {                     // stage the next window of x (zero past kend / M)
            wk0 = kbeg + s * kBK;
            __syncthreads();
            const int vec_per_row = p.xk / 8;
            for (int i = tid; i < Mp * vec_per_row; i += kThreads) {
                const int m = i / vec_per_row, c = i - m * vec_per_row, k = wk0 + 8 * c;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (m < p.M && k < kend) v = *reinterpret_cast<const uint4 *>(x + (size_t)m * p.K + k);
                *reinterpret_cast<uint4 *>(xs + m * xpitch + 16 * c) = v;
            }
            __syncthreads();
        }
        const int slot = s % kStages, k0 = kbeg + s * kBK;
        bar_wait(&bars[slot], (uint32_t)((s / kStages) & 1));
        const unsigned char *st = ring + slot * 16 * kRowPitch;
#pragma unroll
        for (int kk = 0; kk < kBK / 64; ++kk) {
            if (k0 + kk * 64 >= kend) break;
            const uint4 wa = lds128(st + gid * kRowPitch + kk * 64 + 16 * q);
            const uint4 wb = lds128(st + (gid + 8) * kRowPitch + kk * 64 + 16 * q);
            const uint32_t wa_w[4] = {wa.x, wa.y, wa.z, wa.w}, wb_w[4] = {wb.x, wb.y, wb.z, wb.w};
            uint32_t ra[8], rb[8];                            // pair j: weight bytes 2j, 2j+1 of this lane's 16
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                ra[2 * i] = e4m3x2_to<T>(wa_w[i] & 0xffffu);
                ra[2 * i + 1] = e4m3x2_to<T>(wa_w[i] >> 16);
                rb[2 * i] = e4m3x2_to<T>(wb_w[i] & 0xffffu);
                rb[2 * i + 1] = e4m3x2_to<T>(wb_w[i] >> 16);
            }
            const int xoff = 2 * (k0 - wk0 + kk * 64 + 16 * q);
#pragma unroll
            for (int t = 0; t < MT; ++t) {
                const unsigned char *xr = xs + (8 * t + gid) * xpitch + xoff;
                const uint4 x0 = lds128(xr), x1 = lds128(xr + 16);
                const uint32_t xw[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
                // MMA j: slots (2q, 2q+1) <- k 16q + 4j + (0, 1), slots (2q+8, 2q+9) <- k 16q + 4j + (2, 3)
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    Mma<T>::run(acc[t], ra[2 * j], rb[2 * j], ra[2 * j + 1], rb[2 * j + 1], xw[2 * j], xw[2 * j + 1]);
            }
        }
        __syncwarp();
        if (s + kStages < n_stages) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            issue(s + kStages);
        }
    }

    // accumulator (channel gid / gid + 8, x row 8t + 2q + c) -> partial[row][channel]
#pragma unroll
    for (int t = 0; t < MT; ++t)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int m = 8 * t + 2 * q + (c & 1), nl = 16 * warp + gid + 8 * (c >> 1);
            part[m * kBN + nl] = acc[t][c];
        }
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();
    const int rank = (int)cluster.block_rank(), S = (int)cluster.num_blocks();
    const T *bias = static_cast<const T *>(p.bias), *res = static_cast<const T *>(p.residual);
    T *out = static_cast<T *>(p.out);
    for (int e = rank * kThreads + tid; e < p.M * kBN; e += S * kThreads) {
        const int m = e / kBN, nl = e - m * kBN, n = n0 + nl;
        if (n >= p.N) continue;
        float sum = 0.f;
        for (int r = 0; r < S; ++r) sum += cluster.map_shared_rank(part, r)[e];   // rank order: deterministic
        float y = sum * p.scale[n];
        if (bias) y += to_op(bias[n]);
        if (res) y += to_op(res[(size_t)m * p.N + n]);
        out[(size_t)m * p.N + n] = from_op<T>(y);
    }
    cluster.sync();                                           // no CTA leaves while another reads its partial
}

struct Plan {
    int tiles, splits, kc, xk;
    size_t smem;
};

inline Plan make_plan(int M, int N, int K) {
    Plan pl;
    const int mp = (M + 7) / 8 * 8;
    pl.tiles = (N + kBN - 1) / kBN;
    int s = (2 * num_sms() + pl.tiles - 1) / pl.tiles;        // about two CTAs per SM
    s = s < 1 ? 1 : (s > kMaxSplits ? kMaxSplits : s);
    const int k_stages = (K + kBK - 1) / kBK;
    if (s > k_stages) s = k_stages;
    pl.kc = ((k_stages + s - 1) / s) * kBK;
    pl.splits = (K + pl.kc - 1) / pl.kc;
    int xk = kXBudget / (2 * mp) / kBK * kBK;
    if (xk < kBK) xk = kBK;
    pl.xk = xk < pl.kc ? xk : pl.kc;
    pl.smem = (size_t)kRingBytes + (size_t)mp * (2 * pl.xk + 16) + (size_t)mp * kBN * 4 + 4 * kStages * 8;
    return pl;
}

template <typename T, int MT>
int launch(const Params &p, const Plan &pl, cudaStream_t st) {
    auto kernel = linear_fp8_kernel<T, MT>;
    if (int rc = ensure_dynamic_smem<linear_fp8_kernel<T, MT>>(pl.smem)) return rc;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)pl.tiles, (unsigned)pl.splits, 1);
    cfg.blockDim = dim3(kThreads, 1, 1);
    cfg.dynamicSmemBytes = pl.smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1;
    attr[0].val.clusterDim.y = (unsigned)pl.splits;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MMFS_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
    return MMFS_OK;
}

template <typename T>
int dispatch_m(const Params &p, const Plan &pl, cudaStream_t st) {
    switch ((p.M + 7) / 8) {
        case 1: return launch<T, 1>(p, pl, st);
        case 2: return launch<T, 2>(p, pl, st);
        case 3: return launch<T, 3>(p, pl, st);
        case 4: return launch<T, 4>(p, pl, st);
        case 5: return launch<T, 5>(p, pl, st);
        case 6: return launch<T, 6>(p, pl, st);
        case 7: return launch<T, 7>(p, pl, st);
        default: return launch<T, 8>(p, pl, st);
    }
}

}  // namespace lfp8
}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_linear_fp8(const void *x, const uint8_t *w8, const float *scale, const void *bias,
                               const void *residual, void *out, int M, int N, int K, int dtype, void *stream) {
    using namespace mmfs::lfp8;
    MMFS_CHECK_ARG(M > 0 && N > 0 && K > 0, "linear_fp8: bad shape M=%d N=%d K=%d", M, N, K);
    if (M > kMaxM || K % 16 != 0) {
        set_error("linear_fp8: needs M <= %d and K a multiple of 16 (got M=%d K=%d)", kMaxM, M, K);
        return MMFS_EUNSUPPORTED;
    }
    MMFS_CHECK_ARG(x && w8 && scale && out, "linear_fp8: null pointer argument");
    MMFS_CHECK_ARG(((uintptr_t)x | (uintptr_t)w8) % 16 == 0, "linear_fp8: x and w8 must be 16-byte aligned");
    Params p{x, w8, scale, bias, residual, out, M, N, K, 0, 0};
    const Plan pl = make_plan(M, N, K);
    p.kc = pl.kc;
    p.xk = pl.xk;
    return dispatch_dtype<kF16Types, MMFS_EUNSUPPORTED>(dtype, "linear_fp8", [&](auto tag) {
        using T = typename decltype(tag)::type;
        return dispatch_m<T>(p, pl, (cudaStream_t)stream);
    });
}
