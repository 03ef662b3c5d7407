// conv_igemm_sm100.cu -- 2-D convolution as an implicit GEMM on the Hopper tensor cores (wgmma; NHWC, bf16 / f16).
//
// The SD-2.1 UNet convolutions of the denoise step (3x3 stride 1 / 2, 1x1 shortcuts; arithmetic in diffusers 0.20,
// called from utils/monkey_patch/sd_unet_forward_monkey_patch.py:235-366 -- cuDNN in the reference) as ONE kernel:
//   out[b, ho, wo, n] = bias[n] + add_bc[b, n] + residual[b, ho, wo, n] + sum_{kh,kw,c} x[b, ho*s+kh-p, wo*s+kw-p, c] * w[n, kh, kw, c]
// GEMM view: M = output pixels, N = Cout, K = KH*KW*Cin.  No im2col buffer exists anywhere:
//   * an M tile is a TB x TH x TW patch of 128 output pixels; for filter tap (kh, kw) and channel block c0 its A tile
//     is the SAME-shaped box of the input shifted by (kh-p, kw-p): one 4-D TMA load {64 ch, TW, TH, TB} with the tensor
//     map's element strides carrying the conv stride, and TMA's out-of-bounds zero fill providing the padding
//     (negative / overshooting coordinates).  It lands in shared memory as 128 rows x 128 B, SWIZZLE_128B -- exactly a
//     K-major wgmma A operand;
//   * the B tile is a {64, BN} box of the weights stored (Cout, KH, KW, Cin) = (N, K) K-major;
//   * the B tile is a {64, BN} box of the weights; BN (the Cout tile) is 160 when it divides Cout (the UNet's
//     320 / 640 / 1280 = 2 / 4 / 8 x 160), else 128 (the VAE decoder's 128 / 256 / 512);
//   * k loop = KH*KW*(Cin/64) pipeline stages; warpgroups 0 and 1 each own 64 of the 128 pixels and issue 4 wgmma
//     m64nBNk16 per stage into a register accumulator, keeping one stage's MMAs in flight while the next one's wait;
//   * 4-stage TMA -> wgmma mbarrier pipeline, warp 8 = TMA producer; epilogue straight from the accumulator fragment
//     (+ bias / per-(b,n) time-embedding term / residual, 4-byte NHWC stores);
//   * 144 KB (BN 160) / 128 KB (BN 128) shared memory, 1 CTA per SM (two would need <= 96 registers per thread; the
//     64 x 160 fp32 accumulator alone takes 80).
//
// UP = true: nearest 2x upsample followed by a 3x3 / pad-1 convolution, without the 4x-size upsampled tensor.  Output
// pixel (2i + py, 2j + px) of conv3x3(up2x(X)) reads upsampled rows 2i + py - 1 .. 2i + py + 1, i.e. low-resolution
// rows {i-1, i, i} (py = 0) or {i, i, i+1} (py = 1), and the same along columns.  So each output parity ("phase")
// (py, px) is a 2x2 convolution over X with folded weights -- rows: py = 0 -> {w0, w1 + w2} at pad 1, py = 1 ->
// {w0 + w1, w2} at pad 0 -- read from (4, Cout, 2, 2, Cin) (ops.fold_up2x_weights).  blockIdx.z is the phase; the
// tiles walk the (H, W) low-resolution grid and the epilogue stores pixel (ho, wo) to (2 ho + py, 2 wo + px) of the
// (2H, 2W) output.  TMA's zero fill at X[-1] / X[H] is exactly the padding of the upsampled map.
//
// The VAE encoder's downsampler, conv3x3(F.pad(x, (0, 1, 0, 1)), stride 2), is the UP = false kernel at pad 0 / stride 2
// with the (H/2, W/2) output grid given by its entry point: the one-sided pad is the zero fill of row H / column W.
// Roofline: tensor (2*M*N*K flop).
#include "tc_common.cuh"

namespace mmfs {

constexpr int kConvStages = 4;
constexpr int kConvThreads = 288;     // 2 consumer warpgroups + 1 producer warp
constexpr int kConvConsumers = 256;

struct ConvParams {
    void *out;
    const void *bias, *add_bc, *residual;   // each may be null; bias (Cout), add_bc (B, Cout), residual like out
    int B, Ho, Wo, Cin, Cout, KH, KW, stride, pad;   // UP: Ho, Wo = the low-resolution H, W; KH = KW = 2
    int TW, TH, TB;                         // M tile = TB x TH x TW = 128 output pixels
    int tiles_w, tiles_h;                   // tiles per image along w / h
};

template <typename T> __device__ __forceinline__ uint32_t cpack2(float a, float b);
template <> __device__ __forceinline__ uint32_t cpack2<__nv_bfloat16>(float a, float b) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&t);
}
template <> __device__ __forceinline__ uint32_t cpack2<__half>(float a, float b) {
    __half2 t = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&t);
}
template <typename T> __device__ __forceinline__ float2 cunpack2(const T *p);
template <> __device__ __forceinline__ float2 cunpack2<__nv_bfloat16>(const __nv_bfloat16 *p) {
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(p));
}
template <> __device__ __forceinline__ float2 cunpack2<__half>(const __half *p) {
    return __half22float2(*reinterpret_cast<const __half2 *>(p));
}

template <typename T, int BN, bool UP>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_w, const ConvParams p) {
    static_assert(BN == 160 || BN == 128, "Cout tile");
    constexpr uint32_t A_BYTES = 128 * 128, B_BYTES = BN * 128, STAGE_BYTES = A_BYTES + B_BYTES;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    if ((s_addr(smem_raw) & 1023u) != 0u) { asm volatile("trap;"); }
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + kConvStages * STAGE_BYTES);
    uint64_t *full = bars, *empty = bars + kConvStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // M tile -> (batch group, h tile, w tile)
    int t = blockIdx.x;
    const int wt = t % p.tiles_w; t /= p.tiles_w;
    const int ht = t % p.tiles_h; t /= p.tiles_h;
    const int b0 = t * p.TB, h0 = ht * p.TH, w0 = wt * p.TW;
    const int n0 = blockIdx.y * BN;
    const int kc = p.Cin / 64;
    const int n_k = p.KH * p.KW * kc;

    if (threadIdx.x == 0) {
        for (int i = 0; i < kConvStages; ++i) { bar_init(full + i, 1); bar_init(empty + i, kConvConsumers); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int it = 0; it < n_k; ++it) {
                const int s = it % kConvStages;
                const uint32_t ph = (it / kConvStages) & 1;
                bar_wait(empty + s, ph ^ 1);
                const int tap = it / kc, cb = it - tap * kc;
                const int kh = tap / p.KW, kw = tap - kh * p.KW;
                uint8_t *sa = smem_raw + s * STAGE_BYTES;
                bar_expect_tx(full + s, STAGE_BYTES);
                // input coordinates of the tile's first output pixel for this tap; out-of-range -> zero fill = padding
                if constexpr (UP) {                   // phase (py, px): pad 1 - py rows, 1 - px columns; weights of the phase
                    const int phase = blockIdx.z;
                    tma_load_4d(sa, &map_x, full + s, cb * 64, w0 + kw - 1 + (phase & 1), h0 + kh - 1 + (phase >> 1), b0);
                    tma_load_2d(sa + A_BYTES, &map_w, full + s, tap * p.Cin + cb * 64, phase * p.Cout + n0);
                } else {
                    tma_load_4d(sa, &map_x, full + s, cb * 64, w0 * p.stride + kw - p.pad, h0 * p.stride + kh - p.pad, b0);
                    tma_load_2d(sa + A_BYTES, &map_w, full + s, tap * p.Cin + cb * 64, n0);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2;                         // pixels [64 wg, 64 wg + 64) of the tile
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int it = 0; it < n_k; ++it) {
        const int s = it % kConvStages;
        bar_wait(full + s, (it / kConvStages) & 1);
        const uint32_t sa = s_addr(smem_raw) + s * STAGE_BYTES;
        reg_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint64_t da = smem_desc(sa + wg * 64 * 128 + kk * 32, 16, 1024), db = smem_desc(sa + A_BYTES + kk * 32, 16, 1024);
            if constexpr (BN == 160) Wgmma<T>::ss_n160(acc, da, db, 1);
            else Wgmma<T>::ss_n128(acc, da, db, 1);
        }
        wgmma_commit();
        wgmma_wait<1>();                              // the previous stage's MMAs have retired: release its buffers
        reg_fence(acc);
        if (it > 0) bar_arrive(empty + (it - 1) % kConvStages);
    }
    wgmma_wait<0>();
    reg_fence(acc);

    // epilogue: thread holds pixels (row, row + 8) x channels 8 j + 2 (lane % 4) + {0, 1}
    const int tq = lane & 3;
    const T *bp = p.bias ? static_cast<const T *>(p.bias) + n0 + 2 * tq : nullptr;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
        const int pw = row % p.TW, phh = (row / p.TW) % p.TH, pb = row / (p.TW * p.TH);
        const int b = b0 + pb, ho = h0 + phh, wo = w0 + pw;
        if (b >= p.B || ho >= p.Ho || wo >= p.Wo) continue;
        size_t pix;
        if constexpr (UP) pix = ((size_t)b * 2 * p.Ho + 2 * ho + (blockIdx.z >> 1)) * 2 * p.Wo + 2 * wo + (blockIdx.z & 1);
        else pix = ((size_t)b * p.Ho + ho) * p.Wo + wo;
        T *op = static_cast<T *>(p.out) + pix * p.Cout + n0 + 2 * tq;
        const T *rp = p.residual ? static_cast<const T *>(p.residual) + pix * p.Cout + n0 + 2 * tq : nullptr;
        const T *ap = p.add_bc ? static_cast<const T *>(p.add_bc) + (size_t)b * p.Cout + n0 + 2 * tq : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            float e0 = acc[j * 4 + 2 * i], e1 = acc[j * 4 + 2 * i + 1];
            if (bp) { const float2 f = cunpack2<T>(bp + j * 8); e0 += f.x; e1 += f.y; }
            if (ap) { const float2 f = cunpack2<T>(ap + j * 8); e0 += f.x; e1 += f.y; }
            if (rp) { const float2 f = cunpack2<T>(rp + j * 8); e0 += f.x; e1 += f.y; }
            *reinterpret_cast<uint32_t *>(op + j * 8) = cpack2<T>(e0, e1);
        }
    }
}

}  // namespace mmfs

using namespace mmfs;

namespace {

// Cout tile: 160 when it divides Cout, else 128; 0 when neither does
int conv_bn(int Cout) { return Cout % 160 == 0 ? 160 : Cout % 128 == 0 ? 128 : 0; }

template <auto kern>
int launch(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap &mx, const CUtensorMap &mw, const ConvParams &p) {
    const int rc = ensure_dynamic_smem<kern>(smem);
    if (rc != MMFS_OK) return rc;
    kern<<<grid, kConvThreads, smem, st>>>(mx, mw, p);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}

// Output grid (Ho, Wo) from the caller: the (H, W) low-resolution grid per phase for UP (KH = KW = 2; the per-phase
// padding is set in the kernel), the symmetric-padding size for mmfs_conv2d_nhwc, (H/2, W/2) for the one-sided pad
template <bool UP>
int launch_conv(const char *what, const void *x, const void *w, const void *bias, const void *add_bc, const void *residual,
                void *out, int B, int H, int W, int Ho, int Wo, int Cin, int Cout, int KH, int KW, int stride, int pad,
                int dtype, void *stream) {
    int TW, TH, TB;
    if (Wo % 16 == 0 && Ho % 8 == 0) { TW = 16; TH = 8; TB = 1; }
    else if (Wo == 8 && Ho == 8 && B % 2 == 0) { TW = 8; TH = 8; TB = 2; }
    else { set_error("%s: output %dx%d (B=%d) is not tileable by the 128-pixel patches", what, Ho, Wo, B); return MMFS_EUNSUPPORTED; }
    const int BN = conv_bn(Cout);
    if (!(dtype == MMFS_BF16 || dtype == MMFS_F16) || Cin % 64 != 0 || BN == 0 || stride > 2 ||
        ((uintptr_t)x | (uintptr_t)w | (uintptr_t)out | (uintptr_t)bias | (uintptr_t)add_bc | (uintptr_t)residual) % 16 != 0) {
        set_error("%s: needs bf16/f16, Cin %% 64 == 0, Cout %% 160 == 0 or Cout %% 128 == 0, stride <= 2, 16-byte aligned "
                  "pointers (Cin=%d Cout=%d)", what, Cin, Cout);
        return MMFS_EUNSUPPORTED;
    }
    EncodeTiledFn enc = tensor_map_encoder();
    if (!enc) { set_error("%s: cuTensorMapEncodeTiled unavailable", what); return MMFS_ECUDA; }
    const CUtensorMapDataType dt = dtype == MMFS_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const int phases = UP ? 4 : 1;          // UP: the weights are (4, Cout, 2, 2, Cin) = (4 Cout, K) rows
    CUtensorMap mx, mw;
    {
        const cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
        const cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
        const cuuint32_t box[4] = {64, (cuuint32_t)(TW * stride), (cuuint32_t)(TH * stride), (cuuint32_t)TB};
        const cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
        CUresult r = enc(&mx, dt, 4, const_cast<void *>(x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("%s: tensor map (input) failed (%d)", what, (int)r); return MMFS_ECUDA; }
    }
    {
        const cuuint64_t K = (cuuint64_t)KH * KW * Cin;
        const cuuint64_t dims[2] = {K, (cuuint64_t)Cout * phases};
        const cuuint64_t strides[1] = {K * 2};
        const cuuint32_t box[2] = {64, (cuuint32_t)BN};
        const cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&mw, dt, 2, const_cast<void *>(w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { set_error("%s: tensor map (weights) failed (%d)", what, (int)r); return MMFS_ECUDA; }
    }
    ConvParams p;
    p.out = out; p.bias = bias; p.add_bc = add_bc; p.residual = residual;
    p.B = B; p.Ho = Ho; p.Wo = Wo; p.Cin = Cin; p.Cout = Cout; p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad;
    p.TW = TW; p.TH = TH; p.TB = TB; p.tiles_w = Wo / TW; p.tiles_h = Ho / TH;
    const size_t smem = (size_t)kConvStages * (128 * 128 + BN * 128) + 2 * kConvStages * 8;
    dim3 grid((unsigned)(p.tiles_w * p.tiles_h * (B / TB)), (unsigned)(Cout / BN), (unsigned)phases);
    cudaStream_t st = (cudaStream_t)stream;
    return dispatch_dtype<kF16Types>(dtype, what, [&](auto tag) {
        using T = typename decltype(tag)::type;
        return BN == 160 ? launch<conv_igemm_kernel<T, 160, UP>>(grid, smem, st, mx, mw, p)
                         : launch<conv_igemm_kernel<T, 128, UP>>(grid, smem, st, mx, mw, p);
    });
}

}  // namespace

// x (B, H, W, Cin) NHWC, w (Cout, KH, KW, Cin), out (B, Ho, Wo, Cout) NHWC; bias (Cout), add_bc (B, Cout), residual like out: may be null
extern "C" int mmfs_conv2d_nhwc(const void *x, const void *w, const void *bias, const void *add_bc, const void *residual, void *out,
                                int B, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad,
                                int dtype, void *stream) {
    MMFS_CHECK_ARG(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && KH > 0 && KW > 0 && stride > 0 && pad >= 0, "conv2d_nhwc: bad dimension");
    MMFS_CHECK_ARG(x && w && out, "conv2d_nhwc: null pointer argument");
    const int Ho = (H + 2 * pad - KH) / stride + 1, Wo = (W + 2 * pad - KW) / stride + 1;
    return launch_conv<false>("conv2d_nhwc", x, w, bias, add_bc, residual, out, B, H, W, Ho, Wo, Cin, Cout, KH, KW, stride,
                              pad, dtype, stream);
}

// x (B, H, W, Cin) NHWC, w_phases (4, Cout, 2, 2, Cin) folded per output parity, out (B, 2H, 2W, Cout) NHWC; bias (Cout) may be null
extern "C" int mmfs_conv2d_up2x_nhwc(const void *x, const void *w_phases, const void *bias, void *out, int B, int H, int W, int Cin,
                                     int Cout, int dtype, void *stream) {
    MMFS_CHECK_ARG(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv2d_up2x_nhwc: bad dimension");
    MMFS_CHECK_ARG(x && w_phases && out, "conv2d_up2x_nhwc: null pointer argument");
    return launch_conv<true>("conv2d_up2x_nhwc", x, w_phases, bias, nullptr, nullptr, out, B, H, W, H, W, Cin, Cout, 2, 2, 1, 0,
                             dtype, stream);
}

// x (B, H, W, Cin) NHWC, w (Cout, 3, 3, Cin), out (B, H/2, W/2, Cout) NHWC; bias (Cout) may be null.
// conv3x3(pad(x, bottom 1, right 1), stride 2): diffusers' Downsample2D(padding=0).  Pad 0, stride 2: the last output
// row reads input rows H-2 .. H, and row H (column W) is TMA's zero fill -- exactly the one-sided pad.
extern "C" int mmfs_conv2d_down2x_nhwc(const void *x, const void *w, const void *bias, void *out, int B, int H, int W, int Cin,
                                       int Cout, int dtype, void *stream) {
    MMFS_CHECK_ARG(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "conv2d_down2x_nhwc: bad dimension");
    MMFS_CHECK_ARG(x && w && out, "conv2d_down2x_nhwc: null pointer argument");
    MMFS_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "conv2d_down2x_nhwc: odd H or W");
    return launch_conv<false>("conv2d_down2x_nhwc", x, w, bias, nullptr, nullptr, out, B, H, W, H / 2, W / 2, Cin, Cout, 3, 3,
                              2, 0, dtype, stream);
}
