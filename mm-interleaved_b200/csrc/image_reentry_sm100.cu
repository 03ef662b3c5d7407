// image_reentry_sm100.cu -- a generated image re-entering the context as the visual tokenizer's input, on the device.
//
//   mmfs_image_reentry   (N, 3, S, S) fp32 image in [0, 1]  ->  (N, 3, R, R) fp32 tokenizer input
//
// Bit-identical to the host path of the interleaved inference loop (PIL 8-bit resampling, Resample.c):
//   1. quantisation of tensor_to_pil: u = uint8(clamp(x * 255 + 0.5, 0, 255)), each operation rounded in fp32;
//   2. center_crop_arr: BOX resizes to floor(size / 2) while size >= 2R, then a BICUBIC resize to R (skipped when the
//      size already is R: PIL returns a copy), then the centre crop, which is empty for a square image;
//   3. transform_numpy's tail: float32(u) / 255 in fp32, HWC -> CHW.
// Every resize is PIL's separable pass pair, horizontal first, each pass rounded and clipped to uint8: output index
// o of a resize in -> out takes the taps [xmin, xmin + n) of
//   scale = in / out, fs = max(scale, 1), support = filter_support * fs, center = (o + 0.5) * scale,
//   xmin = max((int)(center - support + 0.5), 0), xmax = min((int)(center + support + 0.5), in),
//   w_j = filter((xmin + j - center + 0.5) / fs) normalised by their sum, k_j = (int)(w_j * 2^22 +- 0.5),
//   pixel = clip8((2^21 + sum_j k_j * in_j) >> 22),
// with the weights computed in double exactly as PIL does (the device code uses the _rn intrinsics, so no operation is
// contracted into an FMA).
//
// One launch.  A CTA owns `tile` output rows of one image and walks the stage chain backwards once to find the rows
// of every intermediate image those rows depend on; it then runs the passes forwards over just those rows, with the
// intermediates in shared memory (uint8, HWC): the first pass reads and quantises the fp32 image straight from global
// memory, the last writes the fp32 output.  Each stage first tabulates its taps per output index in shared memory
// (square images: the horizontal and the vertical pass use the same table).  Neighbouring CTAs recompute the few rows their windows share.  Every output
// is computed by one thread in a fixed order with integer arithmetic: two runs are bit-identical.
#include "common.cuh"

namespace mmfs {
namespace reentry {

constexpr int kPrecisionBits = 22;   // PIL's PRECISION_BITS for 8-bit images: 32 - 8 - 2
constexpr int kMaxStages = 16;
constexpr int kMaxSize = 16384;
constexpr int kTileRows = 4;         // output rows per CTA (halved while the shared memory does not fit)
constexpr int kThreads = 256;
constexpr size_t kMaxSmem = 227 * 1024;
enum Filter { kBox = 0, kBicubic = 1 };

#ifdef __CUDA_ARCH__
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
#else
inline double dmul(double a, double b) { return a * b; }
inline double dadd(double a, double b) { return a + b; }
inline double ddiv(double a, double b) { return a / b; }
inline float fmul(float a, float b) { return a * b; }
inline float fadd(float a, float b) { return a + b; }
inline float fdiv(float a, float b) { return a / b; }
#endif

__host__ __device__ inline double filter_support(int f) { return f == kBox ? 0.5 : 2.0; }

__host__ __device__ inline double filter_eval(int f, double x) {
    if (f == kBox) return (x > -0.5 && x <= 0.5) ? 1.0 : 0.0;
    if (x < 0.0) x = -x;                                        // bicubic, a = -0.5
    if (x < 1.0) return dadd(dmul(dmul(dadd(dmul(1.5, x), -2.5), x), x), 1.0);
    if (x < 2.0) return dmul(dadd(dmul(dadd(dmul(dadd(x, -5.0), x), 8.0), x), -4.0), -0.5);
    return 0.0;
}

// Taps of output index o of a resize in -> out: writes the fixed-point weights to k (when not null) and the first
// tap to *xmin; returns the tap count.  The weights are evaluated twice (for the sum, then normalised) rather than
// kept in a local array.
__host__ __device__ inline int taps(int in, int out, int f, int o, int *k, int *xmin) {
    const double scale = ddiv((double)in, (double)out);
    const double fs = scale < 1.0 ? 1.0 : scale;
    const double support = dmul(filter_support(f), fs);
    const double center = dmul(dadd((double)o, 0.5), scale);
    const double ss = ddiv(1.0, fs);
    int lo = (int)dadd(dadd(center, -support), 0.5);
    if (lo < 0) lo = 0;
    int hi = (int)dadd(dadd(center, support), 0.5);
    if (hi > in) hi = in;
    const int n = hi - lo;
    *xmin = lo;
    if (k == nullptr) return n;
    double ww = 0.0;
    for (int j = 0; j < n; ++j) ww = dadd(ww, filter_eval(f, dmul(dadd(dadd((double)(lo + j), -center), 0.5), ss)));
    for (int j = 0; j < n; ++j) {
        const double w = filter_eval(f, dmul(dadd(dadd((double)(lo + j), -center), 0.5), ss));
        const double v = dmul(ww != 0.0 ? ddiv(w, ww) : w, (double)(1 << kPrecisionBits));
        k[j] = v < 0.0 ? (int)dadd(-0.5, v) : (int)dadd(0.5, v);
    }
    return n;
}

// Most taps of one output index of a resize in -> out: PIL's ksize, (int)ceil(support) * 2 + 1.
inline int max_taps(int in, int out, int f) {
    const double scale = (double)in / out;
    return (int)ceil(filter_support(f) * (scale < 1.0 ? 1.0 : scale)) * 2 + 1;
}

__host__ __device__ inline unsigned char clip8(int acc) {
    const int v = acc >> kPrecisionBits;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__host__ __device__ inline unsigned char quantise(float x) {   // tensor_to_pil
    float v = fadd(fmul(x, 255.f), 0.5f);
    v = v > 0.f ? v : 0.f;                                      // NaN -> 0
    v = v < 255.f ? v : 255.f;
    return (unsigned char)(int)v;
}

struct Plan {
    int n_stages;                     // resizes: the BOX halvings, then the bicubic one unless the size already is R
    int size[kMaxStages + 1];         // size[0] = S, size[n_stages] = R
    int filter[kMaxStages];
    int ksize[kMaxStages];            // taps table stride of each stage
    int tile;                         // output rows per CTA
    int bytes_x, bytes_y, bytes_t;    // shared memory: stage inputs, horizontal-pass outputs, the taps table
};

// Rows [lo[s], hi[s]) of the image after s resizes that output rows [a, b) need.
__host__ __device__ inline void row_spans(const Plan &p, int a, int b, int *lo, int *hi) {
    lo[p.n_stages] = a;
    hi[p.n_stages] = b;
    for (int s = p.n_stages - 1; s >= 0; --s) {
        int x0, x1;
        taps(p.size[s], p.size[s + 1], p.filter[s], lo[s + 1], nullptr, &x0);
        const int n1 = taps(p.size[s], p.size[s + 1], p.filter[s], hi[s + 1] - 1, nullptr, &x1);
        lo[s] = x0;
        hi[s] = x1 + n1;
    }
}

// Each pass is a loop over its items by (tid, nthr); the kernel separates them by barriers.
// The taps of stage s for every output index: table[o * ksize ...] weights, first[o] and count[o].  Images are square,
// so the horizontal and the vertical pass of a stage share them.
__host__ __device__ inline void fill_taps(const Plan &p, int s, int *table, int *first, int *count, int tid, int nthr) {
    for (int o = tid; o < p.size[s + 1]; o += nthr)
        count[o] = taps(p.size[s], p.size[s + 1], p.filter[s], o, table + o * p.ksize[s], first + o);
}

// Horizontal pass of stage s: rows [lo[s], hi[s]) of the stage input (the fp32 image for s = 0, else region x) into
// region y at the output width.
__host__ __device__ inline void pass_horizontal(const Plan &p, int s, const int *lo, const int *hi, const int *table,
                                                const int *first, const int *count, const float *img,
                                                const unsigned char *x, unsigned char *y, int tid, int nthr) {
    const int win = p.size[s], wout = p.size[s + 1], S = p.size[0], ks = p.ksize[s];
    const int items = (hi[s] - lo[s]) * wout;
    for (int i = tid; i < items; i += nthr) {
        const int r = i / wout, o = i - r * wout;
        const int *k = table + o * ks, x0 = first[o], n = count[o];
        int acc[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
        for (int j = 0; j < n; ++j) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int u = s == 0 ? quantise(img[((long)c * S + lo[0] + r) * S + x0 + j])
                                     : x[((long)r * win + x0 + j) * 3 + c];
                acc[c] += u * k[j];
            }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) y[((long)r * wout + o) * 3 + c] = clip8(acc[c]);
    }
}

// Vertical pass of stage s: region y into rows [lo[s + 1], hi[s + 1]) of region x, or, for the last stage, into the
// fp32 output (CHW, / 255).
__host__ __device__ inline void pass_vertical(const Plan &p, int s, const int *lo, const int *hi, const int *table,
                                              const int *first, const int *count, const unsigned char *y,
                                              unsigned char *x, float *out, int tid, int nthr) {
    const int w = p.size[s + 1], R = p.size[p.n_stages], ks = p.ksize[s];
    const bool last = s == p.n_stages - 1;
    const int items = (hi[s + 1] - lo[s + 1]) * w;
    for (int i = tid; i < items; i += nthr) {
        const int r = i / w, o = i - r * w, row = lo[s + 1] + r;
        const int *k = table + row * ks, y0 = first[row], n = count[row];
        int acc[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
        for (int j = 0; j < n; ++j) {
#pragma unroll
            for (int c = 0; c < 3; ++c) acc[c] += y[((long)(y0 + j - lo[s]) * w + o) * 3 + c] * k[j];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const unsigned char u = clip8(acc[c]);
            if (last)
                out[((long)c * R + row) * R + o] = fdiv((float)u, 255.f);
            else
                x[((long)r * w + o) * 3 + c] = u;
        }
    }
}

// No resize at all (S == R): the quantised image divided by 255.
__host__ __device__ inline void pass_copy(const Plan &p, int a, int b, const float *img, float *out, int tid, int nthr) {
    const int R = p.size[0];
    const int items = 3 * (b - a) * R;
    for (int i = tid; i < items; i += nthr) {
        const int c = i / ((b - a) * R), rem = i - c * (b - a) * R;
        const long off = ((long)c * R + a) * R + rem;
        out[off] = fdiv((float)quantise(img[off]), 255.f);
    }
}

// Shared-memory layout of a CTA: region x, region y, then the taps table, first taps and counts of one stage.
struct Smem {
    unsigned char *x, *y;
    int *table, *first, *count;
};

__host__ __device__ inline Smem carve(const Plan &p, int s, unsigned char *base) {
    Smem m;
    m.x = base;
    m.y = base + p.bytes_x;
    m.table = (int *)(base + p.bytes_x + p.bytes_y);
    m.first = m.table + p.size[s + 1] * p.ksize[s];
    m.count = m.first + p.size[s + 1];
    return m;
}

__global__ void __launch_bounds__(kThreads) reentry_kernel(const float *__restrict__ images, float *__restrict__ out,
                                                           const Plan p) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int lo[kMaxStages + 1], hi[kMaxStages + 1];
    const int S = p.size[0], R = p.size[p.n_stages];
    const int a = blockIdx.x * p.tile, b = min(a + p.tile, R);
    const float *img = images + (long)blockIdx.y * 3 * S * S;
    float *dst = out + (long)blockIdx.y * 3 * R * R;
    if (p.n_stages == 0) {
        pass_copy(p, a, b, img, dst, threadIdx.x, blockDim.x);
        return;
    }
    if (threadIdx.x == 0) row_spans(p, a, b, lo, hi);
    for (int s = 0; s < p.n_stages; ++s) {
        const Smem m = carve(p, s, smem);
        fill_taps(p, s, m.table, m.first, m.count, threadIdx.x, blockDim.x);
        __syncthreads();
        pass_horizontal(p, s, lo, hi, m.table, m.first, m.count, img, m.x, m.y, threadIdx.x, blockDim.x);
        __syncthreads();
        pass_vertical(p, s, lo, hi, m.table, m.first, m.count, m.y, m.x, dst, threadIdx.x, blockDim.x);
        __syncthreads();
    }
}

// The stage chain of S -> R and, for `tile` output rows per CTA, the largest shared-memory regions any CTA needs.
inline void make_plan(int S, int R, int tile, Plan *p) {
    p->n_stages = 0;
    p->size[0] = S;
    int size = S;
    while (size >= 2 * R) {                                     // center_crop_arr's BOX halvings
        p->filter[p->n_stages] = kBox;
        size /= 2;
        p->size[++p->n_stages] = size;
    }
    if (size != R) {                                            // round(size * R / size) == R for a square image
        p->filter[p->n_stages] = kBicubic;
        p->size[++p->n_stages] = R;
    }
    p->tile = tile;
    long bx = 0, by = 0, bt = 0;
    for (int s = 0; s < p->n_stages; ++s) {
        p->ksize[s] = max_taps(p->size[s], p->size[s + 1], p->filter[s]);
        const long t = (long)p->size[s + 1] * (p->ksize[s] + 2) * 4;
        if (t > bt) bt = t;
    }
    int lo[kMaxStages + 1], hi[kMaxStages + 1];
    for (int a = 0; a < R && p->n_stages > 0; a += tile) {
        row_spans(*p, a, a + tile < R ? a + tile : R, lo, hi);
        for (int s = 0; s < p->n_stages; ++s) {
            const long ys = (long)(hi[s] - lo[s]) * p->size[s + 1] * 3;
            const long xs = (long)(hi[s + 1] - lo[s + 1]) * p->size[s + 1] * 3;
            if (ys > by) by = ys;
            if (s + 1 < p->n_stages && xs > bx) bx = xs;
        }
    }
    p->bytes_x = (int)((bx + 15) / 16 * 16);
    p->bytes_y = (int)((by + 15) / 16 * 16);
    p->bytes_t = (int)((bt + 15) / 16 * 16);
}

}  // namespace reentry
}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_image_reentry(const float *images, float *out, int N, int C, int H, int W, int R, void *stream) {
    using namespace mmfs::reentry;
    MMFS_CHECK_ARG(N >= 0 && C > 0 && H > 0 && W > 0 && R > 0, "image_reentry: bad shape");
    if (C != 3 || H != W || H > kMaxSize || R > kMaxSize) {
        set_error("image_reentry: needs (N, 3, S, S) images and S, R <= %d (got C=%d H=%d W=%d R=%d)", kMaxSize, C, H, W,
                  R);
        return MMFS_EUNSUPPORTED;
    }
    if (N == 0) return MMFS_OK;
    MMFS_CHECK_ARG(images && out, "image_reentry: null pointer argument");
    MMFS_CHECK_ARG(N <= 65535, "image_reentry: more than 65535 images");
    Plan p;
    int tile = kTileRows;
    for (;; tile /= 2) {
        make_plan(H, R, tile, &p);
        if ((size_t)p.bytes_x + p.bytes_y + p.bytes_t <= kMaxSmem || tile == 1) break;
    }
    const size_t smem = (size_t)p.bytes_x + p.bytes_y + p.bytes_t;
    if (smem > kMaxSmem) {
        set_error("image_reentry: %d -> %d needs %zu bytes of shared memory per row", H, R, smem);
        return MMFS_EUNSUPPORTED;
    }
    if (int rc = ensure_dynamic_smem<reentry_kernel>(smem)) return rc;
    const dim3 grid((unsigned)((R + tile - 1) / tile), (unsigned)N);
    reentry_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(images, out, p);
    MMFS_CUDA(cudaGetLastError());
    return MMFS_OK;
}
