// capi.cu -- process-wide pieces of the C ABI: error text, device info, the host-buffer
// entry point.  No torch / ATen types anywhere in this library.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace mmfs {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what) {
    set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
    return MMFS_ECUDA;
}

int current_device() {
    int dev = -1;
    return cudaGetDevice(&dev) == cudaSuccess ? dev : -1;
}

int num_sms() {
    static int cached[kMaxDevices] = {};             // per device: a process may drive several GPUs
    const int dev = current_device();
    if (dev >= 0 && dev < kMaxDevices && cached[dev] > 0) return cached[dev];
    int n = 0;
    if (dev >= 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0) {
        if (dev < kMaxDevices) cached[dev] = n;
        return n;
    }
    return 132;  // H100 SXM
}

// per-thread device scratch for the host-buffer entry points
struct Scratch {
    void *ptr = nullptr;
    size_t cap = 0;
};
static thread_local Scratch g_scratch;

static int scratch_reserve(size_t bytes) {
    if (bytes <= g_scratch.cap) return MMFS_OK;
    if (g_scratch.ptr) {
        MMFS_CUDA(cudaFree(g_scratch.ptr));
        g_scratch.ptr = nullptr;
        g_scratch.cap = 0;
    }
    MMFS_CUDA(cudaMalloc(&g_scratch.ptr, bytes));
    g_scratch.cap = bytes;
    return MMFS_OK;
}

}  // namespace mmfs

using namespace mmfs;

extern "C" int mmfs_abi_version(void) { return MMFS_B200_ABI_VERSION; }
extern "C" const char *mmfs_last_error(void) { return g_err; }

extern "C" void mmfs_release_scratch(void) {
    if (g_scratch.ptr) cudaFree(g_scratch.ptr);
    g_scratch.ptr = nullptr;
    g_scratch.cap = 0;
}

static inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" int mmfs_msda_forward_host(const void *value, const int64_t *shapes, const int64_t *starts,
                                      const void *loc, const void *attn, void *out,
                                      int N, int S, int M, int D, int L, int Lq, int P,
                                      int dtype, unsigned flags, void *stream) {
    const size_t es = dtype_size(dtype);
    MMFS_CHECK_ARG(es != 0, "msda_forward_host: unknown dtype code %d", dtype);
    MMFS_CHECK_ARG(N >= 0 && Lq >= 0 && S > 0 && M > 0 && D > 0 && L > 0 && P > 0,
                   "msda_forward_host: bad dimension");
    if (N == 0 || Lq == 0) return MMFS_OK;
    MMFS_CHECK_ARG(value && shapes && starts && loc && attn && out, "msda_forward_host: null pointer argument");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t b_val = (size_t)N * S * M * D * es;
    const size_t b_loc = (size_t)N * Lq * M * L * P * 2 * es;
    const size_t b_att = (size_t)N * Lq * M * L * P * es;
    const size_t b_out = (size_t)N * Lq * M * D * es;
    const size_t b_shp = (size_t)L * 2 * sizeof(int64_t), b_st = (size_t)L * sizeof(int64_t);
    const size_t o_val = 0, o_loc = o_val + align256(b_val), o_att = o_loc + align256(b_loc),
                 o_out = o_att + align256(b_att), o_shp = o_out + align256(b_out), o_st = o_shp + align256(b_shp);
    int rc = scratch_reserve(o_st + align256(b_st));
    if (rc != MMFS_OK) return rc;
    char *d = (char *)g_scratch.ptr;
    MMFS_CUDA(cudaMemcpyAsync(d + o_val, value, b_val, cudaMemcpyHostToDevice, st));
    MMFS_CUDA(cudaMemcpyAsync(d + o_loc, loc, b_loc, cudaMemcpyHostToDevice, st));
    MMFS_CUDA(cudaMemcpyAsync(d + o_att, attn, b_att, cudaMemcpyHostToDevice, st));
    MMFS_CUDA(cudaMemcpyAsync(d + o_shp, shapes, b_shp, cudaMemcpyHostToDevice, st));
    MMFS_CUDA(cudaMemcpyAsync(d + o_st, starts, b_st, cudaMemcpyHostToDevice, st));
    rc = mmfs_msda_forward(d + o_val, (const int64_t *)(d + o_shp), (const int64_t *)(d + o_st), d + o_loc,
                           d + o_att, d + o_out, N, S, M, D, L, Lq, P, dtype, flags, stream);
    if (rc != MMFS_OK) return rc;
    MMFS_CUDA(cudaMemcpyAsync(out, d + o_out, b_out, cudaMemcpyDeviceToHost, st));
    MMFS_CUDA(cudaStreamSynchronize(st));
    return MMFS_OK;
}
