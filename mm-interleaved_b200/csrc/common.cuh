// common.cuh -- shared helpers for libmmfs_b200.so (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/mmfs_b200.h"

namespace mmfs {

// thread-local last-error text, returned by mmfs_last_error()
void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);

#define MMFS_CHECK_ARG(cond, ...)            \
    do {                                     \
        if (!(cond)) {                       \
            ::mmfs::set_error(__VA_ARGS__);  \
            return MMFS_EINVAL;              \
        }                                    \
    } while (0)

#define MMFS_CUDA(call)                                             \
    do {                                                            \
        cudaError_t _e = (call);                                    \
        if (_e != cudaSuccess) return ::mmfs::cuda_fail(_e, #call); \
    } while (0)

inline size_t dtype_size(int dtype) {
    switch (dtype) {
        case MMFS_F32: return 4;
        case MMFS_F16: return 2;
        case MMFS_BF16: return 2;
        case MMFS_F64: return 8;
        default: return 0;
    }
}

int num_sms();            // of the CURRENT device
int current_device();     // cudaGetDevice, -1 on failure
constexpr int kMaxDevices = 64;

// ---- launch policy shared by the entry points -------------------------------------------------------------------
// Element-type dispatch: returns f(DtypeTag<T>{}) for the element type T of `dtype` when the code is in the set
// Accepted (bits 1 << MMFS_*); only the accepted types are instantiated.  Any other code sets
// "<what>: dtype <code> unsupported" and returns Bad.
template <typename T> struct DtypeTag { using type = T; };
constexpr unsigned kF16Types = (1u << MMFS_F16) | (1u << MMFS_BF16);
constexpr unsigned kF32Types = (1u << MMFS_F32) | kF16Types;
constexpr unsigned kAllTypes = kF32Types | (1u << MMFS_F64);

template <unsigned Accepted, int Bad = MMFS_EINVAL, typename F>
int dispatch_dtype(int dtype, const char *what, F &&f) {
    switch (dtype) {
        case MMFS_F32: if constexpr ((Accepted >> MMFS_F32) & 1u) return f(DtypeTag<float>{}); break;
        case MMFS_F16: if constexpr ((Accepted >> MMFS_F16) & 1u) return f(DtypeTag<__half>{}); break;
        case MMFS_BF16: if constexpr ((Accepted >> MMFS_BF16) & 1u) return f(DtypeTag<__nv_bfloat16>{}); break;
        case MMFS_F64: if constexpr ((Accepted >> MMFS_F64) & 1u) return f(DtypeTag<double>{}); break;
    }
    set_error("%s: dtype %d unsupported", what, dtype);
    return Bad;
}

// Opts Kernel in to `bytes` of dynamic shared memory on the current device.  The attribute is per kernel and per
// device and is only ever raised: sizes within the 48 KiB default or within what was set before make no driver call.
template <auto Kernel>
int ensure_dynamic_smem(size_t bytes) {
    static size_t set[kMaxDevices] = {};
    if (bytes <= 48 * 1024) return MMFS_OK;
    const int dev = current_device();
    const bool tracked = dev >= 0 && dev < kMaxDevices;
    if (tracked && bytes <= set[dev]) return MMFS_OK;
    MMFS_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    if (tracked) set[dev] = bytes;
    return MMFS_OK;
}

// Grid of a grid-stride kernel: `blocks`, capped at per_sm CTAs per SM of the current device.
inline int capped_grid(long blocks, int per_sm) {
    const long cap = (long)num_sms() * per_sm;
    return (int)(blocks < cap ? blocks : cap);
}

// ---- element <-> opmath conversions ---------------------------------------------------
template <typename T> struct OpMath { using type = float; };
template <> struct OpMath<double> { using type = double; };

__device__ __forceinline__ float to_op(float x) { return x; }
__device__ __forceinline__ double to_op(double x) { return x; }
__device__ __forceinline__ float to_op(__half x) { return __half2float(x); }
__device__ __forceinline__ float to_op(__nv_bfloat16 x) { return __bfloat162float(x); }

template <typename T> __device__ __forceinline__ T from_op(typename OpMath<T>::type x);
template <> __device__ __forceinline__ float from_op<float>(float x) { return x; }
template <> __device__ __forceinline__ double from_op<double>(double x) { return x; }
template <> __device__ __forceinline__ __half from_op<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 from_op<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

// 16-byte vector of T unpacked to fp32 lanes
template <typename T> struct Vec16;
template <> struct Vec16<float> {
    static constexpr int N = 4;
    __device__ __forceinline__ static void unpack(const uint4 &v, float (&f)[4]) {
        f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
        f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
    }
    __device__ __forceinline__ static uint4 pack(const float (&f)[4]) {
        return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
    }
};
template <> struct Vec16<__nv_bfloat16> {
    static constexpr int N = 8;
    // bf16 -> fp32 is a 16-bit left shift: exact, one ALU op per element
    __device__ __forceinline__ static void unpack(const uint4 &v, float (&f)[8]) {
        f[0] = __uint_as_float(v.x << 16); f[1] = __uint_as_float(v.x & 0xffff0000u);
        f[2] = __uint_as_float(v.y << 16); f[3] = __uint_as_float(v.y & 0xffff0000u);
        f[4] = __uint_as_float(v.z << 16); f[5] = __uint_as_float(v.z & 0xffff0000u);
        f[6] = __uint_as_float(v.w << 16); f[7] = __uint_as_float(v.w & 0xffff0000u);
    }
    __device__ __forceinline__ static uint4 pack(const float (&f)[8]) {
        uint4 r;
        __nv_bfloat162 a = __floats2bfloat162_rn(f[0], f[1]); r.x = *reinterpret_cast<uint32_t *>(&a);
        __nv_bfloat162 b = __floats2bfloat162_rn(f[2], f[3]); r.y = *reinterpret_cast<uint32_t *>(&b);
        __nv_bfloat162 c = __floats2bfloat162_rn(f[4], f[5]); r.z = *reinterpret_cast<uint32_t *>(&c);
        __nv_bfloat162 d = __floats2bfloat162_rn(f[6], f[7]); r.w = *reinterpret_cast<uint32_t *>(&d);
        return r;
    }
};
template <> struct Vec16<__half> {
    static constexpr int N = 8;
    __device__ __forceinline__ static void unpack(const uint4 &v, float (&f)[8]) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float2 t = __half22float2(*reinterpret_cast<const __half2 *>(&w[i]));
            f[2 * i] = t.x; f[2 * i + 1] = t.y;
        }
    }
    __device__ __forceinline__ static uint4 pack(const float (&f)[8]) {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __half2 t = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
            w[i] = *reinterpret_cast<uint32_t *>(&t);
        }
        return make_uint4(w[0], w[1], w[2], w[3]);
    }
};

// read-only 16-byte gather through L1 (the value slab of one head is re-used by
// neighbouring queries, so we WANT L1 allocation here)
__device__ __forceinline__ uint4 ldg_nc_v4(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
// streaming loads for data touched exactly once (sampling locations / weights)
__device__ __forceinline__ uint32_t ldg_stream_u32(const void *p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream_v2(const void *p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint16_t ldg_stream_u16(const void *p) {
    uint16_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_v4(void *p, const uint4 &v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- mbarrier and bulk async copy (TMA engine) --------------------------------------------------------------------
__device__ __forceinline__ uint32_t s_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void bar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_addr(bar)) : "memory");
}
__device__ __forceinline__ void bar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "W_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra D_%=;\n\t"
        "bra W_%=;\n\t"
        "D_%=:\n\t}" ::"r"(s_addr(bar)), "r"(parity) : "memory");
}
// `bytes` (a multiple of 16) from global to shared memory, completing on `bar`
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
                 "r"(s_addr(dst)), "l"(src), "r"(bytes), "r"(s_addr(bar)) : "memory");
}

}  // namespace mmfs
