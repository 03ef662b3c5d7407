// attn_common.cuh -- parameter block and register-level helpers of the wgmma attention kernel (attn_fwd_sm100.cu).
#pragma once
#include <stdlib.h>

#include "tc_common.cuh"

namespace mmfs {

struct AttnParams {
    void *out;                 // (B, Tq, H, hd), strides o_bs / o_ts elements
    const uint8_t *key_mask;   // (B, Tkv) or null
    int B, H, Tq, Tkv, causal, past;
    long o_bs, o_ts;
    float scale_log2e;         // scale * log2(e)
};

template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&t);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
    __half2 t = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&t);
}
__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

}  // namespace mmfs
