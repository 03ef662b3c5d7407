/*
 * include/mmfs_b200.h -- C ABI of libmmfs_b200.so (hand-written sm_90a kernels for
 * the MM-Interleaved interleaved image-text forward hot path).
 *
 * Plain pointers and sizes only: no torch / ATen types cross this boundary.  Every
 * entry point returns MMFS_OK (0) or a negative status; the message for the calling
 * thread's last failure is available from mmfs_last_error().  All kernels are
 * enqueued asynchronously on the caller's stream (cudaStream_t passed as void*; NULL =
 * the legacy default stream) and retain no references to their arguments, matching
 * the reference op's contract (ops/src/cuda/ms_deform_attn_cuda.cu:66: current ATen
 * stream, asynchronous return).  Unlike the reference, launch errors are returned to
 * the caller rather than printf-ed (ops/src/cuda/ms_deform_im2col_cuda.cuh:951-955).
 *
 * The reference-side binding for each symbol is shown in INTEGRATION.md.
 */
#ifndef MMFS_B200_H_
#define MMFS_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MMFS_B200_ABI_VERSION 1

/* status codes */
#define MMFS_OK            0
#define MMFS_EINVAL       (-1) /* bad argument (null pointer, non-positive dim, ...)    */
#define MMFS_EUNSUPPORTED (-2) /* shape / dtype outside what the kernels implement      */
#define MMFS_ECUDA        (-3) /* CUDA runtime / launch error, text in mmfs_last_error() */

/* element types (the reference dispatches double/float/half: cu:65; bf16 is a superset) */
#define MMFS_F32  0
#define MMFS_F16  1
#define MMFS_BF16 2
#define MMFS_F64  3

/* flags for mmfs_msda_forward */
#define MMFS_MSDA_STRICT 1u /* also fetch taps whose attention weight is exactly 0 (the
                               reference multiplies them in, which only matters when
                               `value` holds inf/nan); default skips those fetches */
#define MMFS_MSDA_W16    2u /* 16-bit element types only: round each tap weight (lerp * attention weight) to the
                               element type and accumulate value x weight with one fp32 FMA of the widened 16-bit
                               operands -- fewer instructions per fetch; the reference keeps fp32 weights, so
                               this is opt-in (error << one storage ulp of the result) */

/* flags for mmfs_sampler_forward (in addition to MMFS_MSDA_STRICT) */
#define MMFS_SAMPLER_EXACT_WEIGHTS 4u /* keep fp32 tap weights in the specialised 16-bit kernel (default there: weights
                                         rounded to the element type, mixed-precision FMA accumulate; bound in mmfs_sampler_v2_sm100.cu) */
#define MMFS_SAMPLER_GENERIC       8u /* force the generic kernel (A/B runs, tests) */

int mmfs_abi_version(void);
const char *mmfs_last_error(void);

/*
 * Multi-scale deformable attention forward.
 * Replaces ms_deform_attn_forward / ms_deform_attn_cuda_forward
 *   (ops/src/ms_deform_attn.h:20-39, ops/src/cuda/ms_deform_attn_cuda.cu:21-81) and the
 *   kernel + launcher ms_deformable_im2col_gpu_kernel / ms_deformable_im2col_cuda
 *   (ops/src/cuda/ms_deform_im2col_cuda.cuh:240-302, 926-957).
 *
 *   value           (N, S, M, D)        dtype, device, contiguous
 *   spatial_shapes  (L, 2) int64 [H,W]  DEVICE pointer (reference reads it on device, cu:68)
 *   level_start     (L,)   int64        DEVICE pointer (cu:69)
 *   sampling_loc    (N, Lq, M, L, P, 2) dtype, last dim (x, y) normalised to [0,1]
 *   attn_weight     (N, Lq, M, L, P)    dtype
 *   out             (N, Lq, M*D)        dtype; fully overwritten (no pre-zeroing needed;
 *                                       the reference allocates it with at::zeros, cu:55)
 * All N batch entries are processed by ONE launch (the reference launches N /
 * im2col_step kernels, cu:62-76; im2col_step only partitions launches and does not
 * change results, so it is not part of this ABI -- the Python shim validates it).
 * Accumulation is fp32 for f32/f16/bf16 and fp64 for f64 (at::opmath_type, cuh:32),
 * with one rounding to dtype at the store (cuh:300).
 */
int mmfs_msda_forward(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                      const void *sampling_loc, const void *attn_weight, void *out,
                      int N, int S, int M, int D, int L, int Lq, int P,
                      int dtype, unsigned flags, void *stream);

/*
 * Multi-scale deformable attention backward (training path).
 * Replaces ms_deform_attn_backward / ms_deform_attn_cuda_backward (ops/src/ms_deform_attn.h:41-61,
 * ops/src/cuda/ms_deform_attn_cuda.cu:84-166) and the col2im kernels (ops/src/cuda/ms_deform_im2col_cuda.cuh:304-923).
 * grad_out (N, Lq, M*D) dtype.  The three gradient buffers are FP32 (the reference also accumulates half
 * inputs in fp32 and casts afterwards, cu:122-129,156-160): grad_value (N,S,M,D) must be ZERO-INITIALISED by the
 * caller (it is accumulated with atomics, as in the reference); grad_loc (N,Lq,M,L,P,2) and grad_attn (N,Lq,M,L,P)
 * are fully overwritten.  dtype f32 / f16 / bf16; D in {32, 64, 128}.
 */
int mmfs_msda_backward(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                       const void *sampling_loc, const void *attn_weight, const void *grad_out,
                       float *grad_value, float *grad_loc, float *grad_attn,
                       int N, int S, int M, int D, int L, int Lq, int P, int dtype, void *stream);

/*
 * Same gradients, run-to-run REPRODUCIBLE (SURVEY.md 8 f4): grad_value contributions are accumulated as 64-bit fixed point
 * with integer atomics (associative => order-independent) and converted to fp32 once.  grad_value_fixed (N,S,M,D) int64
 * must be ZERO-INITIALISED by the caller; grad_value (N,S,M,D) fp32, grad_loc and grad_attn are fully overwritten;
 * scratch2 = two device floats (the fixed-point scale derived from max|grad_out| and its inverse).
 */
int mmfs_msda_backward_deterministic(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                                     const void *sampling_loc, const void *attn_weight, const void *grad_out,
                                     long long *grad_value_fixed, float *grad_value, float *grad_loc, float *grad_attn,
                                     float *scratch2, int N, int S, int M, int D, int L, int Lq, int P, int dtype, void *stream);

/*
 * Integer index stream of the sampler, for parity checking of the sampling-point index
 * math (same device function as the forward kernels use).  idx is int32
 * (N, Lq, M, L, P, 8) = [in_range, h_low, w_low, valid_mask(bit k = corner k+1 fetched),
 * ptr1, ptr2, ptr3, ptr4] with ptr_k the element offset of channel 0 relative to the level
 * base exactly as cuh:50-80 computes it (-1 when the corner is not fetched; all-zero /
 * -1 record when the point fails the in-range predicate of cuh:291).
 */
int mmfs_msda_index_stream(const int64_t *spatial_shapes, const int64_t *level_start,
                           const void *sampling_loc, int32_t *idx,
                           int N, int M, int D, int L, int Lq, int P,
                           int dtype, void *stream);

/*
 * Same op through HOST buffers: copies the inputs host->device, runs
 * mmfs_msda_forward, copies `out` back and synchronises the stream before returning.
 * This is the end-to-end form a host-side caller of the reference plugin would use;
 * spatial_shapes / level_start are HOST pointers here.  Device scratch is cached per
 * thread and grown on demand; mmfs_release_scratch() frees it.
 */
int mmfs_msda_forward_host(const void *value, const int64_t *spatial_shapes, const int64_t *level_start,
                           const void *sampling_loc, const void *attn_weight, void *out,
                           int N, int S, int M, int D, int L, int Lq, int P,
                           int dtype, unsigned flags, void *stream);
void mmfs_release_scratch(void);

/* Tuning knobs (benchmarks / tests only): rows per warp per tile (0 = automatic); mapping bit 0 =
 * plain tile order instead of the per-SM swizzle. */
int mmfs_msda_set_tuning(int rows_per_warp, int mapping);
/* Same for the specialised fused sampler: rows per warp per tile (0 = automatic); wmode 1 = 16-bit tap weights +
 * mixed-precision FMA (default), 0 = fp32 tap weights everywhere. */
int mmfs_sampler_set_tuning(int rows_per_warp, int wmode);

/*
 * Fused MMFS sampler: relpos-conditioned offsets / logits, image mask, null-slot softmax, sampling
 * locations and the deformable gather in one kernel.
 * Replaces MMFS.forward's middle section, ops/modules/mmfs.py:178-273 (everything between the
 * query projections and output_proj), including its MSDeformAttnFunction.apply call.
 *
 *   value        (N, S, M, D)  dtype; S = n_img * sum(H_l*W_l)               (mmfs.py:165-172)
 *   shapes       (n_img*n_lvl, 2) int64 [H,W], device; starts (n_img*n_lvl,) int64, device
 *   qproj        (N, Lq, C) dtype, C = M*P*2 + M*n_lvl*(P+1): [sampling_offsets | attention_weights]
 *                applied to dynamic_offset_mask(query), biases included   (mmfs.py:175,181,188)
 *   rtable       (R, C) dtype: the same two linears (no bias) applied to query_relpos.weight
 *   relpos       (N, n_img, Lq_r) uint8, Lq_r in {1, Lq}: relative image index, 0 = masked
 *                                                                            (mmfs.py:154-163)
 *   refpts       (Nr, Lq, Lr, 2) fp32, Nr in {1,N}, Lr in {1, n_img*n_lvl}   (mmfs.py:243-250)
 *   scale_ratios (n_lvl,) fp32                                                (mmfs.py:80-83)
 *   out          (N, Lq, M*D) dtype: the sampled features (input of output_proj, before the
 *                ignore-token term)
 *   null_mass    (N, Lq, M) fp32 or NULL: sum over levels of the null-slot weights, the factor of
 *                ignore_token in mmfs.py:236-241
 */
int mmfs_sampler_forward(const void *value, const int64_t *shapes, const int64_t *starts,
                         const void *qproj, const void *rtable, const uint8_t *relpos,
                         const float *refpts, const float *scale_ratios, void *out, float *null_mass,
                         int N, int S, int M, int D, int n_img, int n_lvl, int Lq, int P,
                         int Lq_r, int Nr, int Lr, int R, int dtype, unsigned flags, void *stream);

/*
 * Same front-end, but materialises what the reference materialises: sampling_locations
 * (N,Lq,M,L,P,2) and attention_weights (N,Lq,M,L,P) in dtype (mmfs.py:226-234, 243-265), L =
 * n_img*n_lvl.  Parity instrumentation, and the route for head sizes without a fused gather path
 * (follow with mmfs_msda_forward).
 */
int mmfs_sampler_locw(const int64_t *shapes, const int64_t *starts, const void *qproj, const void *rtable,
                      const uint8_t *relpos, const float *refpts, const float *scale_ratios,
                      void *loc_out, void *attn_out, float *null_mass,
                      int N, int M, int n_img, int n_lvl, int Lq, int P,
                      int Lq_r, int Nr, int Lr, int R, int dtype, void *stream);

/*
 * Row-wise / element-wise kernels of the Llama-MMFS decoder layer (csrc/llama_ops_sm100.cu).
 *   mmfs_rmsnorm   replaces LlamaRMSNorm.forward            decoders/modeling_llama_mmfs.py:53-70
 *   mmfs_layernorm nn.LayerNorm over the last dim (weight / bias may be NULL)
 *   mmfs_rope_qk   replaces apply_rotary_pos_emb            decoders/modeling_llama_mmfs.py:158-172
 *                  q, k are rotated IN PLACE in the (B, T, H, hd) layout of the projection output
 *                  (row strides in elements); cos/sin tables are fp32 (max_pos, hd) as built by
 *                  LlamaRotaryEmbedding (:119-151); position_ids int64 (B*T) or (T) when pos_per_batch=0
 *   mmfs_swiglu    replaces act_fn(gate_proj(x)) * up_proj(x) decoders/modeling_llama_mmfs.py:188-189
 *                  on one (rows, 2*inter) buffer holding [gate | up]
 */
int mmfs_rmsnorm(const void *x, const void *weight, void *y, long rows, int cols, float eps, int dtype, void *stream);
int mmfs_layernorm(const void *x, const void *weight, const void *bias, void *y, long rows, int cols, float eps,
                   int dtype, void *stream);
int mmfs_rope_qk(void *q, void *k, const float *cos_table, const float *sin_table, const int64_t *position_ids,
                 long n_tokens, int T_len, int H, int hd, int q_stride, int k_stride, int pos_per_batch,
                 int dtype, void *stream);
/* RoPE + KV-cache append in one pass (static-cache extension of LlamaAttention.forward, modeling_llama_mmfs.py:230-239):
 * q (n_tokens rows, q_stride elements apart, H x hd dense) is rotated in place; the rotated k and the v of token t of
 * batch entry b are written to row (slot + t) of k_cache / v_cache ((B, T_max, H, hd), batch / row strides cache_bs /
 * cache_ts in elements).  slot = *slot_dev when slot_dev != NULL (device int64: the graphed decode step), else slot_host.
 * The k operand itself is left unrotated. */
int mmfs_rope_qk_append(void *q, const void *k, const void *v, const float *cos_table, const float *sin_table,
                        const int64_t *position_ids, void *k_cache, void *v_cache, const int64_t *slot_dev, long slot_host,
                        long n_tokens, int T_len, int H, int hd, int q_stride, int k_stride, int v_stride, long cache_bs,
                        long cache_ts, int pos_per_batch, int dtype, void *stream);
int mmfs_swiglu(const void *gate_up, void *out, long rows, int inter, int dtype, void *stream);
/* GEGLU of the SD-UNet feed-forward (diffusers GEGLU: hidden, gate = proj(x).chunk(2); hidden * gelu(gate), exact erf
 * GELU), on one (rows, 2*inter) buffer holding [value | gate]. */
int mmfs_geglu(const void *value_gate, void *out, long rows, int inter, int dtype, void *stream);

/* Decode-step linear: y[M, N] = prologue(x)[M, K] . w[N, K]^T (+ residual[M, N]) for M <= 8 rows, f16 / bf16 -- the
 * q/k/v, o_proj, gate/up and down projections of one generated token (LlamaAttention.forward
 * decoders/modeling_llama_mmfs.py:217-280, LlamaMLP.forward :188-189) with the operator in front of them folded in:
 *   prologue 0: x as given;  1: LlamaRMSNorm(x) * norm_weight (:53-70, eps);  2: x is [M, 2K] = [gate | up] and the
 *   operand is act_fn(gate) * up (:188-189).
 * residual (may be NULL, may alias y) is added in fp32 before the single rounding of the result.  w rows are streamed
 * from HBM exactly once (HBM roofline: N * K * sizeof(T) bytes).  N % 32 == 0, K % 512 == 0, all pointers 16-byte aligned,
 * contiguous rows.  scratch: mmfs_linear_skinny_scratch_floats(N) floats that must be ZERO before the first call; every
 * call leaves them zero again (arrival tickets of the split between SMs + fp32 partial tiles), so one zeroed buffer of
 * the largest N serves every call made on one stream.  MMFS_EUNSUPPORTED for shapes outside these limits. */
long mmfs_linear_skinny_scratch_floats(int N);
/* measurement hooks: mode 0 = default (tensor-map TMA kernel when N % 128 == 0), 1 = per-lane cp.async kernel, 2 = TMA
 * kernel, + 4 = record per-CTA {entry, first stage, last stage, exit} globaltimer stamps, read back by ..._probe */
int mmfs_linear_skinny_set_tuning(int mode);
int mmfs_linear_skinny_probe(unsigned long long *host_out, int n_ctas);
int mmfs_linear_skinny(const void *x, const void *w, void *y, const void *residual, const void *norm_weight, float *scratch,
                       int M, int N, int K, int prologue, float eps, int dtype, void *stream);

/*
 * softmax(q k^T * scale + mask) v for decode (q_len = 1 over a KV cache) and small / odd shapes;
 * the tensor-core path for prefill shapes is mmfs_attn_forward.
 * Replaces the eager attention of LlamaAttention.forward (decoders/modeling_llama_mmfs.py:246-264).
 * q (B,Tq,H,hd), k/v (B,Tkv,H,hd), out (B,Tq,H,hd) with batch / token strides in elements;
 * key_mask (B,Tkv) uint8 1 = attend, or NULL; causal: query i sees keys j <= past + i.
 */
int mmfs_attn_generic(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                      int B, int H, int Tq, int Tkv, int hd,
                      long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                      float scale, int causal, int past, int dtype, void *stream);
/* Single-query attention over a KV cache (the decode step of generate_texts, q_len = 1), split over the key range:
 * q (B, 1, H, hd) with batch stride q_bs; k / v (B, Tkv, H, hd) views of the cache (row strides in elements, 16-byte
 * aligned rows); out (B, 1, H, hd).  scratch: mmfs_attn_decode_scratch_floats(B, H, Tkv, hd) floats of device memory,
 * private to the call until it completes (per-(b, h) arrival tickets, zeroed by the call itself on `stream`, + partials).
 * causal != 0: the query sits at position `past` and sees keys 0..past.  f32 / f16 / bf16, hd % 32 == 0, hd <= 256. */
long mmfs_attn_decode_scratch_floats(int B, int H, int Tkv, int hd);
/* measurement hook: warps per 256-key CTA of the hd-128 16-bit decode kernel: 4 (64 keys per warp, default) or 8 (32) */
int mmfs_attn_decode_set_tuning(int warps);
int mmfs_attn_decode(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask, float *scratch,
                     int B, int H, int Tkv, int hd, long q_bs, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs,
                     float scale, int causal, int past, int dtype, void *stream);

/*
 * softmax(q k^T * scale + mask) v on the tensor cores (wgmma, register accumulators, TMA tiles):
 * the prefill path.  Same argument meaning as mmfs_attn_generic; requires hd in {64, 128}, dtype
 * bf16 / f16, 16-byte aligned pointers and strides (MMFS_EUNSUPPORTED otherwise -- callers route
 * those cases to mmfs_attn_generic).  Replaces LlamaAttention.forward's eager attention
 * (decoders/modeling_llama_mmfs.py:246-264), CLIPXAttention.forward's xformers call
 * (encoders/vit_adapter/xattn.py:70-72) and the SD-UNet attention (decoders/sd.py:64-65).
 */
int mmfs_attn_forward(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                      int B, int H, int Tq, int Tkv, int hd,
                      long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                      float scale, int causal, int past, int dtype, void *stream);

/* The same op as a PERSISTENT kernel: the resident CTAs (1 per SM at hd 128, 2 at hd 64) walk the (batch, query tile,
 * head) items handed out by an atomic counter, with barriers and tensor maps set up once and the K / V ring running on
 * across items.  Taken when there are more items than resident CTAs (else the call runs the kernel above).
 * work_counter: one device uint32 that is ZERO when the kernel starts and private to the call until it completes. */
int mmfs_attn_forward_persistent(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                                 int B, int H, int Tq, int Tkv, int hd,
                                 long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                                 float scale, int causal, int past, int dtype, unsigned *work_counter, void *stream);

/*
 * 2-D convolution as an implicit GEMM on the tensor cores (wgmma, TMA-shifted input boxes, no im2col buffer).
 * Replaces the cuDNN convolutions diffusers' UNet issues in the denoise step (called from
 * utils/monkey_patch/sd_unet_forward_monkey_patch.py:235-366; 3x3 stride 1/2 and 1x1, NHWC).
 *   x (B,H,W,Cin) NHWC; w (Cout,KH,KW,Cin); out (B,Ho,Wo,Cout) NHWC; optional fused epilogue terms: bias (Cout),
 *   add_bc (B,Cout) [the ResNet block's time-embedding projection], residual (like out).
 * Requires bf16/f16, Cin % 64 == 0, Cout % 160 == 0, stride <= 2, output tileable by 8x16 (or 8x8 with even B) pixel
 * patches: MMFS_EUNSUPPORTED otherwise (callers keep those few layers -- conv_in / conv_out -- on the library path).
 */
int mmfs_conv2d_nhwc(const void *x, const void *w, const void *bias, const void *add_bc, const void *residual, void *out,
                     int B, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dtype, void *stream);

/*
 * GroupNorm (+ SiLU when silu != 0) on NHWC activations: the nn.GroupNorm(32) in front of every UNet convolution
 * (same call sites as mmfs_conv2d_nhwc).  x, y (B, HW, C) NHWC; gamma/beta (C) or NULL; stats = caller-provided
 * scratch of 128*B*G floats (per-chunk partial sums; reduced in a fixed order, so results are run-to-run reproducible).  f32 / f16 / bf16; C % (16/sizeof) == 0 and C*sizeof <= 16 KiB.
 */
int mmfs_groupnorm_nhwc(const void *x, const void *gamma, const void *beta, void *y, float *stats, int B, int HW, int C,
                        int G, float eps, int silu, int dtype, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MMFS_B200_H_ */
