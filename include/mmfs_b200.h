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

#define MMFS_B200_ABI_VERSION 3

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

/* flags for mmfs_sampler_forward (in addition to MMFS_MSDA_STRICT) */
#define MMFS_SAMPLER_EXACT_WEIGHTS 4u /* keep fp32 tap weights in the specialised 16-bit kernel for this call (without
                                         it that kernel rounds each tap weight to the element type and accumulates with
                                         a mixed-precision FMA; error bound in mmfs_sampler_v2_sm100.cu).  Bit 2u is
                                         unused. */
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
 * With more (batch, query tile, head) items than resident CTAs (1 per SM at hd 128, 2 at hd 64) the kernel runs
 * PERSISTENT: the resident CTAs walk the items handed out by an atomic counter, with barriers and tensor maps set up
 * once and the K / V ring running on across items.  work_counter: one device uint32 of scratch, private to the call
 * until it completes; the call zeroes it on `stream` when it runs persistent (the caller need not).
 */
int mmfs_attn_forward(const void *q, const void *k, const void *v, void *out, const uint8_t *key_mask,
                      int B, int H, int Tq, int Tkv, int hd,
                      long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                      float scale, int causal, int past, int dtype, unsigned *work_counter, void *stream);

/*
 * mmfs_attn_forward that also writes the row log-sum-exp the backward pass needs (training path).  Same arguments,
 * requirements and output (O is bit-identical to mmfs_attn_forward's), plus
 *   lse  (B, H, Tq) fp32, contiguous: lse[b,h,i] = ln sum_j exp(scale * q_i . k_j) over the keys row i sees, in
 *        NATURAL-log units; +INFINITY for a row that sees no key (its output row is 0, and +inf makes every
 *        recomputed probability of that row exp(s - inf) = 0, so it gets zero gradient).
 */
int mmfs_attn_forward_lse(const void *q, const void *k, const void *v, void *out, float *lse, const uint8_t *key_mask,
                          int B, int H, int Tq, int Tkv, int hd,
                          long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                          float scale, int causal, int past, int dtype, unsigned *work_counter, void *stream);

/*
 * Gradient of out = softmax(q k^T * scale + mask) v for the causal prefill of LlamaAttention under autograd
 * (decoders/modeling_llama_mmfs.py:246-264): query i sees keys j <= i with key_mask[b, j] != 0 (key_mask (B, T) uint8
 * or NULL); Tq = Tkv = T, no KV cache.  q, k, v, out, d_out, dq, dk, dv are (B, T, H, 128) views with batch / token
 * strides in elements and dense heads (e.g. q / k / v and dq / dk / dv as slices of (B, T, 3, H, 128) buffers); lse
 * (B, H, T) fp32 from mmfs_attn_forward_lse on the same q, k, v, mask and scale; delta: B*H*T floats of device scratch
 * private to the call (it receives rowsum(d_out * out) in fp32).  dq, dk, dv are fully overwritten.
 * Three launches (delta; dK and dV per key tile; dQ per query tile) on mma.sync tensor-core MMAs, each output element
 * accumulated by one thread in a fixed order: no atomics, two runs give bit-identical gradients.
 * Requires hd = 128, bf16 / f16, 16-byte aligned pointers and strides of q, k, v, d_out, dq, dk, dv, B, H <= 65535:
 * MMFS_EUNSUPPORTED otherwise.
 */
int mmfs_attn_backward(const void *q, const void *k, const void *v, const void *out, const void *d_out, const float *lse,
                       void *dq, void *dk, void *dv, float *delta, const uint8_t *key_mask, int B, int H, int T, int hd,
                       long q_bs, long q_ts, long k_bs, long k_ts, long v_bs, long v_ts, long o_bs, long o_ts,
                       long do_bs, long do_ts, long dq_bs, long dq_ts, long dk_bs, long dk_ts, long dv_bs, long dv_ts,
                       float scale, int dtype, void *stream);

/*
 * mmfs_attn_backward for any head dim the forward takes, with or without causality, and with queries and keys of
 * different lengths (the Q-Former's self-attention over its queries and cross-attention to the image tokens): query i
 * sees keys j < Tkv with key_mask[b, j] != 0 (key_mask (B, Tkv) uint8 or NULL) and, when `causal`, j <= i.  q, out,
 * d_out, dq are (B, Tq, H, hd) views and k, v, dk, dv (B, Tkv, H, hd) views, each with its own batch / token strides in
 * elements and dense heads; lse (B, H, Tq) fp32 from mmfs_attn_forward_lse on the same q, k, v, mask, scale and
 * causality; delta: B*H*Tq floats of device scratch private to the call.  dq, dk, dv are fully overwritten (a key no
 * query sees gets zero dk / dv).  Same kernels, launches and determinism as mmfs_attn_backward, which is this call with
 * hd = 128, causal = 1 and Tq = Tkv.
 * Negative B, H <= 0, Tq <= 0, Tkv <= 0, hd <= 0, causal with Tq != Tkv, null pointers: MMFS_EINVAL.  hd not in
 * {64, 128}, a dtype other than bf16 / f16, pointers or strides of q, k, v, d_out, dq, dk, dv not 16-byte aligned,
 * B or H > 65535: MMFS_EUNSUPPORTED.
 */
int mmfs_attn_backward_general(const void *q, const void *k, const void *v, const void *out, const void *d_out,
                               const float *lse, void *dq, void *dk, void *dv, float *delta, const uint8_t *key_mask,
                               int B, int H, int Tq, int Tkv, int hd, long q_bs, long q_ts, long k_bs, long k_ts, long v_bs,
                               long v_ts, long o_bs, long o_ts, long do_bs, long do_ts, long dq_bs, long dq_ts, long dk_bs,
                               long dk_ts, long dv_bs, long dv_ts, float scale, int causal, int dtype, void *stream);

/*
 * Gradient of mmfs_layernorm (training path): dx (rows, cols) from x, weight and dy, with the row mean and biased
 * variance recomputed from x in fp32 (the forward rounds only its output).  With dweight and / or dbias != NULL also
 * dweight (cols) = sum over rows of dy * (x - mean) * rsqrt(var + eps) and dbias (cols) = sum over rows of dy, from
 * per-CTA fp32 partials in `partials` (2 * min(rows, MMFS_RMSNORM_BWD_PARTS) * cols floats of device scratch private to
 * the call) summed in a fixed order: run-to-run reproducible.  partials may be NULL when dweight and dbias are.  bf16 /
 * f16, cols % 8 == 0, cols <= 8192, 16-byte aligned rows: MMFS_EUNSUPPORTED otherwise.
 */
int mmfs_layernorm_backward(const void *x, const void *weight, const void *dy, void *dx, void *dweight, void *dbias,
                            float *partials, long rows, int cols, float eps, int dtype, void *stream);

/*
 * Gradient of mmfs_rmsnorm (training path): dx (rows, cols) from x, weight and dy, fp32 math; the forward's rounding
 * of x * rsqrt(mean(x^2) + eps) to the element type is treated as the identity.  With dweight != NULL also
 * dweight (cols) = sum over rows of dy * cast(x * rsqrt(.)), from per-CTA fp32 partials in `partials`
 * (min(rows, MMFS_RMSNORM_BWD_PARTS) * cols floats of device scratch private to the call) summed in a fixed order:
 * run-to-run reproducible.  partials may be NULL when dweight is.  bf16 / f16, cols % 8 == 0, cols <= 8192, 16-byte
 * aligned rows: MMFS_EUNSUPPORTED otherwise.
 */
#define MMFS_RMSNORM_BWD_PARTS 256
int mmfs_rmsnorm_backward(const void *x, const void *weight, const void *dy, void *dx, void *dweight, float *partials,
                          long rows, int cols, float eps, int dtype, void *stream);

/*
 * Gradient of mmfs_swiglu (training path): d_gate_up (rows, 2*inter) = [d gate | d up] of out = silu(gate) * up from
 * gate_up (rows, 2*inter) and d_out (rows, inter), in fp32.  bf16 / f16, inter % 8 == 0, 16-byte aligned rows:
 * MMFS_EUNSUPPORTED otherwise.  (The backward of mmfs_rope_qk is mmfs_rope_qk itself with the sin table negated: the
 * transpose of a rotation by theta is the rotation by -theta.)
 */
int mmfs_swiglu_backward(const void *gate_up, const void *d_out, void *d_gate_up, long rows, int inter, int dtype,
                         void *stream);

/*
 * Gradient of mmfs_geglu (training path, diffusers' GEGLU with the exact erf GELU): d_value_gate (rows, 2*inter) =
 * [d value | d gate] of out = value * gelu(gate) from value_gate (rows, 2*inter) and d_out (rows, inter):
 * d value = d_out * gelu(gate), d gate = d_out * value * (Phi(gate) + gate * phi(gate)), in fp32 with one rounding at the
 * store.  16-byte vectors when inter % 8 == 0 and the pointers are 16-byte aligned, one element per step otherwise.
 * rows < 0, inter <= 0, null pointers: MMFS_EINVAL.  A dtype other than bf16 / f16: MMFS_EUNSUPPORTED.
 */
int mmfs_geglu_backward(const void *value_gate, const void *d_out, void *d_value_gate, long rows, int inter, int dtype,
                        void *stream);

/*
 * Gradient of CLIP's quick_gelu, y = h * sigmoid(1.702 h) (training path): dh = dy * (s + 1.702 h s (1 - s)) with
 * s = sigmoid(1.702 h), over n elements of h, dy and dh, in fp32 with one rounding at the store.  16-byte vectors and a
 * scalar tail, so any n >= 0.  n < 0, null pointers: MMFS_EINVAL.  A dtype other than bf16 / f16, pointers not 16-byte
 * aligned: MMFS_EUNSUPPORTED.
 */
int mmfs_quick_gelu_backward(const void *h, const void *dy, void *dh, long n, int dtype, void *stream);

/*
 * Gradient of a bilinear resize with align_corners=False and a given scale factor (F.interpolate(x, scale_factor=f,
 * mode="bilinear"), the ViT-Adapter's x4 / x2 / x0.5 output resizes), training path.  scale_h, scale_w = 1 / f per axis:
 * output index o samples input r = max(scale * (o + 0.5) - 0.5, 0) along that axis, PyTorch's source-index rule with its
 * edge clamps.  Gather form without atomics: every input pixel sums, in fp32 and in a fixed order (output rows, then
 * columns, increasing), the weighted dy of the output pixels that sample it, and is rounded once: run-to-run
 * reproducible.
 *   dy (B, C, Hout, Wout): element (b, c, p), p = oy * Wout + ox, at dy[b * dy_bs + c * dy_cs + p * dy_ps] (NCHW: (C*Hout*Wout,
 *   Hout*Wout, 1); token layout (B, Hout*Wout, C): (Hout*Wout*C, 1, C)); dx (B, Hin * Win, C) contiguous, fully overwritten
 *   (token layout: the transpose back to (B, C, Hin, Win) is the caller's view).
 * Negative B, non-positive C / sizes / scales, null pointers: MMFS_EINVAL.  A dtype other than bf16 / f16, C % 8 != 0, dx
 * not 16-byte aligned: MMFS_EUNSUPPORTED.
 */
int mmfs_resize_bilinear_backward(const void *dy, void *dx, int B, int C, int Hin, int Win, int Hout, int Wout, long dy_bs,
                                  long dy_cs, long dy_ps, float scale_h, float scale_w, int dtype, void *stream);

/*
 * 2-D convolution as an implicit GEMM on the tensor cores (wgmma, TMA-shifted input boxes, no im2col buffer).
 * Replaces the cuDNN convolutions diffusers' UNet issues in the denoise step (called from
 * utils/monkey_patch/sd_unet_forward_monkey_patch.py:235-366; 3x3 stride 1/2 and 1x1, NHWC).
 *   x (B,H,W,Cin) NHWC; w (Cout,KH,KW,Cin); out (B,Ho,Wo,Cout) NHWC; optional fused epilogue terms: bias (Cout),
 *   add_bc (B,Cout) [the ResNet block's time-embedding projection], residual (like out).
 * Requires bf16/f16, Cin % 64 == 0, Cout % 160 == 0 or Cout % 128 == 0, stride <= 2, output tileable by 8x16 (or 8x8
 * with even B) pixel patches: MMFS_EUNSUPPORTED otherwise (callers keep those few layers -- conv_in / conv_out -- on the
 * library path).
 */
int mmfs_conv2d_nhwc(const void *x, const void *w, const void *bias, const void *add_bc, const void *residual, void *out,
                     int B, int H, int W, int Cin, int Cout, int KH, int KW, int stride, int pad, int dtype, void *stream);

/*
 * Nearest 2x upsample followed by a 3x3 / pad-1 convolution (diffusers' Upsample2D with use_conv), without the
 * upsampled intermediate: each of the four output parities is a 2x2 convolution over the low-resolution input.
 *   x (B,H,W,Cin) NHWC; w_phases (4,Cout,2,2,Cin): the 3x3 filter folded per parity p = 2*py + px (rows: py = 0 ->
 *   {w0, w1+w2}, py = 1 -> {w0+w1, w2}; columns alike); bias (Cout) or NULL; out (B,2H,2W,Cout) NHWC.
 * Same requirements as mmfs_conv2d_nhwc on (Cin, Cout, dtype, alignment), with the H x W grid tileable.
 */
int mmfs_conv2d_up2x_nhwc(const void *x, const void *w_phases, const void *bias, void *out, int B, int H, int W, int Cin,
                          int Cout, int dtype, void *stream);

/*
 * 3x3 / stride-2 convolution after a one-sided zero pad of one row at the bottom and one column at the right (diffusers'
 * Downsample2D with padding=0, the VAE encoder's downsampler): conv3x3(F.pad(x, (0, 1, 0, 1)), stride 2).
 *   x (B,H,W,Cin) NHWC with H and W even; w (Cout,3,3,Cin); bias (Cout) or NULL; out (B,H/2,W/2,Cout) NHWC.
 * Null pointers, non-positive or odd H / W: MMFS_EINVAL.  Same requirements as mmfs_conv2d_nhwc on (Cin, Cout, dtype,
 * alignment), with the H/2 x W/2 output tileable.
 */
int mmfs_conv2d_down2x_nhwc(const void *x, const void *w, const void *bias, void *out, int B, int H, int W, int Cin,
                            int Cout, int dtype, void *stream);

/*
 * GroupNorm (+ SiLU when silu != 0) on NHWC activations: the nn.GroupNorm(32) in front of every UNet convolution
 * (same call sites as mmfs_conv2d_nhwc).  x, y (B, HW, C) NHWC; gamma/beta (C) or NULL; stats = caller-provided
 * scratch of 128*B*G floats (per-chunk partial sums; reduced in a fixed order, so results are run-to-run reproducible).  f32 / f16 / bf16; C % (16/sizeof) == 0 and C*sizeof <= 16 KiB.
 */
int mmfs_groupnorm_nhwc(const void *x, const void *gamma, const void *beta, void *y, float *stats, int B, int HW, int C,
                        int G, float eps, int silu, int dtype, void *stream);

/*
 * Gradient dx of mmfs_groupnorm_nhwc (training path, affine parameters frozen: no dgamma / dbeta).  With z = gamma xhat
 * + beta: dz = dy, or with silu != 0 dz = dy s (1 + z (1 - s)), s = sigmoid(z) at z rounded to the element type as the
 * forward rounds it; g = dz gamma; dx = r (g - mean(g) - xhat mean(g xhat)) per (image, group), r = 1 / sqrt(var + eps).
 * The statistics are recomputed from x exactly as the forward computes them.  Three kernels; every sum is reduced in a
 * fixed order without atomics, so dx is run-to-run reproducible.
 *   x, dy, dx (B, HW, C) NHWC; gamma / beta (C) or NULL; scratch = 256*B*G floats of device memory private to the call.
 * Null x / dy / dx / scratch, non-positive sizes, C % G != 0, B > 65535: MMFS_EINVAL.  f64 or an unknown dtype,
 * C % (16/sizeof) != 0, C*sizeof > 8 KiB, tensors not 16-byte aligned: MMFS_EUNSUPPORTED.
 */
int mmfs_groupnorm_nhwc_backward(const void *x, const void *gamma, const void *beta, const void *dy, void *dx,
                                 float *scratch, int B, int HW, int C, int G, float eps, int silu, int dtype, void *stream);

/* modes of mmfs_decode_select */
#define MMFS_SELECT_GREEDY 0
#define MMFS_SELECT_SAMPLE 1

/*
 * One decode step's token choice for B rows of fp32 logits (B, V), row stride ld >= V, V <= 131072; one CTA per row.
 * Replaces, in HF's order (transformers 4.31, generation/logits_process.py): RepetitionPenaltyLogitsProcessor (every
 * distinct id of out_ids[b, :step] gets s * p if s < 0 else s / p; skipped when p == 1), MinLengthLogitsProcessor
 * (every eos id -inf while step < min_length), then either the arg-max (MMFS_SELECT_GREEDY; first index wins ties, like
 * torch.argmax) or TemperatureLogitsWarper + TopPLogitsWarper + the multinomial draw (MMFS_SELECT_SAMPLE): tokens whose
 * ascending cumulative softmax mass is <= 1 - top_p are dropped, the most likely token is always kept, and tokens tied
 * exactly at the threshold are all kept (HF's sort keeps an arbitrary subset of them); the id is drawn by inverse CDF
 * over the kept set in vocabulary order with u = uniforms[b] when uniforms != NULL, else from Philox4x32-10 keyed by
 * (*seed, b, step).  Then the bookkeeping of the eager loop: a row with finished[b] set emits pad_id, finished[b] |=
 * (id in eos_ids), and the id is written to out_ids[b, step] and next_ids[b].
 *   out_ids (B, max_new) int64; step: DEVICE int64 (nothing is written unless 0 <= step < max_new); finished (B) uint8;
 *   next_ids (B) int64; eos_ids (n_eos) int64 device, NULL iff n_eos == 0; params: DEVICE fp32 {repetition_penalty,
 *   temperature, top_p}; seed: DEVICE int64, may be NULL in greedy mode or with uniforms; uniforms (B) fp32 or NULL.
 * The per-call values (step, params, seed) are read on the device, so one captured CUDA graph serves any of them.
 * Sampling sums the softmax mass in 2^-40 fixed point with integer atomics: the choice is run-to-run reproducible.
 */
int mmfs_decode_select(const float *logits, long ld, int64_t *out_ids, const int64_t *step, uint8_t *finished,
                       int64_t *next_ids, const int64_t *eos_ids, int n_eos, long pad_id, int min_length,
                       const float *params, const int64_t *seed, const float *uniforms, int B, int V, int max_new,
                       int mode, void *stream);

/*
 * One step of beam search for B sequences of num_beams rows each (R = B * num_beams rows of fp32 logits, row stride
 * ld >= V, V <= 131072): the scoring and BeamSearchScorer.process of HF beam_search (transformers 4.31,
 * early_stopping=False), in two launches (rows, then sequences).  Per row: log_softmax, RepetitionPenaltyLogitsProcessor
 * on the log-probs of every distinct id of history[r, :step] (s * p if s < 0 else s * (1/p), the fp32 reciprocal, as
 * mmfs_decode_select), MinLengthLogitsProcessor (eos ids -inf while step < min_length), + beam_scores[r], and the row's
 * top K with K = max(2, 1 + n_eos) * num_beams.  Per sequence: the top K of its rows' union, ordered by higher score
 * first and, on exactly equal scores, by the lower flat index row_in_group * V + token (torch.topk leaves that order
 * unspecified); then, in rank order, an eos candidate of rank < num_beams becomes a hypothesis scored
 * sum_logprobs / max(step, 1) ** length_penalty (double), an eos candidate of rank >= num_beams is skipped, non-eos
 * candidates fill the num_beams next beams (slots left over get pad_id, score 0, parent b * num_beams).  A sequence is
 * done once it holds num_beams hypotheses whose worst is >= best candidate / (step + 1) ** length_penalty.  A sequence
 * already done emits pad_id, score 0 and parent b * num_beams and changes no hypothesis.  Writes beam_scores, next_ids
 * and parent (absolute row index) per row, reorders history by parent and appends the new token at column step.
 *   params: DEVICE double {repetition_penalty, length_penalty}; step: DEVICE int64 (nothing is done unless
 *   0 <= step < max_new); history (R, max_new) int64; beam_scores (R) fp32; next_ids, parent (R) int64; done (B) uint8;
 *   hypotheses, num_beams slots per sequence: hyp_scores (B, num_beams) double, hyp_ids (B, num_beams, max_new) int64,
 *   hyp_meta (B, num_beams, 2) int64 {length, insertion serial}, length -1 = free slot.  A full set replaces its first
 *   (lowest serial) lowest-scored hypothesis, so sorting by serial gives the eager loop's list order.
 *   eos_ids (n_eos) int64 device, NULL iff n_eos == 0; scratch: R * K uint64 of device memory private to the call.
 * Limits: num_beams <= 8, n_eos <= 4, K <= V; outside them MMFS_EINVAL.  The per-call values (step, params) are read
 * on the device, so one captured CUDA graph serves any of them.
 */
int mmfs_beam_select(const float *logits, long ld, const int64_t *step, const double *params, float *beam_scores,
                     int64_t *history, int64_t *next_ids, int64_t *parent, uint8_t *done, double *hyp_scores,
                     int64_t *hyp_ids, int64_t *hyp_meta, const int64_t *eos_ids, int n_eos, long pad_id, int min_length,
                     uint64_t *scratch, int B, int num_beams, int V, int max_new, void *stream);

/*
 * One step of beam-sample decoding (HF GenerationMixin.beam_sample, transformers 4.31), two launches like
 * mmfs_beam_select, with the same buffers and the same scorer; only the candidates differ.  Per row r the score s of
 * token i is mmfs_beam_select's (log_softmax, repetition penalty, min-length ban, + beam_scores[r]), then the warpers:
 * s / temperature (times the fp32 reciprocal), top-k with k = min(max(top_k, 2), V) (top_k == 0: none; every s below
 * the k-th largest removed, ties at it kept), and top-p over the remaining tokens with mmfs_decode_select's rule (2^-40
 * fixed-point masses, ties at the threshold kept), never removing the two largest (min_tokens_to_keep = 2; skipped when
 * top_p >= 1).  The draw: per sequence, the 2 * num_beams largest keys s - log(-log u) over its kept tokens, an exact
 * draw without replacement proportional to softmax(s) (torch.multinomial's law), u from Philox4x32-10 keyed by
 * (*seed, step, r, i) or u = uniforms[r * V + i] when uniforms != NULL (values in (0, 1)).  The drawn candidates are
 * ordered by s, higher first, then by the lower flat index row_in_group * V + token, and BeamSearchScorer.process runs
 * on them as in mmfs_beam_select; the new beam scores are their (warped) s.  A sequence left with fewer than num_beams
 * non-eos candidates sets *error = 1 (sticky; 4.31 raises ValueError) and fills the missing beams with pad_id.
 *   params: DEVICE double {repetition_penalty, length_penalty, temperature, top_p}; seed: DEVICE int64, may be NULL
 *   with uniforms; uniforms (R, V) fp32 or NULL; error: DEVICE int32; scratch: R * 4 * num_beams uint64 of device
 *   memory private to the call; every other argument as mmfs_beam_select.
 * Limits: num_beams <= 8, n_eos <= 4, 2 * num_beams <= V <= 131072, top_k >= 0; outside them MMFS_EINVAL.  The
 * per-call values (step, params, seed) are read on the device, so one captured CUDA graph serves any of them.
 */
int mmfs_beam_sample(const float *logits, long ld, const int64_t *step, const double *params, const int64_t *seed,
                     const float *uniforms, float *beam_scores, int64_t *history, int64_t *next_ids, int64_t *parent,
                     uint8_t *done, double *hyp_scores, int64_t *hyp_ids, int64_t *hyp_meta, int32_t *error,
                     const int64_t *eos_ids, int n_eos, long pad_id, int min_length, int top_k, uint64_t *scratch, int B,
                     int num_beams, int V, int max_new, void *stream);

/*
 * The KV-cache reorder of beam search, in place and over the generated positions only: for each of n_caches cache
 * tensors (base pointer cache + i * cache_stride bytes) and each group of num_beams rows, row j gets the contents of
 * row parent[j] (an absolute row index in the same group) at positions [*cur - *step, *cur); the prompt positions are
 * identical across the beams of a sequence and are left alone.  Groups with done[g] set are skipped (done may be NULL).
 * Row r, position p of cache i starts at cache + i * cache_stride + r * row_stride + p * pos_stride and holds row_bytes
 * bytes.  cur, step: DEVICE int64; *step <= max_positions (the grid covers max_positions positions).  The pointer,
 * strides and row_bytes must be multiples of 16 bytes; num_beams <= 8 and rows % num_beams == 0, else MMFS_EINVAL.
 */
int mmfs_kv_beam_reorder(void *cache, int n_caches, long cache_stride, int rows, long row_stride, long pos_stride,
                         long row_bytes, int num_beams, const int64_t *parent, const int64_t *cur, const int64_t *step,
                         const uint8_t *done, int max_positions, void *stream);

/*
 * A generated image re-entering the context: (N, 3, S, S) fp32 images in [0, 1] (contiguous) to the visual tokenizer's
 * (N, 3, R, R) fp32 input (contiguous), bit-identical to the host path tensor_to_pil -> center_crop_arr(R) -> float32
 * / 255 of the reference's inference loop: the uint8 quantisation x * 255 + 0.5 (fp32, clamped to [0, 255],
 * truncated), PIL's BOX halvings while the size is >= 2R, PIL's BICUBIC resize to R with its antialiasing support and
 * 8-bit fixed-point passes (horizontal then vertical, each rounded and clipped), the (empty) centre crop, then u / 255
 * in fp32.  One launch; two runs are bit-identical.  A NaN pixel quantises to 0.
 * N < 0, non-positive C / H / W / R, N > 65535, null pointers with N > 0: MMFS_EINVAL.  C != 3, H != W, S or R above
 * 16384, or a resize whose rows do not fit in shared memory: MMFS_EUNSUPPORTED.
 */
int mmfs_image_reentry(const float *images, float *out, int N, int C, int H, int W, int R, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MMFS_B200_H_ */
