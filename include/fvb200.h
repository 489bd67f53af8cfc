/* fvb200.h -- C ABI of libfvb200.so, the H100 (sm_90a) implementation of FastVideo's Wan DiT
 * denoising hot path and Wan VAE decode.
 *
 * Every entry point takes plain device pointers, sizes, element strides and a cudaStream_t (passed as
 * void*); the caller allocates all outputs; calls are stream-ordered and never synchronise. The return
 * value is FVB_OK or an FVB_ERR_* code; fvb_last_error() returns a thread-local description.
 *
 * The reference (hao-ai-lab/FastVideo) has no C ABI: its natives are reached through pybind11
 * (fastvideo-kernel/csrc/common_extension.cpp:42-69) and torch.library custom ops
 * (fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:103-217). Each function below cites
 * the reference interface it stands behind; fastvideo_b200/ (Python) mirrors those interfaces on top
 * of this library and INTEGRATION.md shows the binding a FastVideo maintainer would add.
 *
 * All activations are bf16 unless stated; "row-major [R, C] with ld" means element (r, c) lives at
 * base + r*ld + c (ld in elements).
 */
#ifndef FVB200_H
#define FVB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FVB_OK 0
#define FVB_ERR_INVALID_ARG 1
#define FVB_ERR_CUDA 2
#define FVB_ERR_NO_DEVICE 3
#define FVB_ERR_UNSUPPORTED 4

#define FVB_ABI_VERSION 2

int fvb_abi_version(void);
const char* fvb_last_error(void);

/* --------------------------------------------------------------------------------------------
 * Linear layers (wgmma GEMM, TMA-fed, fused epilogues)
 * Replaces: ReplicatedLinear.forward -> UnquantizedLinearMethod.apply -> F.linear
 *   (fastvideo/layers/linear.py:146-156, 293-300) plus the op that follows it in
 *   WanTransformerBlock.forward (fastvideo/models/dits/wanvideo.py:394-431):
 *   GELU(tanh) of MLP (fastvideo/layers/mlp.py:47-51), the gated residuals of
 *   ScaleResidual / ScaleResidualLayerNormScaleShift (fastvideo/layers/layernorm.py:91-109,159-188).
 *
 *   acc[m, n] = sum_k x[m, k] * w[n, k]        (fp32 accumulation on the tensor cores)
 *   y = bf16(acc + bias[n])                    (bias may be NULL)
 * epilogue:
 *   FVB_EPI_BIAS            out_bf16 = y
 *   FVB_EPI_BIAS_GELU_TANH  out_bf16 = bf16(gelu_tanh(float(y)))
 *   FVB_EPI_RESID_GATE_F32  out_f32  = float(resid) + float(y) * gate[n]      (fp32 mul, then fp32 add)
 *   FVB_EPI_RESID_GATE_BF16 out_bf16 = bf16(float(resid) + float(y) * gate[n])
 *   FVB_EPI_RESID_BF16      out_bf16 = bf16(float(resid) + float(y))
 * x: [M, K] ld=ldx, w: [N, K] ld=ldw, bias: [N] bf16, resid: [M, N] bf16 ld=ldr, out: [M, N] ld=ldo.
 * gate: fp32 [N] when gate_rows == 0; otherwise rows [i*gate_rows, (i+1)*gate_rows) use gate + i*gate_stride
 * (per-latent-frame gates of the causal blocks, fastvideo/layers/layernorm.py:99-109, 159-188 with a 4-D gate). ldx, ldw, ldo, ldr multiples of 8 (16-byte rows); N a multiple of 8 when bias / residual are used.
 * -------------------------------------------------------------------------------------------- */
#define FVB_EPI_BIAS 0
#define FVB_EPI_BIAS_GELU_TANH 1
#define FVB_EPI_RESID_GATE_F32 2
#define FVB_EPI_RESID_GATE_BF16 3
#define FVB_EPI_RESID_BF16 4
#define FVB_EPI_DIV 5       /* internal to fvb_gemm_batched_bf16 */
#define FVB_EPI_RESID_GATE_BF16R 7 /* out_bf16 = bf16(float(resid) + bf16(float(y) * gate[n])): bf16 gate tensors */
#define FVB_EPI_SCALE_F32 6 /* internal to fvb_gemm_f32out */

int fvb_linear_bf16(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias, void* out,
                    int64_t ldo, const void* resid, int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride,
                    int M, int N, int K, int epilogue, void* stream);

/* fvb_linear_bf16 for sequence-parallel buffers, so the Ulysses all-to-all needs no pack/unpack copies
 * (the transpose().contiguous() pairs of fastvideo/distributed/device_communicators/base_device_communicator.py:147-179):
 *   out_col_offsets (optional, int64 [N/128]): output column block j (a head) is written at
 *       out + out_col_offsets[j] + row*ldo + (col % 128)  -- e.g. straight into the all-to-all send buffer
 *       [dest rank][token][q|k|v|g][local head][d].
 *   x_seg_len / x_seg_stride: x's K axis is cut in segments of x_seg_len elements (multiple of 64) that live
 *       x_seg_stride elements apart -- e.g. the all-to-all receive buffer [src rank][token][local head][d] read as
 *       [token, all heads * d]. x_seg_len = 0: plain row-major x. */
int fvb_linear_bf16_sp(const void* x, int64_t ldx, int x_seg_len, int64_t x_seg_stride, const void* w, int64_t ldw,
                       const void* bias, void* out, int64_t ldo, const int64_t* out_col_offsets, const void* resid,
                       int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride, int M, int N, int K,
                       int epilogue, void* stream);

/* --------------------------------------------------------------------------------------------
 * Backward of the bf16 linear y = bf16(x w^T + b) (FVB_EPI_BIAS), for training. M, N, K keep the forward's meaning:
 * x [M, K], w [N, K], dy [M, N], all bf16 with unit inner stride and row strides (ldx, ldw, lddy, lddx, lddw; multiples of
 * 8) so column slices of fused buffers work in place. Each output is fp32-accumulated and rounded to bf16 once -- torch's
 * rounding points for bf16 F.linear autograd. No split-K and no atomics: two calls give the same bits.
 *
 * fvb_linear_dgrad_bf16:  dx[m, k] = bf16(sum_n dy[m, n] * w[n, k])      K a multiple of 8 (dx's columns)
 * fvb_linear_wgrad_bf16:  dw[n, k] = bf16(sum_m dy[m, n] * x[m, k])      K a multiple of 8 (dw's columns)
 *   Both run the forward's wgmma GEMM with MN-major (transposed) shared-memory operands; reduction tails (N for dgrad, M
 *   for wgrad) are zero-filled on load. Only [0, M) x [0, K) of dx and [0, N) x [0, K) of dw are written.
 * fvb_bias_grad_bf16:     db[n] = bf16(sum_m float(dy[m, n]))             N a multiple of 8
 *   Deterministic: each of min(M, 256) row sets (rows p, p + 256, ...) is summed in row order into an fp32 partial per
 *   column, then the partials are added in row-set order and rounded once. workspace: device memory of
 *   fvb_bias_grad_bf16_workspace_bytes(M, N) bytes, 16-byte aligned.
 * -------------------------------------------------------------------------------------------- */
int fvb_linear_dgrad_bf16(const void* dy, int64_t lddy, const void* w, int64_t ldw, void* dx, int64_t lddx, int M, int N, int K,
                          void* stream);
int fvb_linear_wgrad_bf16(const void* dy, int64_t lddy, const void* x, int64_t ldx, void* dw, int64_t lddw, int M, int N, int K,
                          void* stream);
int64_t fvb_bias_grad_bf16_workspace_bytes(int M, int N);
int fvb_bias_grad_bf16(const void* dy, int64_t lddy, void* db, float* workspace, int64_t workspace_bytes, int M, int N,
                       void* stream);

/* Pieces of the Wan block backward that live in GEMM epilogues (bf16 operands, the arguments of fvb_linear_bf16):
 * fvb_linear_bf16_aux: fvb_linear_bf16 that also stores the bf16 y = bf16(acc + bias) its epilogue consumes to
 *   aux[m * ldaux + n] (ldaux a multiple of 8, >= N; N a multiple of 8). Epilogues FVB_EPI_BIAS_GELU_TANH (aux = the fc_in
 *   output before the GELU), FVB_EPI_RESID_GATE_F32, FVB_EPI_RESID_GATE_BF16 and FVB_EPI_RESID_GATE_BF16R (with its gate_rows
 *   grouping; aux = the projection before the gate multiply). `out` gets the same bits as fvb_linear_bf16, and aux the same
 *   bits as fvb_linear_bf16 with FVB_EPI_BIAS.
 * fvb_linear_dgrad_gelu_bf16: fvb_linear_dgrad_bf16 with the GELU(tanh) backward in its epilogue, for y = w2 . gelu(h):
 *   dh[m, k] = bf16(float(bf16(sum_n dy[m, n] * w[n, k])) * gelu_tanh'(h[m, k]))     h bf16 [M, K] (ldh a multiple of 8)
 *   gelu_tanh'(h) = 0.5 (1 + t) + 0.5 h (1 - t^2) sqrt(2/pi) (1 + 3 * 0.044715 h^2), t = tanh(sqrt(2/pi) (h + 0.044715 h^3)),
 *   t evaluated as FVB_EPI_BIAS_GELU_TANH evaluates it. Torch's rounding: bf16 F.linear dgrad, then bf16 gelu_backward. */
int fvb_linear_bf16_aux(const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias, void* out, int64_t ldo,
                        const void* resid, int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride, void* aux,
                        int64_t ldaux, int M, int N, int K, int epilogue, void* stream);
int fvb_linear_dgrad_gelu_bf16(const void* dy, int64_t lddy, const void* w, int64_t ldw, const void* h, int64_t ldh, void* dh,
                               int64_t lddh, int M, int N, int K, void* stream);

/* Backward of the gated residual out = resid + y * gate[n] (FVB_EPI_RESID_GATE_F32 / _BF16) given dout [M, N] (fp32 when
 * dout_is_f32, else bf16) and the saved bf16 y [M, N] (fvb_linear_bf16_aux's aux); gate fp32 [N]:
 *   dy[m, n] = bf16(dout * gate[n])                 bf16 [M, N] (lddy)
 *   d_gate[n] = sum_m dout * y                      fp32 [N]
 *   db[n] = bf16(sum_m float(dy[m, n]))             bf16 [N], the projection's bias gradient (db NULL: skipped)
 * The residual's gradient is dout itself (nothing is written for it). N a multiple of 8; strides keep rows 16-byte aligned.
 * Column sums as in fvb_bias_grad_bf16: min(M, 256) fixed row sets summed in row order, partials added in row-set order;
 * no atomics. workspace: fvb_resid_gate_bwd_workspace_bytes(M, N) bytes, 16-byte aligned. */
int64_t fvb_resid_gate_bwd_workspace_bytes(int M, int N);
int fvb_resid_gate_bwd(const void* dout, int dout_is_f32, int64_t lddout, const void* y, int64_t ldy, const float* gate, void* dy,
                       int64_t lddy, float* d_gate, void* db, float* workspace, int64_t workspace_bytes, int M, int N,
                       void* stream);

/* --------------------------------------------------------------------------------------------
 * FP8 (e4m3) linear layers: row-quantised activations x per-output-channel-quantised weights
 * Stands behind FastVideo's FP8 linear (fastvideo/layers/fp8linear.py, fastvideo/layers/quantization/) with this
 * library's own arithmetic, below.
 *
 * fvb_quantize_fp8_rows: x bf16 [M, K] (row stride ldx, a multiple of 8: 16-byte rows; K a multiple of 8)
 *   -> q e4m3 [M, K] (one byte per element, row stride ldq, a multiple of 8) and scale fp32 [M]:
 *   amax = max_k |x[r, k]| (fp32, exact);
 *   amax == 0: scale[r] = 1, q[r, :] = 0;
 *   else inv = 448.0f / amax, q[r, k] = e4m3_satfinite_rn(x[r, k] * inv), scale[r] = amax / 448.0f
 *   (IEEE round-to-nearest division and multiplication; e4m3_satfinite_rn = __nv_cvt_float_to_fp8(v, __NV_SATFINITE,
 *   __NV_E4M3)). Used for activations (one scale per token) and for weights w[N, K] (one scale per output channel).
 *
 * fvb_linear_fp8: xq e4m3 [M, K] ld=ldx with x_scale fp32 [M]; wq e4m3 [N, K] ld=ldw with w_scale fp32 [N]:
 *   acc[m, n] = sum_k xq[m, k] * wq[n, k]                (fp32: partial sums leave the tensor core every 128 k)
 *   y = bf16(((acc * x_scale[m]) * w_scale[n]) + bias[n])  (fp32 round-to-nearest, in that order; bias may be NULL)
 *   then the epilogue exactly as in fvb_linear_bf16: FVB_EPI_BIAS, BIAS_GELU_TANH, RESID_GATE_F32, RESID_GATE_BF16,
 *   RESID_GATE_BF16R, RESID_BF16, with the same gate / gate_rows grouping.
 *   ldx, ldw multiples of 16 (16-byte rows); ldo, ldr multiples of 8; N a multiple of 8 when bias / residual are used.
 *   K tails (K not a multiple of 128) are zero-filled on load.
 * -------------------------------------------------------------------------------------------- */
int fvb_quantize_fp8_rows(const void* x, int64_t ldx, int M, int K, void* q, int64_t ldq, float* scale, void* stream);

int fvb_linear_fp8(const void* xq, int64_t ldx, const float* x_scale, const void* wq, int64_t ldw, const float* w_scale,
                   const void* bias, void* out, int64_t ldo, const void* resid, int64_t ldr, const float* gate, int gate_rows,
                   int64_t gate_stride, int M, int N, int K, int epilogue, void* stream);

/* --------------------------------------------------------------------------------------------
 * INT8 weight-only linear layers: bf16 activations x per-output-channel int8 weights
 *
 * fvb_linear_w8_sp: x bf16 [M, K] (ld=ldx, or segmented by x_seg_len / x_seg_stride as in fvb_linear_bf16_sp);
 *   wq int8 [N, K] ld=ldw (a multiple of 16: 16-byte rows) with w_scale fp32 [N]:
 *   acc[m, n] = sum_k x[m, k] * wq[n, k]   (every bf16 x int8 product is exact in fp32; int8 -> bf16 is exact, so the
 *                                           accumulation is the bf16 GEMM's)
 *   y = bf16((acc * w_scale[n]) + bias[n])  (fp32 round-to-nearest, in that order, no contraction; bias may be NULL)
 *   then the epilogue exactly as in fvb_linear_bf16: FVB_EPI_BIAS, BIAS_GELU_TANH, RESID_GATE_F32, RESID_GATE_BF16,
 *   RESID_GATE_BF16R, RESID_BF16, with the same gate / gate_rows grouping. out_col_offsets, x_seg_len, x_seg_stride and
 *   every other argument follow the rules of fvb_linear_bf16_sp; x_seg_len = 0 with out_col_offsets = NULL is the plain
 *   linear. K tails (K not a multiple of 64) are zero-filled on load.
 * The weights are typically quantised once at load: scale[n] = amax_n / 127, wq[n, k] = clamp(rint(w[n, k] * (127 /
 * amax_n)), -127, 127); an all-zero row has scale 1 and wq = 0.
 * -------------------------------------------------------------------------------------------- */
int fvb_linear_w8_sp(const void* x, int64_t ldx, int x_seg_len, int64_t x_seg_stride, const void* wq, int64_t ldw,
                     const float* w_scale, const void* bias, void* out, int64_t ldo, const int64_t* out_col_offsets,
                     const void* resid, int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride, int M, int N,
                     int K, int epilogue, void* stream);

/* --------------------------------------------------------------------------------------------
 * W8A8 INT8 linear layers: per-token int8 activations x per-output-channel int8 weights
 *
 * fvb_quantize_int8_rows: x bf16 [M, K] (row stride ldx, a multiple of 8; K a multiple of 8), optionally segmented: with
 *   0 < x_seg_len < K, element k of row r is x[r * ldx + (k / x_seg_len) * x_seg_stride + k % x_seg_len] (x_seg_len a
 *   multiple of 8 dividing K, x_seg_stride a multiple of 8; the meaning of fvb_linear_bf16_sp). x_seg_len = 0: plain rows.
 *   -> q int8 [M, K] (one contiguous row each, row stride ldq, a multiple of 8) and scale fp32 [M]:
 *   amax = max_k |x[r, k]| (fp32, exact, over every segment of the row);
 *   amax == 0: scale[r] = 1, q[r, :] = 0;
 *   else inv = 127.0f / amax, q[r, k] = clamp(rint(x[r, k] * inv), -127, 127), scale[r] = amax / 127.0f
 *   (IEEE round-to-nearest division and multiplication, rint half-to-even): the rule of the load-time weight quantiser.
 *
 * fvb_linear_w8a8_sp: xq int8 [M, K] ld=ldx with x_scale fp32 [M]; wq int8 [N, K] ld=ldw with w_scale fp32 [N]
 *   (ldx, ldw multiples of 16: 16-byte rows):
 *   acc[m, n] = sum_k xq[m, k] * wq[n, k]                          (s32, exact: K <= 133144 keeps 127^2 K below 2^31;
 *                                                                   larger K is rejected)
 *   y = bf16(((float(acc) * x_scale[m]) * w_scale[n]) + bias[n])   (float() and fp32 round-to-nearest, in that order, no
 *                                                                   contraction; bias may be NULL)
 *   then the epilogue exactly as in fvb_linear_bf16: FVB_EPI_BIAS, BIAS_GELU_TANH, RESID_GATE_F32, RESID_GATE_BF16,
 *   RESID_GATE_BF16R, RESID_BF16, with the same gate / gate_rows grouping. out_col_offsets follows fvb_linear_bf16_sp
 *   (N % 128 == 0); the A operand is never segmented (fvb_quantize_int8_rows gathers segmented rows). K tails (K not a
 *   multiple of 128) are zero-filled on load.
 * -------------------------------------------------------------------------------------------- */
int fvb_quantize_int8_rows(const void* x, int64_t ldx, int x_seg_len, int64_t x_seg_stride, int M, int K, void* q,
                           int64_t ldq, float* scale, void* stream);

int fvb_linear_w8a8_sp(const void* xq, int64_t ldx, const float* x_scale, const void* wq, int64_t ldw, const float* w_scale,
                       const void* bias, void* out, int64_t ldo, const int64_t* out_col_offsets, const void* resid,
                       int64_t ldr, const float* gate, int gate_rows, int64_t gate_stride, int M, int N, int K, int epilogue,
                       void* stream);

/* Batched C[i] = bf16(A[i] @ B[i]^T), optionally followed by out = bf16(float(C) / div) (div = 0 or 1: none).
 * A[i]: [M, K] ld=lda, B[i]: [N, K] ld=ldb, out[i]: [M, N] ld=ldo; batch strides in elements (multiples of 8).
 * Replaces the block-level matmuls of video_sparse_attn's compression branch
 * (fastvideo-kernel/python/fastvideo_kernel/ops.py:112-116): scores = q_c @ k_c^T / sqrt(d), out_c = attn @ v_c. */
int fvb_gemm_batched_bf16(const void* a, int64_t lda, int64_t a_batch_stride, const void* b, int64_t ldb,
                          int64_t b_batch_stride, void* out, int64_t ldo, int64_t out_batch_stride, int M, int N, int K,
                          int batch, float div, void* stream);

/* --------------------------------------------------------------------------------------------
 * Row kernels: fvb_layernorm_modulate, fvb_rmsnorm_rope, fvb_rmsnorm_rope_scatter and the backward entry points below
 * (fvb_rmsnorm_bwd, fvb_rmsnorm_rope_bwd, fvb_layernorm_modulate_bwd, the two grouped ones), plus fvb_bias_grad_bf16 and
 * fvb_resid_gate_bwd above. They access their rows, per-column vectors (w, b, scale, shift, gain, gate), cos / sin tables
 * and workspace with 128-bit vectors: every such pointer must be 16-byte aligned, else the call returns
 * FVB_ERR_INVALID_ARG. Outputs written one element at a time (dw, db, d_gate, d_gain, d_offset, d_scale, d_shift) and
 * index arrays (rope_row, col_offsets) need only their natural alignment.
 * -------------------------------------------------------------------------------------------- */

/* --------------------------------------------------------------------------------------------
 * LayerNorm + AdaLN modulation (one pass over the row, fp32 statistics)
 * Replaces: FP32LayerNorm / ScaleResidualLayerNormScaleShift / LayerNormScaleShift
 *   (fastvideo/layers/layernorm.py:115-125, 159-213, 216-273) as used at
 *   fastvideo/models/dits/wanvideo.py:393 (norm1), :419 (self_attn_residual_norm), :425
 *   (cross_attn_residual_norm) and :755 (norm_out).
 *   t   = (x - mean) * rsqrt(var + eps) [* w + b]         x: bf16, or fp32 when x_is_f32
 *   t   = bf16(t)                       if round_ln & 1    (LN output dtype == bf16 input dtype)
 *   t   = t * (1 + scale[c]) + shift[c] if scale != NULL   (fp32 mul, then fp32 add)
 *         or, if round_ln & 2 (bf16 scale/shift tensors, every op rounds -- CausalWanTransformerBlock with a bf16 `e`,
 *         fastvideo/models/dits/causal_wanvideo.py:288-296): t = bf16(bf16(t * bf16(1 + scale[c])) + shift[c])
 *   out = bf16(t);  hidden_out = bf16(x) if hidden_out != NULL (residual-stream cast, wanvideo.py:421)
 * w, b: fp32 [D]. scale, shift: fp32 [D] when mod_rows == 0; otherwise rows [i*mod_rows, (i+1)*mod_rows) use
 * scale + i*mod_stride, shift + i*mod_stride -- the per-latent-frame modulation of the causal blocks
 * (fastvideo/models/dits/causal_wanvideo.py:291-296, 326-336). D multiple of 8, <= 8192.
 * -------------------------------------------------------------------------------------------- */
int fvb_layernorm_modulate(const void* x, int x_is_f32, int64_t ldx, const float* w, const float* b,
                           const float* scale, const float* shift, int mod_rows, int64_t mod_stride, int round_ln,
                           void* out, int64_t ldo, void* hidden_out, int64_t ldh, int M, int D, float eps, void* stream);

/* --------------------------------------------------------------------------------------------
 * QK RMSNorm across heads + 3D RoPE, in place, q and k in one launch (x1 may be NULL)
 * Replaces: RMSNorm.forward_native (fastvideo/layers/layernorm.py:48-83; wanvideo.py:398-401) and
 *   _apply_rotary_emb, full-head-dim interleaved-pair branch (fastvideo/layers/rotary_embedding.py:124-135;
 *   call site fastvideo/attention/layer.py:130-132).
 *   n = bf16(bf16(x * rsqrt(mean(x^2) + eps)) * w);   o[2i] = bf16(n[2i]*cos[2i] - n[2i+1]*sin[2i]),
 *   o[2i+1] = bf16(n[2i+1]*cos[2i+1] + n[2i]*sin[2i+1]) per head.  cos/sin: fp32 [S_pos, head_dim]
 *   (get_rotary_pos_embed's table) or NULL (no RoPE: cross-attention); with rope_f64 != 0 the tables are float64 and
 *   the rotation is evaluated in float64 and rounded double -> float -> bf16, as happens in the causal model, which
 *   passes the float64 tables through unconverted (fastvideo/models/dits/causal_wanvideo.py:589-598). rope_row: int32 [M] token ->
 *   table row, or NULL for identity. w: bf16 [D]. `rope_f64` is a flag word: bit 0 = float64 tables (above), bit 1 = the
 *   weights are fp32 [D]: then n = bf16(x * rsqrt(...)) * w is an fp32 product that is NOT rounded before the rotation --
 *   what torch's type promotion does with an fp32 RMSNorm parameter (layernorm.py:73-79) -- and the result is rounded to
 *   bf16 once, at the store. col_offsets (optional, int64 [D/128]): element offset of each
 *   128-column block (= head) inside a row, for the head-scattered layout written by fvb_linear_bf16_sp.
 * -------------------------------------------------------------------------------------------- */
int fvb_rmsnorm_rope(void* x0, const void* w0, int64_t ld0, void* x1, const void* w1, int64_t ld1,
                     const void* cos_t, const void* sin_t, int rope_f64, const int32_t* rope_row,
                     const int64_t* col_offsets, int M, int D, int head_dim, float eps, void* stream);

/* Out-of-place variant for the sequence-parallel exchange: the normalised (and roped) heads of row r are written to
 * y + r*ldy + out_col_offsets[head block] instead of back into x. With out_col_offsets pointing into the peer GPUs'
 * receive buffers (CUDA peer / symmetric memory) this IS the "scatter heads" half of the Ulysses all-to-all
 * (fastvideo/distributed/device_communicators/base_device_communicator.py:123-193), fused into the row pass that has to
 * touch q and k anyway. w == NULL: no normalisation -- the row is copied unchanged (v and gate rows), or, when tables are
 * given, only roped (the window of un-roped keys of the "relativistic" KV-cache policy,
 * fastvideo/models/dits/causal_wanvideo.py:95-97, 140, 174-181). x rows are contiguous (ld strides). */
int fvb_rmsnorm_rope_scatter(const void* x0, const void* w0, int64_t ld0, const void* x1, const void* w1, int64_t ld1, void* y0,
                             void* y1, int64_t ldy, const int64_t* out_col_offsets, const void* cos_t, const void* sin_t,
                             int rope_f64, const int32_t* rope_row, int M, int D, int head_dim, float eps, void* stream);

/* Backward of fvb_rmsnorm_rope without RoPE, n = bf16(bf16(x * r) * w), for one tensor: x, dy, dx bf16 [M, D] rows (row
 * strides ldx / lddy / lddx, multiples of 8), w bf16 [D] or NULL (all ones), D a multiple of 8, <= 8192. Per row, fp32:
 *   r = rsqrt(sum_c x^2 / D + eps) (recomputed from x; the forward stores nothing extra), x^ = x * r,
 *   g = bf16(dy * w) (g = dy without w), s = sum_c g * x (fp32, the row reduced across the CTA),
 *   dx = bf16(r * (g - x^ * ((r * s) / D)))          -- (r * s) is sum_c g * x^
 *   dw[c] = bf16(sum_m float(dy[m, c]) * float(bf16(x^[m, c])))   (dw != NULL, needs w)
 * dw's sum is deterministic: each of min(M, 528) CTAs sums its rows (rows cta, cta + 528, ...) in row order into an fp32
 * partial per column, then the partials are added in CTA order and rounded once. No atomics. workspace: device memory of
 * fvb_rmsnorm_bwd_workspace_bytes(M, D) bytes (only used with dw), 16-byte aligned. */
int64_t fvb_rmsnorm_bwd_workspace_bytes(int M, int D);
int fvb_rmsnorm_bwd(const void* x, int64_t ldx, const void* w, const void* dy, int64_t lddy, void* dx, int64_t lddx, void* dw,
                    float* workspace, int64_t workspace_bytes, int M, int D, float eps, void* stream);

/* Backward of fvb_rmsnorm_rope with RoPE, for x0 (and x1: q and k in one launch, blockIdx.y selects), bf16 weights only;
 * cos / sin fp32 [S_pos, head_dim] and rope_row as in the forward. dy is the gradient of the rotated output. Per pair
 * (2i, 2i+1) of each row, fp32, the forward's rotation transposed:
 *   dn[2i]   = bf16(dy[2i] * cos[2i] + dy[2i+1] * sin[2i+1])
 *   dn[2i+1] = bf16(dy[2i+1] * cos[2i+1] - dy[2i] * sin[2i])
 * then fvb_rmsnorm_bwd's arithmetic with dn in place of dy (dx, and dw0 / dw1 with their own partials when dw0 != NULL).
 * workspace: fvb_rmsnorm_rope_bwd_workspace_bytes(M, D) bytes (two tensors' partials). */
int64_t fvb_rmsnorm_rope_bwd_workspace_bytes(int M, int D);
int fvb_rmsnorm_rope_bwd(const void* x0, int64_t ldx0, const void* w0, const void* dy0, int64_t lddy0, void* dx0, int64_t lddx0,
                         void* dw0, const void* x1, int64_t ldx1, const void* w1, const void* dy1, int64_t lddy1, void* dx1,
                         int64_t lddx1, void* dw1, const float* cos_t, const float* sin_t, const int32_t* rope_row,
                         float* workspace, int64_t workspace_bytes, int M, int D, int head_dim, float eps, void* stream);

/* Backward of fvb_layernorm_modulate's single-row-group forms: n = bf16(t * gain[c] + offset[c]), t = LN(x) =
 * (x - mean) * rstd (fp32, biased variance, recomputed from x), t rounded to bf16 first with round_ln. gain is (1 + scale)
 * with gain_is_scale (modulation: offset = shift) or the affine weight w (offset = the affine bias). x [M, D] bf16, or fp32
 * with x_is_f32; dn bf16 [M, D]; round_ln only with gain_is_scale. Per row, fp32:
 *   dt = dn * gain,  dx = rstd * ((dt - mean_c(dt)) - t~ * mean_c(dt * t~))  (t~ = the unrounded t)  [+ gin]
 *   dx: fp32 when x is fp32, else bf16 (one rounding after the optional incoming gradient gin, fp32 or bf16 per gin_is_f32,
 *   is added: the residual stream's two gradient contributions meet here)
 *   d_gain[c] = sum_m dn * t (t as used in the forward, bf16 with round_ln), d_offset[c] = sum_m dn    (fp32 [D])
 * Column sums as in fvb_rmsnorm_bwd (min(M, 528) CTAs, partials added in CTA order). D a multiple of 8, <= 8192; strides
 * multiples of 8. workspace: fvb_layernorm_modulate_bwd_workspace_bytes(M, D) bytes, 16-byte aligned. */
int64_t fvb_layernorm_modulate_bwd_workspace_bytes(int M, int D);
int fvb_layernorm_modulate_bwd(const void* x, int x_is_f32, int64_t ldx, const void* dn, int64_t lddn, const float* gain,
                               int gain_is_scale, int round_ln, const void* gin, int gin_is_f32, int64_t ldgin, void* dx,
                               int64_t lddx, float* d_gain, float* d_offset, float* workspace, int64_t workspace_bytes, int M,
                               int D, float eps, void* stream);

/* Per-row-group backward of the bf16 modulation flow of the causal Wan blocks (one modulation row per latent frame).
 * Group g is rows [g R, min((g + 1) R, M)), R = mod_rows / gate_rows > 0; its vectors are at scale + g * mod_stride (resp.
 * gate + g * gate_stride), fp32 copies of bf16 values, stride >= the row width and a multiple of 4. G = ceil(M / R).
 *
 * fvb_layernorm_modulate_grouped_bwd: backward of fvb_layernorm_modulate with round_ln = 3 and mod_rows = R, whose forward is
 *   t = bf16(LN(x)), G = bf16(1 + scale[g]), u = bf16(t G), n = bf16(u + shift[g]). x bf16 [M, D], dn bf16 [M, D]. Per row, fp32
 *   (torch's bf16 autograd rounding points):
 *   dt = bf16(dn * G),  dx = bf16(rstd * ((dt - mean_c(dt)) - t~ * mean_c(dt * t~)) [+ gin])   (t~ = the unrounded LN output;
 *   gin optional, fp32 or bf16 per gin_is_f32, added before the one rounding of dx)
 *   d_scale[g, c] = sum_{rows of g} dn * t,  d_shift[g, c] = sum_{rows of g} dn    (fp32 [G, D], row stride ld_dmod >= D)
 *   Group sums: P = clamp(528 / G, 1, R) fixed row sets per group (rows g R + p, g R + p + P, ...) summed in row order, the P
 *   partials added in p order; no atomics. D a multiple of 8, <= 8192; strides multiples of 8.
 *   workspace: fvb_layernorm_modulate_grouped_bwd_workspace_bytes(M, R, D) bytes, 16-byte aligned.
 *
 * fvb_resid_gate_grouped_bwd: backward of FVB_EPI_RESID_GATE_BF16R, out = bf16(resid + bf16(y gate[g])), given dout bf16 [M, N]
 *   and the saved bf16 y [M, N] (fvb_linear_bf16_aux's aux):
 *   dy[m, n] = bf16(dout * gate[g, n])                     bf16 [M, N] (lddy)
 *   d_gate[g, n] = sum_{rows of g} dout * y                fp32 [G, N] (row stride ld_dgate >= N)
 *   db[n] = bf16(sum_m float(dy[m, n]))                    bf16 [N] (db NULL: skipped)
 *   The residual's gradient is dout. Group sums as above with P = clamp(256 / G, 1, R); db adds all G P partials in (g, p)
 *   order. N a multiple of 8; strides keep rows 16-byte aligned. workspace: fvb_resid_gate_grouped_bwd_workspace_bytes(M, R, N)
 *   bytes, 16-byte aligned. */
int64_t fvb_layernorm_modulate_grouped_bwd_workspace_bytes(int M, int mod_rows, int D);
int fvb_layernorm_modulate_grouped_bwd(const void* x, int64_t ldx, const void* dn, int64_t lddn, const float* scale, int mod_rows,
                                       int64_t mod_stride, const void* gin, int gin_is_f32, int64_t ldgin, void* dx, int64_t lddx,
                                       float* d_scale, float* d_shift, int64_t ld_dmod, float* workspace,
                                       int64_t workspace_bytes, int M, int D, float eps, void* stream);
int64_t fvb_resid_gate_grouped_bwd_workspace_bytes(int M, int gate_rows, int N);
int fvb_resid_gate_grouped_bwd(const void* dout, int64_t lddout, const void* y, int64_t ldy, const float* gate, int gate_rows,
                               int64_t gate_stride, void* dy, int64_t lddy, float* d_gate, int64_t ld_dgate, void* db,
                               float* workspace, int64_t workspace_bytes, int M, int N, void* stream);

/* --------------------------------------------------------------------------------------------
 * Attention forward, head_dim 128, bf16, fp32 softmax. Dense or block-list (VSA / STA) keys.
 * Replaces: SDPAImpl.forward (fastvideo/attention/backends/sdpa.py:122-147), LocalAttention cross-attention
 *   (fastvideo/models/dits/wanvideo.py:188-222), block_sparse_attn_from_indices / block_sparse_sm100a_fwd
 *   (fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:347-393,
 *   fastvideo-kernel/csrc/attention/block_sparse_sm100a.cu:53-114), sliding_tile_attention
 *   (fastvideo-kernel/python/fastvideo_kernel/ops.py:21-62).
 * q/k/v/o are addressed as base + b*strides[0] + s*strides[1] + h*strides[2] (+ d), strides in elements,
 * so BSHD, BHSD and the fused-QKV GEMM output are all consumed in place.
 * lse (optional, fp32): lse[b*lse_stride_b + h*lse_stride_h + s] = max(qk*scale*log2e) + log2(sum).
 * Dense mode: sched == NULL; every key < Skv.
 * Block-list mode: 64-row q blocks 2p and 2p+1 share a CTA; sched[(b*sched_stride_b + h*sched_stride_h + p)
 *   * sched_cap + i] = kv_block | flags<<24 (ascending union of the two lists; flag bit0/bit1 = q block
 *   2p / 2p+1 attends it), sched_cnt[...] entries. q_off/kv_off (optional) give the first row of each
 *   block (default 64*block), q_len/kv_len the valid rows (default from offsets, else 64): keys past
 *   kv_len are masked, rows past q_len are not written. Empty lists give zeros and lse = -inf.
 * -------------------------------------------------------------------------------------------- */
int fvb_attention_fwd(const void* q, const void* k, const void* v, void* o, float* lse, const int64_t* q_strides,
                      const int64_t* k_strides, const int64_t* v_strides, const int64_t* o_strides,
                      int64_t lse_stride_b, int64_t lse_stride_h, int B, int H, int Sq, int Skv, int head_dim,
                      float softmax_scale, const int32_t* sched, const int32_t* sched_cnt, int64_t sched_stride_b,
                      int64_t sched_stride_h, int sched_cap, int num_pairs, const int32_t* q_off,
                      const int32_t* q_len, int nqb, const int32_t* kv_off, const int32_t* kv_len, int nkb,
                      void* stream);

/* Block-list attention for 64-row q blocks with per-block key lists (the two q blocks of a CTA merge their lists on the
 * fly, so a key block both select is loaded once). Consumes the reference's index format directly:
 * q2k_idx int32 [.., nqb, cap] ascending kv block ids (first q2k_num[..] valid), q2k_num int32 [.., nqb]
 * (map_to_index, fastvideo-kernel/python/fastvideo_kernel/triton_kernels/index.py:106-144); idx_stride_b / idx_stride_h
 * in q blocks (0 = broadcast over batch / heads). Same q/k/v/o addressing, offsets, lengths, masking, LSE and
 * empty-row semantics as fvb_attention_fwd. Replaces block_sparse_attn_from_indices
 * (fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:347-393) and block_sparse_sm100a_fwd
 * (fastvideo-kernel/csrc/attention/block_sparse_sm100a.cu:53-114). */
int fvb_attention_blocklist_fwd(const void* q, const void* k, const void* v, void* o, float* lse, const int64_t* q_strides,
                                const int64_t* k_strides, const int64_t* v_strides, const int64_t* o_strides,
                                int64_t lse_stride_b, int64_t lse_stride_h, int B, int H, int Sq, int Skv, int head_dim,
                                float softmax_scale, const int32_t* q2k_idx, const int32_t* q2k_num, int64_t idx_stride_b,
                                int64_t idx_stride_h, int cap, const int32_t* q_off, const int32_t* q_len, int nqb,
                                const int32_t* kv_off, const int32_t* kv_len, int nkb, void* workspace,
                                int64_t workspace_bytes, void* stream);
/* Bytes of caller-allocated device workspace (256-byte aligned) fvb_attention_blocklist_fwd accepts. Kept for ABI
 * compatibility only: the sm_90a kernel merges the two lists of a CTA while it walks them and uses no workspace. */
int64_t fvb_attention_blocklist_workspace_bytes(int index_rows, int nqb, int cap);

/* --------------------------------------------------------------------------------------------
 * 8-bit attention forward (opt-in; INT8 Q K^T, FP8 e4m3 P V), head_dim 128, bf16 in and out. The SageAttention2 scheme,
 * a quantised alternative to FastVideo's SAGE_ATTN backends (fastvideo/attention/backends/sage_attn.py) with this
 * library's own arithmetic, below. Per batch b and head h, every op fp32 round-to-nearest unless stated:
 *   K smoothing: k_mean[c] = (sum over all Skv keys of float(k[s, c])) / Skv -- per-256-key chunk sums in key order, then
 *     the chunk sums in chunk order (no atomics: the same result on every run); k'[s, c] = float(k[s, c]) - k_mean[c]. This
 *     adds q . k_mean to every logit of a row, so the softmax does not change.
 *   Q and K' to int8, one scale per (token, head) row of 128: amax = max |x|; amax == 0: scale = 1, row = 0; else
 *     inv = 127 / amax, x8 = clamp(rint(x * inv), -127, 127), scale = amax / 127.
 *   V to e4m3, one scale per (head, channel) over all Skv keys: amax = max_s |v[s, c]|; amax == 0: v_scale = 1, v8 = 0; else
 *     v8 = e4m3_satfinite_rn(v * (448 / amax)), v_scale = amax / 448.
 *   Logits: x = ((float(acc) * q_scale[m]) * k_scale[n]) * (softmax_scale * log2 e), acc the exact integer Q8 . K8 (s32);
 *     keys past a block's valid length are -inf.
 *   Online softmax over the 64-key tiles in the kernel's walk order: m = running max, p = exp2(x - m) (ex2.approx),
 *     l = l * alpha + sum of the unquantised p, alpha = exp2(m_old - m); p8 = e4m3_rn(p * 448).
 *   P V in two levels: T = sum over the tile's 64 key slots of p8 * v8 (tensor-core accumulation, into a fresh register set),
 *     then O = (O * alpha) + T (fp32).
 *   Output: o[m, c] = bf16((O[m, c] * v_scale[c]) * (1 / (448 * l[m]))); a row with no keys gives zeros. No LSE is written.
 *
 * fvb_attention_8bit_quantize: q [B, Sq, H, 128], k / v [B, Skv, H, 128] bf16 through (b, s, h) element strides (multiples of
 * 8; the views of a fused QKV buffer work in place) -> q8 int8 [B, H, Sq, 128], q_scale fp32 [B, H, Sq], k8 int8
 * [B, H, Skv, 128], k_scale fp32 [B, H, Skv], k_mean fp32 [B, H, 128], v_scale fp32 [B, H, 128] and
 *   vt8 e4m3 [B][H][nkb][128 channels][64 key slots]: key block kb, channel c, slot j holds v8 of key
 *     16 (j >> 4) + 2 ((j & 15) >> 2) + (j & 1) + 8 ((j >> 1) & 1) of the block, i.e. slot j of each 16-key group holds key
 *     2 (j >> 2) + (j & 1) + 8 ((j >> 1) & 1) of that group; slots of keys past the block's valid length are 0.
 *   This order lets P go from the S accumulator registers straight into the A-operand registers of the e4m3 wgmma.
 *   Key blocks as in fvb_attention_blocklist_fwd: kv_off (optional, [nkb + 1]) the first row of each block, kv_len (optional,
 *   [nkb]) the valid keys; without kv_off, block i is keys [64 i, 64 i + 64) and nkb must be ceil(Skv / 64).
 *   workspace: device memory of fvb_attention_8bit_workspace_bytes(B, H, Skv) bytes, 256-byte aligned.
 *
 * fvb_attention_8bit_fwd: the attention above on the quantiser's outputs (same B, H, Sq, Skv, key blocks kv_off / kv_len /
 * nkb). o bf16 through (b, s, h) element strides. Dense keys (every key block) with q2k_idx == q2k_num == NULL; otherwise
 * per-q-block lists with the format, q_off / q_len, masking and empty-row rules of fvb_attention_blocklist_fwd. lse must be
 * NULL (FVB_ERR_INVALID_ARG otherwise); the pair-schedule (STA) mode, sched != NULL, returns FVB_ERR_UNSUPPORTED.
 * -------------------------------------------------------------------------------------------- */
int64_t fvb_attention_8bit_workspace_bytes(int B, int H, int Skv);

int fvb_attention_8bit_quantize(const void* q, const void* k, const void* v, const int64_t* q_strides, const int64_t* k_strides,
                                const int64_t* v_strides, int B, int H, int Sq, int Skv, int head_dim, const int32_t* kv_off,
                                const int32_t* kv_len, int nkb, void* q8, float* q_scale, void* k8, float* k_scale,
                                float* k_mean, void* vt8, float* v_scale, void* workspace, int64_t workspace_bytes,
                                void* stream);

int fvb_attention_8bit_fwd(const void* q8, const float* q_scale, const void* k8, const float* k_scale, const void* vt8,
                           const float* v_scale, void* o, float* lse, const int64_t* o_strides, int B, int H, int Sq, int Skv,
                           int head_dim, float softmax_scale, const int32_t* sched, const int32_t* q2k_idx,
                           const int32_t* q2k_num, int64_t idx_stride_b, int64_t idx_stride_h, int cap, const int32_t* q_off,
                           const int32_t* q_len, int nqb, const int32_t* kv_off, const int32_t* kv_len, int nkb, void* stream);

/* Backward of fvb_attention_blocklist_fwd in the padded layout (block i = rows [64 i, 64 i + 64)): dq, dk, dv from q, k, v, o,
 * the forward's LSE (log2 domain) and dO. q2k_* as in the forward; k2q_idx int32 [.., nkb, capk] / k2q_num [.., nkb] list,
 * ascending, the q blocks that selected each kv block (the inverse lists, triton_kernels/index.py:147-250 invert_indices);
 * idx_stride_* / kidx_stride_* in rows of the respective index tensors (0 = broadcast). delta_ws: fp32 [B * H * Sq] workspace.
 * Replaces block_sparse_attn_backward_triton (fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:138-243;
 * triton_kernels/block_sparse_attn_triton.py:165-694). Warp-level mma.sync tiles (csrc/attn_bwd_sm90.cu). */
int fvb_attention_blocklist_bwd(const void* q, const void* k, const void* v, const void* o, const void* dO, const float* lse,
                                void* dq, void* dk, void* dv, float* delta_ws, const int64_t* q_strides,
                                const int64_t* k_strides, const int64_t* v_strides, const int64_t* o_strides,
                                const int64_t* do_strides, const int64_t* dq_strides, const int64_t* dk_strides,
                                const int64_t* dv_strides, int B, int H, int Sq, int Skv, int head_dim, float softmax_scale,
                                const int32_t* q2k_idx, const int32_t* q2k_num, int capq, const int32_t* k2q_idx,
                                const int32_t* k2q_num, int capk, int64_t idx_stride_b, int64_t idx_stride_h,
                                int64_t kidx_stride_b, int64_t kidx_stride_h, const int32_t* kv_len, void* stream);

/* Backward of fvb_attention_fwd in dense mode (sched == NULL): dq, dk, dv for any Sq >= 1, Skv >= 1. q, k, v, o, dO, dq,
 * dk, dv are addressed as in the forward (b, s, h element strides, multiples of 8; base addresses 16-byte aligned), lse is
 * the forward's (log2 domain, lse[b * lse_stride_b + h * lse_stride_h + s]). delta_ws: fp32 [B * H * Sq] workspace.
 * Per (b, h), over every key j < Skv, fp32 accumulation:
 *   delta_i = sum_c dO[i, c] * O[i, c]
 *   P_ij = exp2(q_i . k_j * softmax_scale * log2 e - lse_i)   (ex2.approx)
 *   dP_ij = dO_i . v_j         dS_ij = P_ij * (dP_ij - delta_i) * softmax_scale
 *   dV_j = sum_i bf16(P_ij) dO_i      dK_j = sum_i bf16(dS_ij) q_i      dQ_i = sum_j bf16(dS_ij) k_j
 * The arithmetic of fvb_attention_blocklist_bwd with every key selected. Deterministic: one kernel owns 128 keys per CTA
 * and walks every q tile (dK, dV), a second owns 128 q rows and walks every key tile (dQ; it recomputes S and dP); no
 * float atomics. Rows past Sq (keys past Skv) are neither read into the sums nor stored. wgmma + TMA (csrc/attn_bwd_sm90.cu). */
int fvb_attention_bwd(const void* q, const void* k, const void* v, const void* o, const void* dO, const float* lse,
                      int64_t lse_stride_b, int64_t lse_stride_h, void* dq, void* dk, void* dv, float* delta_ws,
                      const int64_t* q_strides, const int64_t* k_strides, const int64_t* v_strides, const int64_t* o_strides,
                      const int64_t* do_strides, const int64_t* dq_strides, const int64_t* dk_strides,
                      const int64_t* dv_strides, int B, int H, int Sq, int Skv, int head_dim, float softmax_scale,
                      void* stream);

/* Backward of fvb_attention_blocklist_fwd in either layout, on the wgmma kernels of fvb_attention_bwd. Arguments as in
 * fvb_attention_blocklist_bwd, plus the forward's lse strides (lse[b * lse_stride_b + h * lse_stride_h + s]) and its tile
 * addressing: q tile i starts at row q_off[i] (q_off NULL: 64 i) and has q_len[i] valid rows (q_len NULL: q_off[i + 1] -
 * q_off[i], else 64), at most 64 and never past Sq; kv tiles likewise from kv_off / kv_len / Skv. nqb / nkb tiles; q2k lists
 * [.., nqb, capq] of kv tiles, k2q lists [.., nkb, capk] of q tiles, both ascending (k2q = the transposed block map's lists).
 * Per (b, h), for the pairs (q tile, kv tile) the lists select, over valid q rows i and valid keys j, fp32 accumulation:
 *   delta_i = sum_c dO[i, c] * O[i, c]
 *   P_ij = exp2(q_i . k_j * softmax_scale * log2 e - lse_i)   (ex2.approx)
 *   dP_ij = dO_i . v_j         dS_ij = P_ij * (dP_ij - delta_i) * softmax_scale
 *   dV_j = sum_i bf16(P_ij) dO_i      dK_j = sum_i bf16(dS_ij) q_i      dQ_i = sum_j bf16(dS_ij) k_j
 * Tail rules: a kv tile's keys at or past its valid length give P = 0; q rows at or past a q tile's valid length take no
 * part (lse = +inf, delta = 0 for them), so the next tile's rows that a 64-row box starting at off[i] also reads count for
 * nothing. Only the valid rows of each tile are stored: rows outside every tile (pad rows of the padded layout) are not
 * written, and a tile never writes another tile's rows. A tile whose list is empty gets zeros. The arithmetic of
 * fvb_attention_bwd; deterministic (one CTA owns two 64-row tiles and walks the union of their lists; no float atomics). */
int fvb_attention_sparse_bwd(const void* q, const void* k, const void* v, const void* o, const void* dO, const float* lse,
                             int64_t lse_stride_b, int64_t lse_stride_h, void* dq, void* dk, void* dv, float* delta_ws,
                             const int64_t* q_strides, const int64_t* k_strides, const int64_t* v_strides,
                             const int64_t* o_strides, const int64_t* do_strides, const int64_t* dq_strides,
                             const int64_t* dk_strides, const int64_t* dv_strides, int B, int H, int Sq, int Skv, int head_dim,
                             float softmax_scale, const int32_t* q2k_idx, const int32_t* q2k_num, int capq,
                             const int32_t* k2q_idx, const int32_t* k2q_num, int capk, int64_t idx_stride_b,
                             int64_t idx_stride_h, int64_t kidx_stride_b, int64_t kidx_stride_h, const int32_t* q_off,
                             const int32_t* q_len, int nqb, const int32_t* kv_off, const int32_t* kv_len, int nkb,
                             void* stream);

/* --------------------------------------------------------------------------------------------
 * Index / mask construction (integer, bit-exact with the reference)
 * -------------------------------------------------------------------------------------------- */
/* Tile tables of a (T,H,W) token grid cut into (ts,hs,ws) tiles. Replaces get_tile_partition_indices,
 * get_reverse_tile_partition_indices, construct_variable_block_sizes, get_non_pad_index and
 * untile_combined_index (fastvideo/attention/backends/video_sparse_attn.py:32-114, 222; duplicate in
 * fastvideo-kernel/python/fastvideo_kernel/vsa_utils.py:30-109). Any output may be NULL.
 *   tile_partition[S] int64, reverse_partition[S] int64, non_pad[S] int64, untile_combined[S] int64,
 *   variable_block_sizes[n_tiles] int32, block_offsets[n_tiles+1] int32 (exclusive prefix sum of the
 *   block sizes: first row of each block in compact tile-major order; not a reference structure). */
int fvb_vsa_tile_index(int T, int H, int W, int ts, int hs, int ws, int64_t* tile_partition,
                       int64_t* reverse_partition, int64_t* non_pad, int64_t* untile_combined,
                       int32_t* variable_block_sizes, int32_t* block_offsets, void* stream);

/* mask[row, i] = 1 for the k largest scores of the row, ties at the threshold to the smallest index; exactly
 * min(k, n) ones per row. Replaces fused_topk_mask
 * (fastvideo-kernel/python/fastvideo_kernel/triton_kernels/fused_compress_topk.py:211-348).
 * scores_dtype: 0 = bf16, 1 = fp32; strides in elements. */
int fvb_topk_mask(const void* scores, int scores_dtype, int64_t row_stride, uint8_t* mask, int64_t mask_stride,
                  int64_t rows, int n, int k, void* stream);

/* Boolean block map rows -> ascending index lists padded with -1, and counts. Replaces map_to_index
 * (fastvideo-kernel/python/fastvideo_kernel/triton_kernels/index.py:33-61, 106-144).
 * q2k_idx: int32 [rows, n] contiguous; q2k_num: int32 [rows]. */
int fvb_map_to_index(const uint8_t* map, int64_t map_stride, int32_t* q2k_idx, int32_t* q2k_num, int64_t rows, int n,
                     void* stream);

/* fvb_topk_mask + fvb_map_to_index in one pass over bf16 score rows: the k largest scores of each row as an ascending index
 * list padded with -1 (q2k_idx int32 [rows, n]) and its length (q2k_num int32 [rows]); mask (may be NULL when n % 4 == 0,
 * n <= 2048 and rows are 8-byte aligned) additionally receives the boolean row. Same selection rule as fvb_topk_mask
 * (fused_compress_topk.py:211-348) and the same list as map_to_index (triton_kernels/index.py:33-61, 106-144) of that mask. */
int fvb_topk_index(const void* scores, int64_t row_stride, uint8_t* mask, int64_t mask_stride, int32_t* q2k_idx,
                   int32_t* q2k_num, int64_t rows, int n, int k, void* stream);

/* Boolean block map [BH, nq, nkv] -> the pair-union schedule consumed by fvb_attention_fwd:
 * sched int32 [BH, ceil(nq/2), cap], sched_cnt int32 [BH, ceil(nq/2)]. Strides in bytes (= elements). */
int fvb_pair_schedule(const uint8_t* map, int64_t bh_stride, int64_t q_stride, int BH, int nq, int nkv, int32_t* sched,
                      int32_t* sched_cnt, int cap, void* stream);

/* Sliding-tile window block map over tiles: map[head, q_tile, kv_tile] (uint8), tiles (t,h,w)-major;
 * window_thw: int32 [heads, 3] on the device. Mask semantics of generate_sta_mask
 * (fastvideo-kernel/tests/support_flex_sta.py:35-52), which sliding_tile_attention
 * (fastvideo-kernel/python/fastvideo_kernel/ops.py:21-62) is tested against. */
int fvb_sta_map(int canvas_t, int canvas_h, int canvas_w, const int32_t* window_thw, int heads, uint8_t* map,
                void* stream);

/* --------------------------------------------------------------------------------------------
 * Video Sparse Attention, compression branch and token permutations
 * -------------------------------------------------------------------------------------------- */
/* Per-block mean over the valid rows (fp32 accumulate, / block_len) -> out bf16 [B, H, nblk, 128]; out_t
 * (optional) is the same data transposed, [B, H, 128, ldt], the K-major operand of out_c = attn @ v_c.
 * x is addressed with (b, s, h) element strides. block_off (optional, int32 [nblk+1]) gives each block's first
 * row (compact layout); without it block i covers rows [i*block_rows, (i+1)*block_rows) of a zero-padded
 * buffer and block_len (int32 [nblk], = variable_block_sizes) is the divisor.
 * Replaces fused_block_mean (fastvideo-kernel/python/fastvideo_kernel/triton_kernels/fused_compress_topk.py:22-60). */
int fvb_block_mean(const void* x, const int64_t* strides, const int32_t* block_off, const int32_t* block_len,
                   int block_rows, int B, int H, int S, int nblk, void* out, void* out_t, int64_t ldt, void* stream);

/* Row softmax, bf16 in / bf16 out, fp32 math (torch.softmax(scores, -1) on bf16; ops.py:113). n <= 8192. */
int fvb_softmax_rows(const void* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int n, void* stream);

/* out = out_c (broadcast over its block) * gate + out_s, with the reference's bf16 rounding after the product
 * and after the sum (ops.py:117-133). out_s/gate/out use (b, s, h) element strides; out_c is [B, H, nblk, 128];
 * row_block (optional int32 [S]) maps a token row to its block (default row / block_rows). gate may be NULL. */
int fvb_vsa_combine(const void* out_s, const int64_t* s_strides, const void* gate, const int64_t* g_strides,
                    const void* out_c, const int32_t* row_block, int block_rows, void* out, const int64_t* o_strides,
                    int B, int S, int H, int nblk, const int64_t* out_seg_base, int seg_rows, void* stream);
/* (out_seg_base != NULL, B == 1): segmented destination -- row tok is stored at (bf16*)out_seg_base[tok / seg_rows] +
 * (tok % seg_rows) * o_strides[1] + h * o_strides[2]. The sequence-parallel return exchange of DistributedAttention_VSA
 * (fastvideo/attention/layer.py:232-245; base_device_communicator.py:123-193) done by this kernel's stores into the token
 * owners' peer-mapped buffers instead of an all-to-all. */

/* Row r of x [S, width] (bf16, row stride ldx) -> (bf16*)seg_base[r / seg_rows] + (r % seg_rows) * dst_ld. The same
 * return exchange after dense attention (fastvideo/attention/layer.py:147-164). */
int fvb_scatter_rows_to_segments(const void* x, int64_t ldx, int64_t S, int width, const int64_t* seg_base, int seg_rows,
                                 int64_t dst_ld, void* stream);

/* out[b, i, 0:width] = in[b, idx[i], 0:width] (rows of bf16; idx < 0 writes zeros). The tile / untile gathers of
 * VideoSparseAttentionImpl.preprocess_qkv / postprocess_output
 * (fastvideo/attention/backends/video_sparse_attn.py:254-303). idx: int64 (idx_is_i64) or int32, on the device. */
int fvb_gather_rows(const void* in, int64_t in_batch_stride, int64_t in_ld, const void* idx, int idx_is_i64, void* out,
                    int64_t out_batch_stride, int64_t out_ld, int64_t n_out, int width, int B, void* stream);

/* --------------------------------------------------------------------------------------------
 * Video Sparse Attention backward. Padded layout: S = 64 * nblk token rows, tile i = rows [64 i, 64 i + 64) of which
 * the first len[i] = block_len[i] (variable_block_sizes) are valid. The backward of video_sparse_attn
 * (fastvideo-kernel/python/fastvideo_kernel/ops.py:65-133) as torch autograd differentiates it, top-k selection excluded:
 *   combine:      fvb_vsa_combine_bwd
 *   compression:  d_attn = d_out_c v_c^T,  d_v_c = attn^T d_out_c  (fvb_gemm_batched_bf16),
 *                 d_scores' = fvb_softmax_rows_bwd(attn, d_attn, scale = 1 / sqrt(d)),
 *                 d_q_c = d_scores' k_c,  d_k_c = d_scores'^T q_c  (fvb_gemm_batched_bf16)
 *   sparse:       dq_s, dk_s, dv_s = fvb_attention_blocklist_bwd (compact layout: fvb_attention_sparse_bwd)
 *   block means:  fvb_block_mean_bwd (dq from dq_s and d_q_c, dk and dv likewise)
 *
 * Pad rows are not tokens: every gradient below treats dO there as zero (the forward's sparse-branch rows there are zero,
 *   and its LSE is -inf, so fvb_attention_blocklist_bwd gives them no weight either).
 *
 * fvb_vsa_combine_bwd: backward of fvb_vsa_combine. dO, gate, d_gate [B, S, H, 128] through (b, s, h) element strides
 *   (multiples of 8); out_c, d_out_c bf16 [B, H, nblk, 128] contiguous.
 *   d_gate[t, c] = bf16(dO[t, c] * out_c[tile(t), c]) on the valid rows, 0 on the pad rows (only when d_gate != NULL)
 *   d_out_c[i, c] = bf16(sum over the valid rows t of tile i of dO[t, c] * gate[t, c]); gate == NULL: of dO[t, c]
 *   The products are exact in fp32; the sum is fp32 in a fixed order (16 row-group partial sums, each over its rows in
 *   order, then the 16 partials in order), so the same inputs give the same bits. d_out_c_t (optional) receives the same
 *   values transposed, [B, H, 128, ldt] (ldt >= nblk): the K-major operand of d_v_c = attn^T d_out_c.
 *
 * fvb_softmax_rows_bwd: backward of fvb_softmax_rows over batch square blocks [n, n] (n <= 8192): p = the softmax output
 *   and dp = its gradient, bf16, block b at base + b * n * ld, rows of stride ld (a multiple of 8, >= n), 16-byte aligned.
 *   r[i] = sum_j dp[i, j] * p[i, j]                         (fp32 fused multiply-adds, a fixed order)
 *   ds[i, j] = bf16((p[i, j] * (dp[i, j] - r[i])) * scale)   (fp32 round-to-nearest, in that order)
 *   Same layout for ds; ds_t (optional) receives ds transposed (ds_t[j, i] = ds[i, j]) and p_t (optional) p transposed,
 *   both in the same [batch, n, ld] layout. scale = 1 / sqrt(d) folds the score scaling of q_c k_c^T / sqrt(d) into d_scores.
 *
 * fvb_block_mean_bwd: backward of fvb_block_mean (padded layout) added to a gradient that already reaches the rows:
 *   dx[t, c] = bf16(dx_s[t, c] + d_mean[tile(t), c] / len[tile(t)])   for the valid rows t (fp32 division, then addition)
 *   dx[t, c] = 0                                                        for the pad rows
 *   dx_s, dx [B, S, H, 128] through (b, s, h) element strides (multiples of 8); dx may be dx_s (in place). d_mean bf16
 *   [B, H, nblk, 128] contiguous.
 *
 * Compact layout (the *_compact variants): S token rows in tile-major order without pad rows, tile i = rows
 *   [block_off[i], block_off[i + 1]) (block_off int32 [nblk + 1], as fvb_block_mean takes it), row_block int32 [S] = the tile
 *   of each row (as fvb_vsa_combine takes it). Every row is a token, so there are no pad-row zeroes:
 *   fvb_vsa_combine_bwd_compact: d_gate[t, c] = bf16(dO[t, c] * out_c[tile(t), c]) for every row; d_out_c[i, c] = the sum
 *     over rows block_off[i] + r, r < block_off[i + 1] - block_off[i], in the fixed order of fvb_vsa_combine_bwd (row r in
 *     group r % 16). Other arguments as there.
 *   fvb_block_mean_bwd_compact: dx[t, c] = bf16(dx_s[t, c] + d_mean[tile(t), c] / len) for every row t, tile(t) =
 *     row_block[t], len = block_off[tile + 1] - block_off[tile]. Other arguments as in fvb_block_mean_bwd.
 * -------------------------------------------------------------------------------------------- */
int fvb_vsa_combine_bwd(const void* dO, const int64_t* do_strides, const void* gate, const int64_t* g_strides,
                        const void* out_c, const int32_t* block_len, int B, int S, int H, int nblk, void* d_gate,
                        const int64_t* dg_strides, void* d_out_c, void* d_out_c_t, int64_t ldt, void* stream);

int fvb_softmax_rows_bwd(const void* p, const void* dp, int64_t ld, int batch, int n, float scale, void* ds, void* ds_t,
                         void* p_t, void* stream);

int fvb_block_mean_bwd(const void* dx_s, const int64_t* s_strides, const void* d_mean, const int32_t* block_len, int B,
                       int H, int S, int nblk, void* dx, const int64_t* dx_strides, void* stream);

int fvb_vsa_combine_bwd_compact(const void* dO, const int64_t* do_strides, const void* gate, const int64_t* g_strides,
                                const void* out_c, const int32_t* block_off, int B, int S, int H, int nblk, void* d_gate,
                                const int64_t* dg_strides, void* d_out_c, void* d_out_c_t, int64_t ldt, void* stream);

int fvb_block_mean_bwd_compact(const void* dx_s, const int64_t* s_strides, const void* d_mean, const int32_t* block_off,
                               const int32_t* row_block, int B, int H, int S, int nblk, void* dx, const int64_t* dx_strides,
                               void* stream);

/* --------------------------------------------------------------------------------------------
 * Wan VAE decode (channels-last frames x[t][h][w][c], bf16)
 * -------------------------------------------------------------------------------------------- */
/* out_f32[M, N] = (A[M, K] @ B[N, K]^T) * scale, fp32 output (attention logits of WanAttentionBlock). */
int fvb_gemm_f32out(const void* a, int64_t lda, const void* b, int64_t ldb, float* out, int64_t ldo, int M, int N, int K,
                    float scale, void* stream);

/* Causal Conv3d / Conv2d as a TMA-staged implicit GEMM (wgmma). Replaces WanCausalConv3d.forward
 * (fastvideo/models/vaes/wanvae.py:160-207) and the Conv2d of WanResample (wanvae.py:272-281).
 *   x: [T_in][H][W][Cin] input frames: the (<= 2) cached frames of the feature cache followed by the new frames;
 *   t_off = number of cached frames present; output frame j (0 <= j < T_out) is computed from input frames
 *   t_off + j - (kt-1) .. t_off + j (frames before the buffer start are zeros = causal padding); "same" zero padding
 *   in h and w. w_packed: bf16 [Cout][kt*kh*kw][Cin_pad] (fvb packs it from the reference's [Cout, Cin, kt, kh, kw]).
 *   y = bf16(acc + bias); out = bf16(y + resid) if resid. out: [T_out][H][W][out_ld].
 *   interleave_c = Cout/2: output channel c of frame j goes to frame 2j + c / interleave_c, channel c % interleave_c
 *   (the reshape + stack after time_conv in upsample3d, wanvae.py:343-345; out must hold 2*T_out frames).
 *   One TMA box of activations per tap and channel block. */
int fvb_conv3d_cl(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad, int Cout, int kt,
                  int kh, int kw, const void* bias, const void* resid, int64_t resid_ld, void* out, int64_t out_ld,
                  int T_out, int t_off, int interleave_c, void* stream);

/* The same convolution with the CONSUMER's WanRMS_norm (+ SiLU) fused into the epilogue (16 < Cout <= 192: one tile holds a
 * pixel's whole channel row): besides (or instead of: out may be NULL) the raw bf16 output row y it writes
 *   norm_out = silu?( y / max(||y||_2, 1e-12) * sqrt(Cout) * norm_gamma ),  fp32 math on the bf16 values of y,
 * i.e. fvb_rmsnorm_silu_cl(fvb_conv3d_cl(...)) without the extra pass over the activation. In WanResidualBlock
 * (wanvae.py:383-462) conv1 feeds only norm2 -> SiLU -> conv2 (out = NULL), and conv2 + shortcut feeds the next block's
 * norm1 as well as its residual path (both outputs). */
int fvb_conv3d_cl_norm(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad, int Cout, int kt,
                       int kh, int kw, const void* bias, const void* resid, int64_t resid_ld, void* out, int64_t out_ld,
                       int T_out, int t_off, const float* norm_gamma, void* norm_out, int64_t norm_ld, int norm_silu,
                       void* stream);

/* WanRMS_norm (+ SiLU): y = x / max(||x||_2, 1e-12) * sqrt(C) * gamma (+ beta), fp32 math (wanvae.py:210-233). */
int fvb_rmsnorm_silu_cl(const void* x, int64_t ldx, const float* gamma, const float* beta, void* out, int64_t ldo,
                        int64_t npix, int C, int apply_silu, void* stream);

/* --------------------------------------------------------------------------------------------
 * FP8 (e4m3) residual-block convolutions of the Wan VAE decoder
 *
 * Static activation scale. Every conv1 / conv2 of a WanResidualBlock reads v = silu?(y / ||y|| * sqrt(C) * gamma), so
 * |v_c| <= bound = sqrt(C) * max_c |gamma_c| (SiLU never raises the magnitude). The norm that produces v writes it as
 *   q = e4m3_satfinite_rn(v * inv),  inv = 448.0f / bound (IEEE fp32 division);  bound == 0: inv = 0 (q = 0)
 * and the convolution reads it with x_scale = bound / 448 (1 when bound == 0). satfinite absorbs the last-ulp overshoot of
 * the rounded norm. No amax pass; the scale is known when the weights are loaded.
 *
 * fvb_conv3d_cl_fp8: fvb_conv3d_cl with x e4m3 [T_in][H][W][Cin] (Cin % 16 == 0: 16-byte pixel rows) and
 *   w_packed e4m3 [Cout][kt*kh*kw][Cin_pad] with w_scale fp32 [Cout] (fvb_quantize_fp8_rows of the packed bf16 weight:
 *   one scale per output channel; the zero padding does not change the amax):
 *   acc = sum over taps and channels of x * w            (wgmma .e4m3 products, fp32 accumulators in the tensor core)
 *   y = bf16(((acc * x_scale) * w_scale[n]) + bias[n]);  out = bf16(y + resid) if resid  (as fvb_conv3d_cl)
 *   No interleave_c.
 * fvb_conv3d_cl_fp8_norm: the same with the consumer's norm fused as in fvb_conv3d_cl_norm (16 < Cout <= 192);
 *   norm_e4m3 == 0: norm_out bf16; norm_e4m3 != 0: norm_out e4m3 = e4m3_satfinite_rn(normed * (448 / norm_bound)),
 *   normed the fp32 value the bf16 output would round (norm_ld % 16 == 0).
 * fvb_conv3d_cl_norm_e4m3: fvb_conv3d_cl_norm (bf16 operands) writing its normalised output as e4m3 by the same rule
 *   (the upsampler convolution that feeds a residual block).
 * fvb_rmsnorm_silu_cl_e4m3: fvb_rmsnorm_silu_cl (no beta) writing e4m3 by the same rule; the separate pass for
 *   Cout > 192 and after the mid-block attention.
 * -------------------------------------------------------------------------------------------- */
int fvb_conv3d_cl_fp8(const void* x, int T_in, int H, int W, int Cin, float x_scale, const void* w_packed,
                      const float* w_scale, int Cin_pad, int Cout, int kt, int kh, int kw, const void* bias,
                      const void* resid, int64_t resid_ld, void* out, int64_t out_ld, int T_out, int t_off, void* stream);

int fvb_conv3d_cl_fp8_norm(const void* x, int T_in, int H, int W, int Cin, float x_scale, const void* w_packed,
                           const float* w_scale, int Cin_pad, int Cout, int kt, int kh, int kw, const void* bias,
                           const void* resid, int64_t resid_ld, void* out, int64_t out_ld, int T_out, int t_off,
                           const float* norm_gamma, void* norm_out, int64_t norm_ld, int norm_silu, int norm_e4m3,
                           float norm_bound, void* stream);

int fvb_conv3d_cl_norm_e4m3(const void* x, int T_in, int H, int W, int Cin, const void* w_packed, int Cin_pad, int Cout,
                            int kt, int kh, int kw, const void* bias, const void* resid, int64_t resid_ld, void* out,
                            int64_t out_ld, int T_out, int t_off, const float* norm_gamma, void* norm_out, int64_t norm_ld,
                            int norm_silu, float norm_bound, void* stream);

int fvb_rmsnorm_silu_cl_e4m3(const void* x, int64_t ldx, const float* gamma, void* out, int64_t ldo, int64_t npix, int C,
                             int apply_silu, float bound, void* stream);

/* nearest-exact 2x spatial upsample of [T][H][W][C] -> [T][2H][2W][C] (WanUpsample, wanvae.py:236-248). */
int fvb_upsample2x_cl(const void* in, void* out, int T, int H, int W, int C, void* stream);

int fvb_transpose_bf16(const void* in, int64_t ldi, void* out, int64_t ldo, int R, int C, void* stream);

/* bf16 probabilities = softmax(fp32 logits row), any row length. */
int fvb_softmax_rows_f32(const float* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int n, void* stream);

/* [npix][ld] bf16 channels-last (first C channels) -> fp32 [C][npix], clamped to [-1, 1] (wanvae.py:1210-1211). */
int fvb_clamp_to_nchw(const void* in, int64_t ld, float* out, int C, int64_t npix, void* stream);

/* --------------------------------------------------------------------------------------------
 * Scheduler step (closes a denoising step; elementwise, bit-exact with the reference's chains of fp32 torch ops)
 * -------------------------------------------------------------------------------------------- */
/* x0 = sample - sigma * model_output (FlowUniPCMultistepScheduler.convert_model_output, flow_prediction + predict_x0,
 * fastvideo/models/schedulers/scheduling_flow_unipc_multistep.py:296-362). sample / x0 fp32, model_output bf16 or fp32. */
int fvb_sched_convert_x0(const float* sample, const void* model_output, int model_output_is_bf16, float sigma, float* x0,
                         int64_t n, void* stream);
/* out = (a*x - b*m0) - c * ( r0 * ((m1 - m0) / rk) + r1 * (mt - m0) ): multistep_uni_p_bh_update (mt == NULL) and
 * multistep_uni_c_bh_update (mt = this step's converted output) of the same file (:364-489, :491-619), orders 1 (m1 == NULL)
 * and 2, solver bh1/bh2 (the scalars a, b, c, r0, rk, r1 are computed on the host exactly as the reference does). */
int fvb_sched_unipc_update(const float* x, const float* m0, const float* m1, const float* mt, float a, float b, float c,
                           float r0, float rk, float r1, float* out, int64_t n, void* stream);
/* prev = (sample + dt * model_output) -> model_output's dtype (FlowMatchEulerDiscreteScheduler.step,
 * fastvideo/models/schedulers/scheduling_flow_match_euler_discrete.py:436-531, deterministic branch). */
int fvb_sched_euler_step(const float* sample, const void* model_output, int model_output_is_bf16, float dt, void* out,
                         int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FVB200_H */
