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

/* Batched C[i] = bf16(A[i] @ B[i]^T), optionally followed by out = bf16(float(C) / div) (div = 0 or 1: none).
 * A[i]: [M, K] ld=lda, B[i]: [N, K] ld=ldb, out[i]: [M, N] ld=ldo; batch strides in elements (multiples of 8).
 * Replaces the block-level matmuls of video_sparse_attn's compression branch
 * (fastvideo-kernel/python/fastvideo_kernel/ops.py:112-116): scores = q_c @ k_c^T / sqrt(d), out_c = attn @ v_c. */
int fvb_gemm_batched_bf16(const void* a, int64_t lda, int64_t a_batch_stride, const void* b, int64_t ldb,
                          int64_t b_batch_stride, void* out, int64_t ldo, int64_t out_batch_stride, int M, int N, int K,
                          int batch, float div, void* stream);

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
