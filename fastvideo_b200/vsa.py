"""Video Sparse Attention composite on libfvb200 (mirrors fastvideo_kernel.video_sparse_attn,
fastvideo-kernel/python/fastvideo_kernel/ops.py:65-133).

  q_c, k_c, v_c = block means          -> fvb_block_mean
  scores = q_c k_c^T / sqrt(d)         -> fvb_gemm_batched_bf16 (tcgen05)
  out_c  = softmax(scores) v_c         -> fvb_softmax_rows + fvb_gemm_batched_bf16
  mask   = topk(scores)                -> fvb_topk_index (block map + index lists in one pass) / fvb_topk_mask, fvb_pair_schedule
  out_s  = block-sparse attention      -> fvb_attention_fwd (tcgen05)
  out    = out_c * gate + out_s        -> fvb_vsa_combine

Two token layouts are supported by the same kernels:
  * padded  (reference API): [.., S_pad, ..] with every tile occupying 64 rows, zero padded;
  * compact (this engine):   tile-major order without padding; block_off gives each tile's first row.
"""
from __future__ import annotations

import math

import torch

import os

from . import ops

# Sparse-branch kernel: "ws" = per-q-block lists on the weight-stationary M=64 path (fvb_attention_blocklist_fwd),
# "union" = M=128 over the union of two neighbouring q blocks' lists (fvb_attention_fwd block-list mode).
SPARSE_KERNEL = os.environ.get("FVB_VSA_KERNEL", "ws")


def video_sparse_attn_bshd(q, k, v, variable_block_sizes, topk: int, gate=None, block_off=None, row_block=None,
                           out=None, return_aux: bool = False, out_segments=None, attn_8bit: bool = False):
    """q/k/v/gate: [B, S, H, 128] bf16 views (strided ok). variable_block_sizes: int32 [nblk] on device.
    block_off: int32 [nblk+1] for the compact layout, None for the padded one.
    attn_8bit: the sparse branch runs the 8-bit attention (ops.quantize_attention_8bit once, then ops.attention_8bit on the
    per-q-block lists); the compression branch stays bf16.
    out_segments = (int64 device table of P base addresses, rows per segment, (b, s, h) element strides): the result rows
    are stored segment by segment at those addresses (sequence-parallel return path: peer memory) instead of `out`."""
    B, S, H, d = q.shape
    nblk = variable_block_sizes.numel()
    vbs = variable_block_sizes
    if vbs.dtype != torch.int32:
        vbs = vbs.to(torch.int32)
    q_c = ops.block_mean(q, nblk, block_off, vbs)
    k_c = ops.block_mean(k, nblk, block_off, vbs)
    v_c, v_ct = ops.block_mean(v, nblk, block_off, vbs, want_transposed=True)
    scores = ops.gemm_batched(q_c.view(B * H, nblk, d), k_c.view(B * H, nblk, d), div=math.sqrt(d))  # [BH, nq, nk]
    attn = ops.softmax_rows(scores)
    out_c = ops.gemm_batched(attn, v_ct.reshape(B * H, d, -1)).contiguous().view(B, H, nblk, d)
    if attn_8bit:
        q2k_idx, q2k_num, mask = ops.topk_index(scores, topk, want_mask=return_aux)
        q2k_idx, q2k_num = q2k_idx.view(B, H, nblk, nblk), q2k_num.view(B, H, nblk)
        if mask is not None:
            mask = mask.view(B, H, nblk, nblk)
        qin = ops.quantize_attention_8bit(q, k, v, kv_off=block_off, kv_len=vbs, nkb=nblk)
        out_s = ops.attention_8bit(qin, d ** -0.5, q2k_idx, q2k_num, q_off=block_off, q_len=vbs)
    elif SPARSE_KERNEL == "ws":
        # block map and index lists in one pass over the scores (fvb_topk_index); the boolean map only when the caller asks
        q2k_idx, q2k_num, mask = ops.topk_index(scores, topk, want_mask=return_aux)
        q2k_idx, q2k_num = q2k_idx.view(B, H, nblk, nblk), q2k_num.view(B, H, nblk)
        if mask is not None:
            mask = mask.view(B, H, nblk, nblk)
        out_s = ops.attention_blocklist(q, k, v, q2k_idx, q2k_num, softmax_scale=d ** -0.5, q_off=block_off, kv_off=block_off,
                                        q_len=vbs, kv_len=vbs, nkb=nblk)
    else:
        mask = ops.topk_mask(scores, topk).view(B, H, nblk, nblk)
        sched, cnt = ops.pair_schedule(mask)
        out_s = ops.attention(q, k, v, softmax_scale=d ** -0.5, sched=sched, sched_cnt=cnt,
                              q_off=block_off, kv_off=block_off, q_len=vbs, kv_len=vbs, nqb=nblk, nkb=nblk)
    res = ops.vsa_combine(out_s, out_c, gate, row_block=row_block, out=out, out_segments=out_segments)
    if return_aux:
        return res, dict(q_c=q_c, k_c=k_c, v_c=v_c, scores=scores, attn=attn, out_c=out_c, mask=mask, out_s=out_s)
    return res


def video_sparse_attn(q, k, v, variable_block_sizes, q_variable_block_sizes, topk, block_size=64,
                      compress_attn_weight=None):
    """Reference signature (ops.py:65-74): [B, H, S_pad, D] tensors, 64-token tiles, zero padded."""
    if isinstance(block_size, (tuple, list)):
        block_size = math.prod(block_size)
    if block_size != 64:
        raise ValueError("libfvb200 implements the 64-token-tile VSA path")
    if q.shape[2] % 64 or k.shape[2] % 64:
        raise ValueError("q_seq_len and kv_seq_len must be divisible by block_elements=64")
    gate = None if compress_attn_weight is None else compress_attn_weight.transpose(1, 2)
    out = torch.empty_like(q)
    video_sparse_attn_bshd(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), variable_block_sizes, topk, gate=gate,
                           out=out.transpose(1, 2))
    return out
