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


class _VideoSparseAttnFn(torch.autograd.Function):
    """video_sparse_attn with autograd, in either token layout. The forward runs the kernels of video_sparse_attn_bshd's
    block-list path in the same order, so its output is bit-identical, and keeps what the backward needs. The backward is
    what torch autograd computes for the reference composite (ops.py:65-133); the top-k selection has no gradient:
      sparse branch   padded: fvb_attention_blocklist_bwd; compact: fvb_attention_sparse_bwd (kv -> q lists from the
                      transposed block map)
      combine         fvb_vsa_combine_bwd(_compact): d_gate = dO * out_c, d_out_c = per-tile sum of dO * gate
      compression     d_attn = d_out_c v_c^T, d_v_c = attn^T d_out_c, d_scores' = softmax backward / sqrt(d),
                      d_q_c = d_scores' k_c, d_k_c = d_scores'^T q_c (fvb_gemm_batched_bf16; the transposed operands
                      come from the kernels that produce them)
      block means     fvb_block_mean_bwd(_compact): dq = dq_s + d_q_c / len on the token rows, 0 on pad rows (k, v likewise)
    Padded layout (block_off None): q, k, v, gate are [B, H, S_pad, 128] (the reference signature). Compact layout: they are
    [B, S, H, 128] views in tile-major order, block_off int32 [nblk + 1] / row_block int32 [S] the tile tables.
    block_map (bool [B, H, nblk, nblk], or None for the top-k of the block scores) fixes the selection; it is how the
    tests reach q blocks without keys, which top-k never produces."""

    # the order of ctx.saved_tensors (callers that run forward / backward with a stand-in ctx read them by these names)
    SAVED = ("q", "k", "v", "gate", "vbs", "q_ct", "k_ct", "v_c", "attn", "out_c", "out_s", "lse", "q2k_idx", "q2k_num",
             "block_map", "block_off", "row_block")

    @staticmethod
    def forward(ctx, q, k, v, gate, vbs, topk, block_map, block_off=None, row_block=None):
        if SPARSE_KERNEL != "ws":
            raise ops.FvbError("the VSA backward needs the block-list sparse kernel (FVB_VSA_KERNEL=ws)")
        compact = block_off is not None
        if compact:
            B, S, H, d = q.shape
            nblk = vbs.numel()
            qt, kt, vt, gt = q, k, v, gate
        else:
            B, H, S, d = q.shape
            nblk = S // 64
            qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
            gt = None if gate is None else gate.transpose(1, 2)
        q_c, q_ct = ops.block_mean(qt, nblk, block_off, vbs, want_transposed=True)
        k_c, k_ct = ops.block_mean(kt, nblk, block_off, vbs, want_transposed=True)
        v_c, v_ct = ops.block_mean(vt, nblk, block_off, vbs, want_transposed=True)
        scores = ops.gemm_batched(q_c.view(B * H, nblk, d), k_c.view(B * H, nblk, d), div=math.sqrt(d))
        attn = ops.softmax_rows(scores)
        out_c = ops.gemm_batched(attn, v_ct.reshape(B * H, d, -1)).contiguous().view(B, H, nblk, d)
        if block_map is None:
            q2k_idx, q2k_num, block_map = ops.topk_index(scores, topk, want_mask=True)
        else:
            q2k_idx, q2k_num = ops.map_to_index(block_map.contiguous())
        q2k_idx, q2k_num = q2k_idx.view(B, H, nblk, nblk), q2k_num.view(B, H, nblk)
        out_s, lse = ops.attention_blocklist(qt, kt, vt, q2k_idx, q2k_num, softmax_scale=d ** -0.5, q_off=block_off,
                                             kv_off=block_off, q_len=vbs, kv_len=vbs, nkb=nblk, return_lse=True)
        if compact:
            out = ops.vsa_combine(out_s, out_c, gt, row_block=row_block)
        else:
            out = torch.empty_like(q)
            ops.vsa_combine(out_s, out_c, gt, out=out.transpose(1, 2))
        ctx.save_for_backward(q, k, v, gate, vbs, q_ct, k_ct, v_c, attn, out_c, out_s, lse, q2k_idx, q2k_num,
                              block_map.view(B, H, nblk, nblk), block_off, row_block)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (q, k, v, gate, vbs, q_ct, k_ct, v_c, attn, out_c, out_s, lse, q2k_idx, q2k_num, block_map, block_off,
         row_block) = ctx.saved_tensors
        compact = block_off is not None
        want_d_gate = gate is not None and ctx.needs_input_grad[3]
        if compact:
            B, S, H, d = q.shape
            nblk = vbs.numel()
            go = grad_out.to(torch.bfloat16).contiguous()
            qt, kt, vt, gt = q, k, v, gate
            d_gate = torch.empty((B, S, H, d), dtype=torch.bfloat16, device=q.device) if want_d_gate else None
            dgt = d_gate
        else:
            B, H, S, d = q.shape
            nblk = S // 64
            go = grad_out.to(torch.bfloat16).contiguous().transpose(1, 2)
            qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
            gt = None if gate is None else gate.transpose(1, 2)
            d_gate = torch.empty_like(gate) if want_d_gate else None
            dgt = None if d_gate is None else d_gate.transpose(1, 2)
        BH = B * H
        d_out_c, d_out_c_t = ops.vsa_combine_bwd(go, out_c, gt, vbs, d_gate=dgt, block_off=block_off)
        # compression branch
        d_attn = ops.gemm_batched(d_out_c.view(BH, nblk, d), v_c.view(BH, nblk, d))
        d_scores, d_scores_t, attn_t = ops.softmax_rows_bwd(attn, d_attn, scale=d ** -0.5, want_transposed=True)
        d_v_c = ops.gemm_batched(attn_t, d_out_c_t.reshape(BH, d, nblk))
        d_q_c = ops.gemm_batched(d_scores, k_ct.reshape(BH, d, nblk))
        d_k_c = ops.gemm_batched(d_scores_t, q_ct.reshape(BH, d, nblk))
        # sparse branch: kv block -> the q blocks that selected it, from the transposed block map
        k2q_idx, k2q_num = ops.map_to_index(block_map.transpose(-1, -2).contiguous())
        if compact:
            dq, dk, dv = ops.attention_sparse_bwd(qt, kt, vt, out_s, lse, go, q2k_idx, q2k_num, k2q_idx, k2q_num,
                                                  q_off=block_off, q_len=vbs, kv_off=block_off, kv_len=vbs)
        else:
            dq, dk, dv = ops.attention_blocklist_bwd(qt, kt, vt, out_s, lse, go, q2k_idx, q2k_num, k2q_idx, k2q_num, kv_len=vbs)
        for dx, dc in ((dq, d_q_c), (dk, d_k_c), (dv, d_v_c)):
            ops.block_mean_bwd(dx, dc.contiguous().view(B, H, nblk, d), vbs, out=dx, block_off=block_off, row_block=row_block)
        if compact:
            return dq, dk, dv, d_gate, None, None, None, None, None
        return dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2), d_gate, None, None, None, None, None


def video_sparse_attn(q, k, v, variable_block_sizes, q_variable_block_sizes, topk, block_size=64,
                      compress_attn_weight=None):
    """Reference signature (ops.py:65-74): [B, H, S_pad, D] tensors, 64-token tiles, zero padded.
    Differentiable in q, k, v and compress_attn_weight (the gate): when any of them requires grad the call runs through
    _VideoSparseAttnFn, whose forward gives the same bits as the call without grad."""
    if isinstance(block_size, (tuple, list)):
        block_size = math.prod(block_size)
    if block_size != 64:
        raise ValueError("libfvb200 implements the 64-token-tile VSA path")
    if q.shape[2] % 64 or k.shape[2] % 64:
        raise ValueError("q_seq_len and kv_seq_len must be divisible by block_elements=64")
    inputs = (q, k, v) if compress_attn_weight is None else (q, k, v, compress_attn_weight)
    if torch.is_grad_enabled() and any(t.requires_grad for t in inputs):
        vbs = variable_block_sizes.to(torch.int32).contiguous()
        return _VideoSparseAttnFn.apply(q, k, v, compress_attn_weight, vbs, topk, None)
    gate = None if compress_attn_weight is None else compress_attn_weight.transpose(1, 2)
    out = torch.empty_like(q)
    video_sparse_attn_bshd(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), variable_block_sizes, topk, gate=gate,
                           out=out.transpose(1, 2))
    return out
