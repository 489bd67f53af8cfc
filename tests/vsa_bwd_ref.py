"""Restatement of the Video Sparse Attention backward (padded layout, 64-row tiles) that fastvideo_b200.vsa computes.

`composite` is the forward as torch expresses it: block means, compression softmax and matmuls, block-sparse attention as
the dense masked formula on a given block map, and `out_c * gate + out_s`. Torch autograd of it is the truth. Pad rows
(rows past variable_block_sizes in a tile) are not tokens: the composite reads q, k, v through the valid-row mask, attends
from and to valid rows only, and keeps only the valid output rows. Their values are unchanged by that (the padding is
zero), and it defines the gradient as that of the token rows.

`backward` restates the formulas the kernels evaluate, stage by stage (fvb200.h, "Video Sparse Attention backward"):
sparse branch, combine, compression matmuls with the row-softmax backward, and the block-mean backward fused with the
sparse gradients. The per-stage functions are the formulas the per-kernel GPU tests hold the kernels to."""
import math

import torch

from oracle import wan_ref

TILE = 64


def valid_rows(vbs: torch.Tensor) -> torch.Tensor:
    """bool [64 * nblk]: row r of the padded layout is a token."""
    return (torch.arange(TILE)[None, :] < vbs.cpu().long()[:, None]).reshape(-1)


def token_keep(block_map: torch.Tensor, vbs: torch.Tensor) -> torch.Tensor:
    """[B, H, nblk, nblk] block map -> [B, H, S, S] token mask: the block map, valid keys, valid queries."""
    keep = wan_ref.block_keep_mask(block_map, vbs, TILE)
    return keep & valid_rows(vbs).to(keep.device)[None, None, :, None]


def masked_softmax(s: torch.Tensor, keep: torch.Tensor) -> torch.Tensor:
    """softmax over the kept entries of each row; rows without any kept entry give 0 (and no gradient)."""
    p = torch.softmax(s.masked_fill(~keep, float("-inf")), -1)
    return p.masked_fill(~keep.any(-1, keepdim=True), 0.0)


def block_mean(x: torch.Tensor, vbs: torch.Tensor) -> torch.Tensor:
    """fused_block_mean: sum over the (zero padded) tile in fp32 (fp64 for fp64 input) / valid count -> x's dtype."""
    B, H, S, D = x.shape
    acc = torch.float64 if x.dtype == torch.float64 else torch.float32
    xs = x.to(acc).view(B, H, S // TILE, TILE, D).sum(3)
    return (xs / vbs.to(x.device, acc).view(1, 1, -1, 1)).to(x.dtype)


def composite(q, k, v, gate, vbs, block_map):
    """[B, H, S, D] q, k, v (and gate or None) -> out [B, H, S, D] in the inputs' dtype, differentiable by torch."""
    B, H, S, D = q.shape
    m = valid_rows(vbs).to(q.device, q.dtype)[None, None, :, None]
    q, k, v = q * m, k * m, v * m
    q_c, k_c, v_c = block_mean(q, vbs), block_mean(k, vbs), block_mean(v, vbs)
    attn = torch.softmax(q_c @ k_c.transpose(-1, -2) / math.sqrt(D), -1)
    out_c = (attn @ v_c).repeat_interleave(TILE, 2)
    p = masked_softmax((q @ k.transpose(-1, -2)) * D ** -0.5, token_keep(block_map, vbs).to(q.device))
    out_s = p @ v
    out = out_c * gate + out_s if gate is not None else out_c + out_s
    return out * m


# ------------------------------------------------------------------------------------------- the kernels' formulas
def combine_bwd(dO, out_c, gate, vbs):
    """fvb_vsa_combine_bwd on [B, H, S, D] dO / gate and [B, H, nblk, D] out_c, in the inputs' dtype:
    (d_gate = dO * out_c on the valid rows, 0 on pad rows (None without a gate); d_out_c = per-tile sum of dO * gate over
    the valid rows)."""
    B, H, S, D = dO.shape
    m = valid_rows(vbs).to(dO.device, dO.dtype)[None, None, :, None]
    g = dO * m if gate is None else dO * gate * m
    d_out_c = g.view(B, H, S // TILE, TILE, D).sum(3)
    d_gate = None if gate is None else dO * out_c.repeat_interleave(TILE, 2) * m
    return d_gate, d_out_c


def softmax_rows_bwd(p, dp, scale=1.0):
    """fvb_softmax_rows_bwd: p * (dp - rowsum(dp * p)) * scale."""
    return p * (dp - (dp * p).sum(-1, keepdim=True)) * scale


def block_mean_bwd(dx_s, d_mean, vbs):
    """fvb_block_mean_bwd on [B, H, S, D] dx_s and [B, H, nblk, D] d_mean: dx_s + d_mean / len on valid rows, 0 on pad rows."""
    m = valid_rows(vbs).to(dx_s.device, dx_s.dtype)[None, None, :, None]
    return (dx_s + (d_mean / vbs.to(dx_s.device, dx_s.dtype).view(1, 1, -1, 1)).repeat_interleave(TILE, 2)) * m


def sparse_bwd(q, k, v, dO, keep, scale):
    """Backward of the block-sparse branch by its flash-attention formulas (fvb_attention_blocklist_bwd), dense here."""
    p = masked_softmax((q @ k.transpose(-1, -2)) * scale, keep)
    o = p @ v
    delta = (dO * o).sum(-1, keepdim=True)
    ds = p * (dO @ v.transpose(-1, -2) - delta) * scale
    return ds @ k, ds.transpose(-1, -2) @ q, p.transpose(-1, -2) @ dO


def backward(q, k, v, gate, vbs, block_map, dO):
    """(dq, dk, dv, d_gate or None) of `composite` by the stage formulas, in the inputs' dtype."""
    B, H, S, D = q.shape
    m = valid_rows(vbs).to(q.device, q.dtype)[None, None, :, None]
    q, k, v = q * m, k * m, v * m
    q_c, k_c, v_c = block_mean(q, vbs), block_mean(k, vbs), block_mean(v, vbs)
    attn = torch.softmax(q_c @ k_c.transpose(-1, -2) / math.sqrt(D), -1)
    out_c = attn @ v_c
    dq_s, dk_s, dv_s = sparse_bwd(q, k, v, dO * m, token_keep(block_map, vbs).to(q.device), D ** -0.5)
    d_gate, d_out_c = combine_bwd(dO, out_c, gate, vbs)
    d_attn = d_out_c @ v_c.transpose(-1, -2)
    d_v_c = attn.transpose(-1, -2) @ d_out_c
    d_scores = softmax_rows_bwd(attn, d_attn, D ** -0.5)
    d_q_c = d_scores @ k_c
    d_k_c = d_scores.transpose(-1, -2) @ q_c
    return (block_mean_bwd(dq_s, d_q_c, vbs), block_mean_bwd(dk_s, d_k_c, vbs), block_mean_bwd(dv_s, d_v_c, vbs), d_gate)
