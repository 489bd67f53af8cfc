"""Test infrastructure (never imported by the product path): plain-PyTorch CPU restatement of the 8-bit attention arithmetic
of include/fvb200.h -- fvb_attention_8bit_quantize (including the vt8 layout and its key-slot permutation) and
fvb_attention_8bit_fwd (the same 64-key tile walk, running max, P quantisation and per-tile promotion) -- and of the Wan block /
model with their self-attention on it.

The block and model restatements are oracle/wan_ref.wan_block / wan_model themselves: while they run, only the self-attention
call of each block goes to `attention_8bit_bshd` (dense blocks), or the sparse branch of the VSA composite goes to the 8-bit
restatement (VSA blocks); cross-attention and the VSA compression branch keep the oracle's own attention.
"""
from __future__ import annotations

import contextlib

import torch

from oracle import wan_ref

E4M3_MAX = 448.0
LOG2E = 1.4426950408889634
# slot j of every 16-key group of a vt8 row holds key PERM16[j] of that group
PERM16 = [2 * (j >> 2) + (j & 1) + 8 * ((j >> 1) & 1) for j in range(16)]
SLOT_KEY = [16 * (j >> 4) + PERM16[j & 15] for j in range(64)]


def kv_blocks(Skv, kv_off=None, kv_len=None, nkb=None):
    """[(first row, valid keys)] of every key block, as the kernels derive them."""
    if kv_off is None:
        nkb = (Skv + 63) // 64 if nkb is None else nkb
    elif nkb is None:
        nkb = len(kv_off) - 1
    out = []
    for i in range(nkb):
        row0 = int(kv_off[i]) if kv_off is not None else 64 * i
        if kv_len is not None:
            vlen = int(kv_len[i])
        elif kv_off is not None:
            vlen = min(64, int(kv_off[i + 1]) - row0)
        else:
            vlen = 64
        out.append((row0, max(0, min(vlen, 64, Skv - row0))))
    return out


def q_blocks(Sq, nqb=None, q_off=None, q_len=None):
    """[(first row, rows)] of every 64-row q block (dense: nqb None)."""
    if nqb is None:
        return [(64 * i, min(64, Sq - 64 * i)) for i in range((Sq + 63) // 64)]
    out = []
    for i in range(nqb):
        row0 = int(q_off[i]) if q_off is not None else 64 * i
        n = int(q_len[i]) if q_len is not None else (int(q_off[i + 1]) - row0 if q_off is not None else 64)
        out.append((row0, max(0, min(n, 64, Sq - row0))))
    return out


def quantize_rows_int8(x):
    """fp32 [..., 128] -> (int8 [..., 128], fp32 scale [...]): amax == 0 -> scale 1, row 0; else inv = 127 / amax,
    clamp(rint(x * inv), -127, 127), scale = amax / 127 (tensor / tensor division: IEEE fp32 round-to-nearest)."""
    amax = x.abs().amax(dim=-1)
    nz = amax > 0
    c = torch.full_like(amax, 127.0)
    inv = torch.where(nz, c / torch.where(nz, amax, c), torch.zeros_like(amax))
    q = torch.round(x * inv.unsqueeze(-1)).clamp(-127, 127).to(torch.int8)
    q = torch.where(nz.unsqueeze(-1), q, torch.zeros_like(q))
    return q, torch.where(nz, amax / c, torch.ones_like(amax))


def quantize(q, k, v, kv_off=None, kv_len=None, nkb=None, k_mean=None):
    """fvb_attention_8bit_quantize on CPU. q [B, Sq, H, 128], k / v [B, Skv, H, 128] (bf16). k_mean: fp32 [B, H, 128] to use
    instead of this function's own (an fp64 mean rounded to fp32) -- pass the kernel's to compare the rest bit for bit.
    Returns a dict: q8, q_scale, k8, k_scale, k_mean, v8 (e4m3 [B, H, Skv, 128], key order), vt8 (uint8
    [B, H, nkb, 128, 64]), v_scale, blocks."""
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    qf = q.float().transpose(1, 2)  # [B, H, S, d]
    kf = k.float().transpose(1, 2)
    vf = v.float().transpose(1, 2)
    if k_mean is None:
        k_mean = kf.double().mean(dim=2).float()
    q8, q_scale = quantize_rows_int8(qf)
    k8, k_scale = quantize_rows_int8(kf - k_mean.unsqueeze(2))
    amax = vf.abs().amax(dim=2)  # [B, H, d]
    nz = amax > 0
    c = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(nz, c / torch.where(nz, amax, c), torch.zeros_like(amax))
    v8 = (vf * inv.unsqueeze(2)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    v8 = torch.where(nz.unsqueeze(2), v8.view(torch.uint8), torch.zeros_like(v8.view(torch.uint8))).view(torch.float8_e4m3fn)
    v_scale = torch.where(nz, amax / c, torch.ones_like(amax))
    blocks = kv_blocks(Skv, kv_off, kv_len, nkb)
    vt8 = torch.zeros((B, H, len(blocks), d, 64), dtype=torch.uint8)
    v8u = v8.view(torch.uint8)
    for i, (row0, vlen) in enumerate(blocks):
        for j, key in enumerate(SLOT_KEY):
            if key < vlen:
                vt8[:, :, i, :, j] = v8u[:, :, row0 + key, :]
    return dict(q8=q8, q_scale=q_scale, k8=k8, k_scale=k_scale, k_mean=k_mean, v8=v8, vt8=vt8, v_scale=v_scale, blocks=blocks)


def attention(qz, softmax_scale, q2k_idx=None, q2k_num=None, q_off=None, q_len=None, p_e4m3=True):
    """fvb_attention_8bit_fwd on CPU from `quantize`'s dict -> fp32 [B, Sq, H, 128] (before the bf16 rounding; rows the
    kernel does not write are 0). Dense: every key block; otherwise per-q-block lists [B or 1, H or 1, nqb, cap].
    p_e4m3=False keeps P unquantised (the error of the e4m3 P alone is then what the comparison omits)."""
    q8, k8, v8 = qz["q8"], qz["k8"], qz["v8"]
    B, H, Sq, d = q8.shape
    blocks = qz["blocks"]
    nqb = None if q2k_idx is None else q2k_idx.shape[2]
    qbl = q_blocks(Sq, nqb, q_off, q_len)
    c = torch.tensor(softmax_scale * LOG2E, dtype=torch.float32)
    out = torch.zeros((B, Sq, H, d), dtype=torch.float32)
    for b in range(B):
        for h in range(H):
            for qi, (r0, nr) in enumerate(qbl):
                if nr <= 0:
                    continue
                if q2k_idx is None:
                    tiles = range(len(blocks))
                else:
                    ib, ih = min(b, q2k_idx.shape[0] - 1), min(h, q2k_idx.shape[1] - 1)
                    tiles = [int(t) for t in q2k_idx[ib, ih, qi, :int(q2k_num[ib, ih, qi])]]
                qq = q8[b, h, r0:r0 + nr].double()
                sq = qz["q_scale"][b, h, r0:r0 + nr]
                m = torch.full((nr,), float("-inf"))
                l = torch.zeros(nr)
                O = torch.zeros((nr, d))
                for t in tiles:
                    row0, vlen = blocks[t]
                    if vlen <= 0:
                        x = torch.full((nr, 64), float("-inf"))
                        vt = torch.zeros((64, d))
                    else:
                        acc = (qq @ k8[b, h, row0:row0 + vlen].double().T).float()  # exact integers
                        x = acc * sq[:, None] * qz["k_scale"][b, h, row0:row0 + vlen][None, :] * c
                        x = torch.cat([x, torch.full((nr, 64 - vlen), float("-inf"))], 1)
                        vt = torch.cat([v8[b, h, row0:row0 + vlen].float(), torch.zeros((64 - vlen, d))], 0)
                    m_new = torch.maximum(m, x.amax(1))
                    m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
                    alpha = torch.exp2(m - m_use)
                    p = torch.exp2(x - m_use[:, None])
                    l = l * alpha + p.sum(1)
                    m = m_new
                    p8 = (p * E4M3_MAX).to(torch.float8_e4m3fn).float() if p_e4m3 else p * E4M3_MAX
                    T = (p8.double() @ vt.double()).float()
                    O = O * alpha[:, None] + T
                inv = torch.where(l > 0, 1.0 / (E4M3_MAX * l), torch.zeros_like(l))
                out[b, r0:r0 + nr, h] = (O * qz["v_scale"][b, h][None, :]) * inv[:, None]
    return out


def attention_8bit_bshd(q, k, v, scale=None, **kw):
    """The whole 8-bit path, dense keys: quantize + attention, rounded to q's dtype. q/k/v BSHD."""
    scale = scale if scale is not None else q.shape[-1] ** -0.5
    return attention(quantize(q, k, v), scale, **kw).to(q.dtype)


def exact_attention(q, k, v, scale=None, q2k_idx=None, q2k_num=None, q_off=None, q_len=None, kv_off=None, kv_len=None):
    """fp64 softmax(q k^T * scale) v on the unquantised inputs, same blocks / lists / masking / empty rows."""
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    scale = scale if scale is not None else d ** -0.5
    blocks = kv_blocks(Skv, kv_off, kv_len, None if kv_off is None else len(kv_off) - 1)
    nqb = None if q2k_idx is None else q2k_idx.shape[2]
    qbl = q_blocks(Sq, nqb, q_off, q_len)
    out = torch.zeros((B, Sq, H, d), dtype=torch.float64)
    for b in range(B):
        for h in range(H):
            for qi, (r0, nr) in enumerate(qbl):
                if nr <= 0:
                    continue
                if q2k_idx is None:
                    tiles = range(len(blocks))
                else:
                    ib, ih = min(b, q2k_idx.shape[0] - 1), min(h, q2k_idx.shape[1] - 1)
                    tiles = [int(t) for t in q2k_idx[ib, ih, qi, :int(q2k_num[ib, ih, qi])]]
                keys = torch.tensor([r + j for t in tiles for r, n in [blocks[t]] for j in range(n)], dtype=torch.long)
                if keys.numel() == 0:
                    continue
                s = (q[b, r0:r0 + nr, h].double() @ k[b, keys, h].double().T) * scale
                out[b, r0:r0 + nr, h] = torch.softmax(s, -1) @ v[b, keys, h].double()
    return out


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ----------------------------------------------------------------------------------------------- Wan block / model
def _vsa_attn8(q, k, v, vbs, topk, gate=None, block: int = 64, return_aux: bool = False):
    """wan_ref.video_sparse_attn with the sparse branch on the 8-bit restatement. The padded tiles are compacted first
    (the engine's token order), so the K mean and the scales cover exactly the valid keys."""
    B, H, S, D = q.shape
    q_c, k_c, v_c = (wan_ref.block_mean(t, vbs, block) for t in (q, k, v))
    scores = torch.matmul(q_c, k_c.transpose(-2, -1)) / (D ** 0.5)
    attn = torch.softmax(scores, dim=-1)
    out_c = torch.matmul(attn, v_c)
    out_c_full = out_c.view(B, H, S // block, 1, D).repeat(1, 1, 1, block, 1).view(B, H, S, D)
    mask = wan_ref.topk_mask(scores, topk)
    nblk = vbs.numel()
    rows = torch.cat([torch.arange(block * i, block * i + int(vbs[i])) for i in range(nblk)])
    off = torch.cat([torch.zeros(1, dtype=torch.int64), vbs.long().cumsum(0)]).to(torch.int32)
    cq, ck, cv = (t.transpose(1, 2)[:, rows] for t in (q, k, v))  # compact BSHD
    idx = torch.full((B, H, nblk, nblk), -1, dtype=torch.int32)
    num = mask.sum(-1).to(torch.int32)
    for b in range(B):
        for h in range(H):
            for i in range(nblk):
                sel = mask[b, h, i].nonzero().flatten()
                idx[b, h, i, :sel.numel()] = sel.to(torch.int32)
    qz = quantize(cq, ck, cv, kv_off=off, kv_len=vbs, nkb=nblk)
    o_s = attention(qz, D ** -0.5, idx, num, q_off=off, q_len=vbs).to(q.dtype)
    out_s = torch.zeros((B, S, H, D), dtype=q.dtype)
    out_s[:, rows] = o_s
    out_s = out_s.transpose(1, 2)
    return out_c_full * gate + out_s if gate is not None else out_c_full + out_s


class _SelfAttentionRouter:
    """attn_fn for wan_ref.wan_block: the first call after arm() (the block's self-attention) goes to the 8-bit restatement,
    every other call (cross-attention) to the oracle's sdpa."""

    def __init__(self):
        self.armed = False

    def arm(self):
        self.armed = True

    def __call__(self, q, k, v):
        if self.armed:
            self.armed = False
            return attention_8bit_bshd(q, k, v)
        return wan_ref.sdpa(q, k, v)


@contextlib.contextmanager
def _self_attention_in_8bit():
    block, vsa = wan_ref.wan_block, wan_ref.video_sparse_attn
    router = _SelfAttentionRouter()

    def routed_block(x, ctx, temb6, sd, prefix, num_heads, cos, sin, eps=1e-6, attn_fn=None, vsa_meta=None):
        if vsa_meta is None:
            router.arm()
        return block(x, ctx, temb6, sd, prefix, num_heads, cos, sin, eps, router, vsa_meta)

    wan_ref.wan_block, wan_ref.video_sparse_attn = routed_block, _vsa_attn8
    try:
        yield
    finally:
        wan_ref.wan_block, wan_ref.video_sparse_attn = block, vsa


def wan_block_attn8(*args, **kwargs):
    """oracle/wan_ref.wan_block with its self-attention on the 8-bit restatement (same arguments; attn_fn is ignored)."""
    kwargs.pop("attn_fn", None)
    with _self_attention_in_8bit():
        return wan_ref.wan_block(*args, **kwargs)


def wan_model_attn8(*args, **kwargs):
    """oracle/wan_ref.wan_model with every block's self-attention on the 8-bit restatement (same arguments)."""
    kwargs.pop("attn_fn", None)
    with _self_attention_in_8bit():
        return wan_ref.wan_model(*args, **kwargs)
