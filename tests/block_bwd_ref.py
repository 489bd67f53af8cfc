"""Restatements of the Wan block backward kernels (include/fvb200.h): fvb_linear_dgrad_gelu_bf16, fvb_resid_gate_bwd,
fvb_layernorm_modulate_bwd and fvb_rmsnorm_rope_bwd. With bf16_points=True the kernels' roundings are applied (fp32
arithmetic, bf16 where the kernel rounds); otherwise the formulas are evaluated exactly in the inputs' dtype (fp64 in
tests/test_block_bwd_cpu.py, against torch autograd)."""
import math

import torch

from rmsnorm_bwd_ref import rmsnorm_bwd


def _rnd(bf16_points):
    return (lambda t: t.bfloat16().float()) if bf16_points else (lambda t: t)


def gelu_tanh_grad(h):
    k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
    t = torch.tanh(k0 * (h + k1 * h ** 3))
    return 0.5 * (1 + t) + 0.5 * h * (1 - t * t) * k0 * (1 + 3 * k1 * h * h)


def linear_dgrad_gelu(dy, w, h, bf16_points=False):
    """dh = bf16(bf16(dy @ w) * gelu_tanh'(h)); dy [M, N], w [N, K], h [M, K]."""
    rnd = _rnd(bf16_points)
    if bf16_points:
        dy, w, h = dy.double(), w.double(), h.float()
    a = rnd(dy @ w)
    if bf16_points:
        a = a.float()
    dh = a * gelu_tanh_grad(h)
    return dh.bfloat16() if bf16_points else dh


def resid_gate_bwd(dout, y, gate, bf16_points=False):
    """out = resid + y * gate[n]: (dy = bf16(dout * gate), d_gate = sum_m dout * y, db = bf16(sum_m dy))."""
    rnd = _rnd(bf16_points)
    if bf16_points:
        dout, y = dout.double(), y.double()
        gate = gate.double()
    dy = rnd((dout * gate).float() if bf16_points else dout * gate)
    d_gate = (dout * y).sum(0)
    db = dy.double().sum(0) if bf16_points else dy.sum(0)
    if bf16_points:
        return dy.bfloat16(), d_gate.float(), db.bfloat16()
    return dy, d_gate, db


def layernorm_modulate_bwd(x, dn, gain, gain_is_scale, round_ln=False, gin=None, eps=1e-6, bf16_points=False):
    """n = t * g + offset, t = LN(x) (t rounded to bf16 first with round_ln), g = 1 + scale or the affine weight.
    Returns (dx, d_gain = sum_m dn * t, d_offset = sum_m dn); dx gets gin added."""
    dt_ = torch.float64 if bf16_points else x.dtype
    xf, dnf, gf = x.to(dt_), dn.to(dt_), gain.to(dt_)
    D = x.shape[-1]
    mean = xf.mean(-1, keepdim=True)
    var = ((xf - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = (xf - mean) * rstd
    g = 1 + gf if gain_is_scale else gf
    dt = dnf * g
    dx = rstd * (dt - dt.mean(-1, keepdim=True) - xh * (dt * xh).mean(-1, keepdim=True))
    if gin is not None:
        dx = dx + gin.to(dt_)
    t = xh.float().bfloat16().to(dt_) if round_ln else xh
    d_gain, d_off = (dnf * t).sum(0), dnf.sum(0)
    if bf16_points:
        dx = dx.float() if x.dtype == torch.float32 else dx.bfloat16()
        return dx, d_gain.float(), d_off.float()
    return dx, d_gain, d_off


def rope_transpose(dy, cos, sin, bf16_points=False):
    """dn = R^T dy for the interleaved-pair rotation of rmsnorm_rope_ (o[2i] = n[2i] c[2i] - n[2i+1] s[2i],
    o[2i+1] = n[2i+1] c[2i+1] + n[2i] s[2i+1]); cos / sin [M, D] (the table rows tiled over the heads)."""
    if bf16_points:
        dy, cos, sin = dy.float(), cos.float(), sin.float()
    d0, d1 = dy[..., 0::2], dy[..., 1::2]
    dn = torch.empty_like(dy)
    dn[..., 0::2] = d0 * cos[..., 0::2] + d1 * sin[..., 1::2]
    dn[..., 1::2] = d1 * cos[..., 1::2] - d0 * sin[..., 0::2]
    return dn.bfloat16() if bf16_points else dn


def rmsnorm_rope_bwd(x, w, dy, cos, sin, eps, bf16_points=False):
    """fvb_rmsnorm_rope_bwd for one tensor: (dx, dw), cos / sin [M, D]."""
    return rmsnorm_bwd(x, w, rope_transpose(dy, cos, sin, bf16_points), eps, bf16_points)
