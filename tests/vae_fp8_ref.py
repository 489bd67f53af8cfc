"""Test infrastructure (never imported by the product path): plain-PyTorch CPU restatement of the FP8 (e4m3) residual-block
convolutions of the Wan VAE decoder, as include/fvb200.h states them (fvb_conv3d_cl_fp8, the e4m3 norm outputs):

  bound = sqrt(C) * max_c |gamma_c|  (fp32)  -- no WanRMS_norm (+ SiLU) output can exceed it
  q = e4m3_satfinite_rn(v * (448 / bound)),  read back as q * (bound / 448);  bound == 0: q = 0, scale 1
  weights: the bf16 packed weight, one e4m3 scale per output channel (fp8_ref.quantize_fp8_rows)
  y = ((acc * x_scale) * w_scale[n]) + bias[n],  acc = the exact sum of the e4m3 products (fp64 here)

`route_res_convs` runs oracle/vae_ref.decode unchanged with exactly the residual blocks' conv1 / conv2 (matched by tensor
identity) sent to `fp8_causal_conv3d`; every other convolution stays the oracle's fp32 one.
"""
from __future__ import annotations

import contextlib
import re

import torch
import torch.nn.functional as F

from fp8_ref import E4M3_MAX, quantize_fp8_rows
from oracle import vae_ref

RES_CONV = re.compile(r"^decoder\.(mid_block\.resnets|up_blocks\.\d+\.resnets)\.\d+\.conv([12])\.weight$")


def norm_bound(gamma: torch.Tensor) -> float:
    """sqrt(C) * max|gamma| in fp32 (ops.rms_norm_e4m3_bound)."""
    C = gamma.numel()
    return float(torch.tensor(C, dtype=torch.float32).sqrt() * gamma.float().abs().max())


def x_scale(bound: float) -> torch.Tensor:
    """bound / 448 in fp32; 1 when bound == 0."""
    if bound == 0.0:
        return torch.tensor(1.0)
    return torch.tensor(bound, dtype=torch.float32) / torch.tensor(E4M3_MAX, dtype=torch.float32)


def quantize_static(v: torch.Tensor, bound: float) -> torch.Tensor:
    """q = e4m3_satfinite_rn(v * (448 / bound)) with fp32 arithmetic; bound == 0 -> q = 0. (The clamp is the saturation.)"""
    if bound == 0.0:
        return torch.zeros_like(v, dtype=torch.float8_e4m3fn)
    inv = torch.tensor(E4M3_MAX, dtype=torch.float32) / torch.tensor(bound, dtype=torch.float32)
    return (v.float() * inv).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def rms_norm_silu(y: torch.Tensor, gamma: torch.Tensor, silu: bool = True, dim: int = -1) -> torch.Tensor:
    """fvb_rmsnorm_silu_cl in fp32: y / max(||y||, 1e-12) * sqrt(C) * gamma (+ SiLU), over `dim`."""
    y = y.float()
    C = y.shape[dim]
    shape = [1] * y.dim()
    shape[dim] = -1
    n = y.norm(dim=dim, keepdim=True).clamp_min(1e-12)
    v = y / n * torch.tensor(C, dtype=torch.float32).sqrt() * gamma.float().reshape(shape)
    return F.silu(v) if silu else v


def norm_e4m3(y: torch.Tensor, gamma: torch.Tensor, bound: float, silu: bool = True) -> torch.Tensor:
    """fvb_rmsnorm_silu_cl_e4m3: the channels-last norm of y written as e4m3 against bound."""
    return quantize_static(rms_norm_silu(y, gamma, silu), bound)


def quantize_conv_weight(w: torch.Tensor):
    """[Cout, Cin, kt, kh, kw] -> (q e4m3, same shape; scale fp32 [Cout]): the bf16 weight, one scale per output channel
    (the packed [Cout, taps * Cin_pad] rows of the kernel hold the same values plus zeros)."""
    Cout = w.shape[0]
    q, s = quantize_fp8_rows(w.bfloat16().float().reshape(Cout, -1))
    return q.view(w.shape), s


def fp8_conv3d_exact(xq: torch.Tensor, xs, wq: torch.Tensor, ws: torch.Tensor, bias=None, t_pad: int | None = None):
    """The FP8 convolution with exact accumulation (fp64) on channels-first e4m3 input xq [B, Cin, T, H, W]: causal zero
    padding of t_pad frames (default kt - 1), "same" spatial padding. Returns fp64 ((acc * xs) * ws + bias)."""
    kt, kh, kw = wq.shape[2:]
    t_pad = kt - 1 if t_pad is None else t_pad
    x = F.pad(xq.double(), (kw // 2, kw // 2, kh // 2, kh // 2, t_pad, 0))
    acc = F.conv3d(x, wq.double())
    y = acc * float(xs) * ws.double().reshape(1, -1, 1, 1, 1)
    if bias is not None:
        y = y + bias.double().reshape(1, -1, 1, 1, 1)
    return y


def fp8_causal_conv3d(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, bound: float) -> torch.Tensor:
    """vae_ref.causal_conv3d with e4m3 operands: x (a norm + SiLU output, channels-first) quantised against the static
    bound, w per output channel; exact accumulation; fp32 result."""
    xq = quantize_static(x, bound)
    wq, ws = quantize_conv_weight(w)
    return fp8_conv3d_exact(xq, x_scale(bound), wq, ws, b).float()


def res_conv_bounds(sd: dict) -> dict:
    """{id(weight): bound of the norm that feeds it} for conv1 / conv2 of every decoder residual block."""
    out = {}
    for k, w in sd.items():
        m = RES_CONV.match(k)
        if m:
            g = sd[k[: -len(f"conv{m.group(2)}.weight")] + f"norm{m.group(2)}.gamma"]
            out[id(w)] = norm_bound(g.reshape(-1))
    return out


@contextlib.contextmanager
def route_res_convs(sd: dict):
    """While active, vae_ref.causal_conv3d sends exactly the residual blocks' conv1 / conv2 of `sd` to fp8_causal_conv3d.
    Yields the list of routed weight keys' ids, one entry per call."""
    bounds = res_conv_bounds(sd)
    hits = []
    orig = vae_ref.causal_conv3d

    def conv(x, w, b):
        if id(w) in bounds:
            hits.append(id(w))
            return fp8_causal_conv3d(x, w, b, bounds[id(w)])
        return orig(x, w, b)

    vae_ref.causal_conv3d = conv
    try:
        yield hits
    finally:
        vae_ref.causal_conv3d = orig


def decode_fp8(z, sd, dim_mult=(1, 2, 4, 4), num_res_blocks=2, temperal_downsample=(False, True, True)):
    """oracle/vae_ref.decode with the residual-block convolutions in FP8."""
    with route_res_convs(sd):
        return vae_ref.decode(z, sd, dim_mult, num_res_blocks, temperal_downsample)


def real_width_state_dict(seed: int = 1, base: int = 96, mult=(1, 2, 4, 4), nrb: int = 2, tds=(False, True, True)):
    """Random decoder weights at the real channel widths (base_dim 96: 384 / 192 / 96), bf16-representable fp32, the same
    construction as the real-width bf16 decoder test. Returns (sd, generator) -- draw z from the generator."""
    g = torch.Generator().manual_seed(seed)
    dims = [base * u for u in [mult[-1]] + list(mult[::-1])]
    sd = {}

    def conv(name, co, ci, k):
        fan = ci * k[0] * k[1] * k[2]
        sd[name + ".weight"] = (torch.randn(co, ci, *k, generator=g) * (1.5 / fan ** 0.5)).bfloat16().float()
        sd[name + ".bias"] = (0.1 * torch.randn(co, generator=g)).bfloat16().float()

    def res(p, ci, co):
        sd[p + "norm1.gamma"] = (1 + 0.2 * torch.randn(ci, 1, 1, 1, generator=g)).bfloat16().float()
        sd[p + "norm2.gamma"] = (1 + 0.2 * torch.randn(co, 1, 1, 1, generator=g)).bfloat16().float()
        conv(p + "conv1", co, ci, (3, 3, 3))
        conv(p + "conv2", co, co, (3, 3, 3))
        if ci != co:
            conv(p + "conv_shortcut", co, ci, (1, 1, 1))

    conv("post_quant_conv", 16, 16, (1, 1, 1))
    conv("decoder.conv_in", dims[0], 16, (3, 3, 3))
    res("decoder.mid_block.resnets.0.", dims[0], dims[0])
    res("decoder.mid_block.resnets.1.", dims[0], dims[0])
    sd["decoder.mid_block.attentions.0.norm.gamma"] = (1 + 0.2 * torch.randn(dims[0], 1, 1, generator=g)).bfloat16().float()
    for n, co in (("to_qkv", 3 * dims[0]), ("proj", dims[0])):
        sd[f"decoder.mid_block.attentions.0.{n}.weight"] = (torch.randn(co, dims[0], 1, 1, generator=g) / dims[0] ** 0.5).bfloat16().float()
        sd[f"decoder.mid_block.attentions.0.{n}.bias"] = (0.1 * torch.randn(co, generator=g)).bfloat16().float()
    t_up = list(tds)[::-1]
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        if i > 0:
            ci = ci // 2
        cur = ci
        for j in range(nrb + 1):
            res(f"decoder.up_blocks.{i}.resnets.{j}.", cur, co)
            cur = co
        if i != len(mult) - 1:
            p = f"decoder.up_blocks.{i}.upsamplers.0."
            sd[p + "resample.1.weight"] = (torch.randn(co // 2, co, 3, 3, generator=g) * (1.5 / (9 * co) ** 0.5)).bfloat16().float()
            sd[p + "resample.1.bias"] = (0.1 * torch.randn(co // 2, generator=g)).bfloat16().float()
            if t_up[i]:
                conv(p + "time_conv", 2 * co, co, (3, 1, 1))
    sd["decoder.norm_out.gamma"] = (1 + 0.2 * torch.randn(dims[-1], 1, 1, 1, generator=g)).bfloat16().float()
    conv("decoder.conv_out", 3, dims[-1], (3, 3, 3))
    return sd, g
