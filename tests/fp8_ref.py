"""Test infrastructure (never imported by the product path): plain-PyTorch CPU restatement of the FP8 (e4m3) linear
arithmetic of include/fvb200.h -- fvb_quantize_fp8_rows and fvb_linear_fp8 -- and of the Wan block / model with their
token-stream linears in FP8.

The block and model restatements are oracle/wan_ref.wan_block / wan_model themselves: while they run, their module-level
`linear` is routed to `linear_fp8` for exactly the weights WanDiTConfig.fp8_linears quantises (to_q/k/v(/gate_compress),
to_out, attn2.to_q, attn2.to_out, ffn.fc_in, ffn.fc_out of each block), matched by tensor identity; every other linear (the
text-side K/V projections, the embedders, proj_out) keeps wan_ref's bf16 F.linear.
"""
from __future__ import annotations

import contextlib

import torch

from oracle import wan_ref

E4M3_MAX = 448.0
# keys (relative to a block's prefix) of the linears that run in FP8
TOKEN_LINEARS = ("to_q", "to_k", "to_v", "to_gate_compress", "to_out", "attn2.to_q", "attn2.to_out", "ffn.fc_in", "ffn.fc_out")


def quantize_fp8_rows(x):
    """fvb_quantize_fp8_rows: x [..., K] -> (q float8_e4m3fn [..., K], scale fp32 [...]). amax = max|x| in fp32; amax == 0 ->
    scale 1, q 0; else inv = 448 / amax, q = e4m3_satfinite_rn(x * inv), scale = amax / 448, every op an IEEE fp32
    round-to-nearest one. Tensor / tensor division keeps torch from turning the scalar forms into a reciprocal multiply;
    the clamp is the saturation (torch maps out-of-range values to NaN)."""
    xf = x.float()
    amax = xf.abs().amax(dim=-1)
    nz = amax > 0
    c = torch.full_like(amax, E4M3_MAX)
    inv = torch.where(nz, c / torch.where(nz, amax, c), torch.zeros_like(amax))
    q = (xf * inv.unsqueeze(-1)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    q = torch.where(nz.unsqueeze(-1), q.view(torch.uint8), torch.zeros_like(q.view(torch.uint8))).view(torch.float8_e4m3fn)
    scale = torch.where(nz, amax / c, torch.ones_like(amax))
    return q, scale


def fp8_linear_f32(xq, xs, wq, ws, b=None):
    """fvb_linear_fp8 before the output rounding: ((acc * s_x[m]) * s_w[n]) + bias[n] in fp32, where acc is the sum of the
    e4m3 products. The products and their sum are exact in fp64 (e4m3 products span 2^-18 .. 2^17, so 2^14 terms stay
    inside 53 bits), so acc here is the exact sum rounded once to fp32. Returns (fp32 value, fp64 value without any fp32
    rounding)."""
    acc64 = xq.double() @ wq.double().transpose(-1, -2)
    exact = acc64 * xs.double().unsqueeze(-1) * ws.double()
    y = (acc64.float() * xs.float().unsqueeze(-1)) * ws.float()
    if b is not None:
        y = y + b.float()
        exact = exact + b.double()
    return y, exact


def linear_fp8(x, w, b):
    """F.linear with both operands row-quantised to e4m3 (activations per token, weights per output channel), result rounded
    to x's dtype like F.linear's."""
    xq, xs = quantize_fp8_rows(x)
    wq, ws = quantize_fp8_rows(w)
    y, _ = fp8_linear_f32(xq, xs, wq, ws, b)
    return y.to(x.dtype)


@contextlib.contextmanager
def _token_linears_in_fp8(sd, prefixes):
    fp8_ids = {id(sd[p + n + ".weight"]) for p in prefixes for n in TOKEN_LINEARS if p + n + ".weight" in sd}
    bf16_linear = wan_ref.linear

    def routed(x, w, b):
        return linear_fp8(x, w, b) if id(w) in fp8_ids else bf16_linear(x, w, b)

    wan_ref.linear = routed
    try:
        yield
    finally:
        wan_ref.linear = bf16_linear


def wan_block_fp8(x, ctx, temb6, sd, prefix, *args, **kwargs):
    """oracle/wan_ref.wan_block with its token-stream linears in FP8 (same arguments)."""
    with _token_linears_in_fp8(sd, [prefix]):
        return wan_ref.wan_block(x, ctx, temb6, sd, prefix, *args, **kwargs)


def wan_model_fp8(latents, text, timestep, sd, *args, **kwargs):
    """oracle/wan_ref.wan_model with every block's token-stream linears in FP8 (same arguments)."""
    n = 0
    while f"blocks.{n}.to_q.weight" in sd:
        n += 1
    with _token_linears_in_fp8(sd, [f"blocks.{i}." for i in range(n)]):
        return wan_ref.wan_model(latents, text, timestep, sd, *args, **kwargs)
