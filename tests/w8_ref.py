"""Test infrastructure (never imported by the product path): plain-PyTorch CPU restatement of the INT8 weight-only linear
arithmetic of include/fvb200.h -- the load-time quantiser and fvb_linear_w8_sp -- and of the Wan block / model and the
causal block / model with their block linears on INT8 weights.

The block and model restatements are the oracles themselves (oracle/wan_ref.wan_block / wan_model, oracle/causal_ref.
causal_block / causal_model_inference): while they run, their module-level linear (`wan_ref.linear`, `causal_ref._lin`) is
routed to `linear_w8` for exactly the weights WanDiTConfig.int8_weights quantises (every linear of a block: to_q/k/v
(/gate_compress), to_out, attn2.to_q/k/v, attn2.add_k_proj/add_v_proj, attn2.to_out, ffn.fc_in, ffn.fc_out), matched by
tensor identity; the embedders, patch embedding and proj_out keep the oracle's own F.linear.

Everything works on bf16 inputs (the bf16 restatement, output rounded to bf16 like F.linear's) and on fp32 inputs (the fp32
restatement: the same int8 weights, no output rounding), so a result can be held to the usual bf16 parity gate.
"""
from __future__ import annotations

import contextlib

import torch

from oracle import causal_ref, wan_ref

# keys (relative to a block's prefix) of the linears that run on INT8 weights
BLOCK_LINEARS = ("to_q", "to_k", "to_v", "to_gate_compress", "to_out", "attn2.to_q", "attn2.to_k", "attn2.to_v",
                 "attn2.add_k_proj", "attn2.add_v_proj", "attn2.to_out", "ffn.fc_in", "ffn.fc_out")


def quantize_int8_rows(w):
    """The load-time quantiser (ops.Int8Weight.quantize): w [N, K] -> (q int8 [N, K], scale fp32 [N]).
    amax = max|w[n]| (fp32); amax == 0 -> scale 1, q 0; else scale = amax / 127, q = clamp(rint(w * (127 / amax)), -127, 127),
    every op an IEEE fp32 round-to-nearest one (tensor / tensor division, so torch does not turn it into a reciprocal
    multiply). The row rule of attn8_ref.quantize_rows_int8 applied to K-wide rows."""
    wf = w.float()
    amax = wf.abs().amax(dim=-1)
    nz = amax > 0
    c = torch.full_like(amax, 127.0)
    one = torch.ones_like(amax)
    inv = torch.where(nz, c / torch.where(nz, amax, one), one)
    q = torch.clamp(torch.round(wf * inv.unsqueeze(-1)), -127, 127).to(torch.int8)
    q = torch.where(nz.unsqueeze(-1), q, torch.zeros_like(q))
    scale = torch.where(nz, amax / c, one)
    return q, scale


def w8_linear_f32(x, q, s, b=None):
    """fvb_linear_w8_sp before the output rounding: (fp32(acc) * s[n]) + b[n] in fp32, acc = sum_k x[m, k] * q[n, k] in
    fp64 (the bf16 x int8 products are exact; so is their sum at these K). Returns (fp32 value, fp64 value)."""
    acc64 = x.double() @ q.double().transpose(-1, -2)
    exact = acc64 * s.double()
    y = acc64.float() * s.float()
    if b is not None:
        y = y + b.float()
        exact = exact + b.double()
    return y, exact


def linear_w8(x, q, s, b):
    """F.linear with int8 weights q [N, K] and scales s [N]; result in x's dtype (bf16 inputs: rounded once, like the
    kernel's bf16(acc * s + b); fp32 inputs: the fp32 value)."""
    y, _ = w8_linear_f32(x, q, s, b)
    return y.to(x.dtype)


def _int8_ids(sd, prefixes):
    return {id(sd[p + n + ".weight"]) for p in prefixes for n in BLOCK_LINEARS if p + n + ".weight" in sd}


def _routed(ids, fallback):
    cache = {}

    def lin(x, w, b):
        if id(w) not in ids:
            return fallback(x, w, b)
        if id(w) not in cache:
            cache[id(w)] = quantize_int8_rows(w.to(torch.bfloat16))  # the engine quantises the bf16 weight
        q, s = cache[id(w)]
        return linear_w8(x, q, s, b)
    return lin


@contextlib.contextmanager
def _wan_block_linears_in_int8(sd, prefixes):
    bf16_linear = wan_ref.linear
    wan_ref.linear = _routed(_int8_ids(sd, prefixes), bf16_linear)
    try:
        yield
    finally:
        wan_ref.linear = bf16_linear


@contextlib.contextmanager
def _causal_block_linears_in_int8(sd, prefixes):
    lin = causal_ref._lin
    routed = _routed(_int8_ids(sd, prefixes), lin)
    causal_ref._lin = lambda x, w, b: routed(x.to(w.dtype), w, b)  # _lin casts the activation to the weight dtype
    try:
        yield
    finally:
        causal_ref._lin = lin


def _layers(sd):
    n = 0
    while f"blocks.{n}.to_q.weight" in sd:
        n += 1
    return [f"blocks.{i}." for i in range(n)]


def wan_block_w8(x, ctx, temb6, sd, prefix, *args, **kwargs):
    """oracle/wan_ref.wan_block with its linears on INT8 weights (same arguments)."""
    with _wan_block_linears_in_int8(sd, [prefix]):
        return wan_ref.wan_block(x, ctx, temb6, sd, prefix, *args, **kwargs)


def wan_model_w8(latents, text, timestep, sd, *args, **kwargs):
    """oracle/wan_ref.wan_model with every block's linears on INT8 weights (same arguments)."""
    with _wan_block_linears_in_int8(sd, _layers(sd)):
        return wan_ref.wan_model(latents, text, timestep, sd, *args, **kwargs)


def causal_block_w8(x, ctx, temb, sd, prefix, *args, **kwargs):
    """oracle/causal_ref.causal_block with its linears on INT8 weights (same arguments)."""
    with _causal_block_linears_in_int8(sd, [prefix]):
        return causal_ref.causal_block(x, ctx, temb, sd, prefix, *args, **kwargs)


def causal_model_w8(latents, text, timestep, sd, *args, **kwargs):
    """oracle/causal_ref.causal_model_inference with every block's linears on INT8 weights (same arguments)."""
    with _causal_block_linears_in_int8(sd, _layers(sd)):
        return causal_ref.causal_model_inference(latents, text, timestep, sd, *args, **kwargs)
