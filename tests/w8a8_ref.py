"""Test infrastructure (never imported by the product path): plain-PyTorch CPU restatement of the W8A8 INT8 linear arithmetic
of include/fvb200.h -- fvb_quantize_int8_rows and fvb_linear_w8a8_sp -- and of the Wan block / model and the causal block /
model with their block linears on int8 weights and int8 activations.

As in tests/w8_ref.py, the block and model restatements are the oracles themselves (oracle/wan_ref, oracle/causal_ref), run
unchanged while their module-level linear is routed to `linear_w8a8` for exactly the weights WanDiTConfig.int8_weights
quantises (matched by tensor identity); the embedders, patch embedding and proj_out keep the oracle's own F.linear.

bf16 inputs give the bf16 restatement (output rounded to bf16 once, like the kernel); fp32 inputs give the fp32 restatement
(the same quantisation rule applied to the fp32 activations, no output rounding).
"""
from __future__ import annotations

import contextlib

import torch

from oracle import causal_ref, wan_ref
from w8_ref import BLOCK_LINEARS, _int8_ids, _layers, quantize_int8_rows  # noqa: F401 (BLOCK_LINEARS re-exported)

# |acc| <= 127^2 K < 2^31 (fvb_linear_w8a8_sp rejects larger K)
MAX_K = 133144


def quantize_rows(x):
    """fvb_quantize_int8_rows on the last dimension (any leading shape): the rule of the load-time weight quantiser,
    amax = max|x[r]|, inv = 127 / amax, q = clamp(rint(x * inv), -127, 127), scale = amax / 127 (amax == 0: scale 1, q 0)."""
    return quantize_int8_rows(x)


def w8a8_acc(xq, q):
    """The exact integer dot products sum_k xq[m, k] * q[n, k] (int64)."""
    return torch.matmul(xq.long(), q.long().transpose(-1, -2))


def w8a8_linear_f32(x, q, s, b=None):
    """fvb_linear_w8a8_sp before the output rounding: ((float(acc) * x_scale[m]) * s[n]) + b[n], each step fp32
    round-to-nearest. Returns (fp32 value, int64 acc, x_scale)."""
    xq, xs = quantize_rows(x)
    acc = w8a8_acc(xq, q)
    assert acc.abs().max().item() < 2 ** 31
    y = (acc.float() * xs.unsqueeze(-1)) * s.float()
    if b is not None:
        y = y + b.float()
    return y, acc, xs


def linear_w8a8(x, q, s, b):
    """F.linear with int8 weights q [N, K] / scales s [N] and int8-quantised activations; result in x's dtype."""
    y, _, _ = w8a8_linear_f32(x, q, s, b)
    return y.to(x.dtype)


def _routed(ids, fallback):
    cache = {}

    def lin(x, w, b):
        if id(w) not in ids:
            return fallback(x, w, b)
        if id(w) not in cache:
            cache[id(w)] = quantize_int8_rows(w.to(torch.bfloat16))  # the engine quantises the bf16 weight
        q, s = cache[id(w)]
        return linear_w8a8(x, q, s, b)
    return lin


@contextlib.contextmanager
def wan_block_linears_in_w8a8(sd, prefixes):
    bf16_linear = wan_ref.linear
    wan_ref.linear = _routed(_int8_ids(sd, prefixes), bf16_linear)
    try:
        yield
    finally:
        wan_ref.linear = bf16_linear


@contextlib.contextmanager
def _causal_block_linears_in_w8a8(sd, prefixes):
    lin = causal_ref._lin
    routed = _routed(_int8_ids(sd, prefixes), lin)
    causal_ref._lin = lambda x, w, b: routed(x.to(w.dtype), w, b)  # _lin casts the activation to the weight dtype
    try:
        yield
    finally:
        causal_ref._lin = lin


def wan_block_w8a8(x, ctx, temb6, sd, prefix, *args, **kwargs):
    """oracle/wan_ref.wan_block with its linears on W8A8 (same arguments)."""
    with wan_block_linears_in_w8a8(sd, [prefix]):
        return wan_ref.wan_block(x, ctx, temb6, sd, prefix, *args, **kwargs)


def wan_model_w8a8(latents, text, timestep, sd, *args, **kwargs):
    """oracle/wan_ref.wan_model with every block's linears on W8A8 (same arguments)."""
    with wan_block_linears_in_w8a8(sd, _layers(sd)):
        return wan_ref.wan_model(latents, text, timestep, sd, *args, **kwargs)


def causal_block_w8a8(x, ctx, temb, sd, prefix, *args, **kwargs):
    """oracle/causal_ref.causal_block with its linears on W8A8 (same arguments)."""
    with _causal_block_linears_in_w8a8(sd, [prefix]):
        return causal_ref.causal_block(x, ctx, temb, sd, prefix, *args, **kwargs)


def causal_model_w8a8(latents, text, timestep, sd, *args, **kwargs):
    """oracle/causal_ref.causal_model_inference with every block's linears on W8A8 (same arguments)."""
    with _causal_block_linears_in_w8a8(sd, _layers(sd)):
        return causal_ref.causal_model_inference(latents, text, timestep, sd, *args, **kwargs)
