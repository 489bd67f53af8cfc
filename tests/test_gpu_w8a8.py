"""GPU: W8A8 INT8 linears -- fvb_quantize_int8_rows and fvb_linear_w8a8_sp held bit for bit to the formulas of include/fvb200.h
(the integer products are exact, so the only roundings are the epilogue's), their sequence-parallel options, and every Wan
path with WanDiTConfig(int8_weights=True, int8_activations=True) against the oracle with exactly the engine's block linears
routed to the restatement (tests/w8a8_ref.py).

The model-level bounds are measured, not derived. The GPU and the restatement share the integer products, but the engine's
bf16 arithmetic upstream of each linear (attention, norms, the fp32 accumulation of the bf16 GEMMs) differs from the CPU
oracle's in the last bits, and such a difference can move an activation across an int8 rounding boundary. Measured on an
H100 80GB HBM3 (700 W), relative L2 from the routed bf16 oracle: dense block 6.0e-3, I2V block 6.0e-3, VSA block 6.7e-3
(median row), dense block with attention_8bit 4.5e-3, 2-layer model 6.4e-3, causal block rollouts <= 6.4e-3 and causal
model rollouts <= 6.7e-3 (worst call, either RoPE cache policy). The bf16 engine sits 3.5-6e-3 from the bf16 oracle on the
same fixtures. Every bound is 1e-2, about 1.5x the largest measured value.
"""
import json
import os
import socket
import subprocess
import sys
from ctypes import c_int, c_int64

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attn8_ref
import w8a8_ref
from conftest import ROOT
from oracle import causal_ref, vsa_index, wan_ref
from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu


def cuda_sd(sd):
    return {k: v.cuda() for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ fvb_quantize_int8_rows
def _ref_rows(x):
    q, s = w8a8_ref.quantize_rows(x.cpu())
    return q.cuda(), s.cuda()


def _bits_equal(q, s, rq, rs):
    return torch.equal(q, rq) and torch.equal(s.view(torch.int32), rs.view(torch.int32))


def test_quantize_int8_rows_bit_exact():
    from fastvideo_b200 import ops
    torch.manual_seed(0)
    # plain, a wide row (register cache overflow), K tails of the 16-byte q rows
    for M, K in ((333, 5120), (7, 13824), (64, 40), (1, 8)):
        x = (torch.randn(M, K, device="cuda") * torch.logspace(-3, 2, M, device="cuda")[:, None]).bfloat16()
        q, s = ops.quantize_int8_rows(x)
        assert q.shape == (M, K) and q.stride(0) % 16 == 0 and q.dtype == torch.int8
        assert _bits_equal(q, s, *_ref_rows(x)), (M, K)
    # strided rows and an all-zero row
    base = torch.randn(50, 1024 + 64, device="cuda").bfloat16()
    base[17] = 0
    x = base[:, 32:32 + 1024]
    q, s = ops.quantize_int8_rows(x)
    assert _bits_equal(q, s, *_ref_rows(x))
    assert s[17].item() == 1.0 and (q[17] == 0).all()
    # ties: amax 127 -> inv 1, x.5 rounds to even
    t = torch.tensor([[127.0, 0.5, 1.5, 2.5, -0.5, -1.5, 126.5, -126.5]], device="cuda").bfloat16()
    q, s = ops.quantize_int8_rows(t)
    assert q[0].tolist() == [127, 0, 2, 2, 0, -2, 126, -126] and s.item() == 1.0


def test_quantize_int8_rows_segmented_equals_gathered():
    """The SP out-projection's A operand: the return buffer [src rank][token][local heads * d] read as one row per token."""
    from fastvideo_b200 import ops
    torch.manual_seed(1)
    world, M, Hl, d = 4, 300, 3, 128
    seg = Hl * d
    back = torch.randn(world, M, seg, device="cuda").bfloat16()
    back[:, 5] = 0  # a token that is zero in every segment
    back[2, 9] *= 100  # a token whose amax sits in one segment only
    gathered = back.permute(1, 0, 2).reshape(M, world * seg).contiguous()
    q, s = ops._quantize_int8_rows_sp(back, M, world * seg, seg, seg, M * seg)
    qp, sp = ops.quantize_int8_rows(gathered)
    assert _bits_equal(q, s, qp, sp)
    assert _bits_equal(q, s, *_ref_rows(gathered))


def test_quantize_int8_rows_rejects_bad_arguments():
    from fastvideo_b200 import ops
    x = torch.randn(4, 100, device="cuda").bfloat16()
    with pytest.raises(ops.FvbError):
        ops.quantize_int8_rows(x[:, :90])  # K % 8 != 0
    with pytest.raises(ops.FvbError):
        ops.quantize_int8_rows(x.float())
    y = torch.randn(4, 96, device="cuda").bfloat16()
    with pytest.raises(ops.FvbError):
        ops._quantize_int8_rows_sp(y, 4, 96, 96, 36, 96)  # segment does not divide K
    with pytest.raises(ops.FvbError):
        ops._quantize_int8_rows_sp(y, 4, 96, 96, 12, 100)  # segment stride not a multiple of 8


# ------------------------------------------------------------------------------------------------ fvb_linear_w8a8_sp
def formula(x, w, b, epi, resid, gate, gate_rows):
    """(fp64 value of the bf16-x linear with the restated int8 operands, the formula with its exact rounding points)."""
    xq, xs = _ref_rows(x)
    # |acc| < 2^31: every partial sum is an integer that fp64 holds exactly, so the fp64 GEMM on the GPU is the exact
    # integer accumulator (checked against int64 on the CPU in test_w8a8_cpu)
    acc = xq.double() @ w.q.double().t()
    exact = acc * xs.double()[:, None] * w.scale.double()[None, :]
    y32 = (acc.float() * xs[:, None]) * w.scale[None, :]
    if b is not None:
        exact = exact + b.double()
        y32 = y32 + b.float()
    y = y32.bfloat16().float()
    if gate is not None:
        g = gate if gate_rows == 0 else gate.repeat_interleave(gate_rows, 0)[: x.shape[0]]
    if epi == 0: return exact, y.bfloat16()
    if epi == 1: return F.gelu(exact, approximate="tanh"), F.gelu(y, approximate="tanh").bfloat16()
    if epi == 2: return resid.double() + exact * g.double(), resid.float() + y * g
    if epi == 3: return resid.double() + exact * g.double(), (resid.float() + y * g).bfloat16()
    if epi == 7: return resid.double() + exact * g.double(), (resid.float() + (y * g).bfloat16().float()).bfloat16()
    if epi == 4: return resid.double() + exact, (resid.float() + y).bfloat16()


def _case(M, N, K, epi, gate_rows):
    from fastvideo_b200 import ops
    torch.manual_seed(M + N + K + epi + gate_rows)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    resid = torch.randn(M, N, device="cuda").bfloat16() if epi >= 2 else None
    gate = None
    if epi in (2, 3, 7):
        gate = torch.randn(N, device="cuda") if gate_rows == 0 else torch.randn((M + gate_rows - 1) // gate_rows, N, device="cuda")
    return x, ops.Int8Weight.quantize(w, int8_activations=True), b, resid, gate


# (M, N, K, epilogue, gate_rows). BN 256: N % 256 == 0 or ragged N >= 192; BN 128: N % 128 == 0 otherwise; BN 64: the rest.
# M = 1 and ragged M, K tails (K % 128 != 0) and K = 13 824.
EXACT_CASES = [(1, 1536, 256, 0, 0), (333, 200, 200, 0, 0), (300, 64, 512, 0, 0), (130, 136, 264, 0, 0),
               (1000, 1152, 1536, 2, 0), (1000, 1152, 1536, 2, 64), (777, 1536, 1536, 3, 0), (777, 1536, 1536, 3, 100),
               (777, 1536, 1536, 7, 0), (777, 1536, 1536, 7, 128), (777, 1536, 1536, 4, 0), (4680, 5120, 5120, 0, 0),
               (4680, 5120, 5120, 7, 1560), (2048, 5120, 13824, 4, 0), (4680, 1000, 5120, 2, 0), (129, 384, 13824, 3, 0)]


@pytest.mark.parametrize("M,N,K,epi,gate_rows", EXACT_CASES)
def test_linear_w8a8_bit_exact(M, N, K, epi, gate_rows):
    from fastvideo_b200 import ops
    x, w, b, resid, gate = _case(M, N, K, epi, gate_rows)
    out = ops.linear_any(x, w, b, epi, resid, gate, gate_rows=gate_rows)
    _, rounded = formula(x, w, b, epi, resid, gate, gate_rows)
    assert out.dtype == (torch.float32 if epi == 2 else torch.bfloat16)
    bad = (out.view(torch.int16 if out.dtype == torch.bfloat16 else torch.int32)
           != rounded.view(torch.int16 if out.dtype == torch.bfloat16 else torch.int32))
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} outputs off the formula"


@pytest.mark.parametrize("M,N,K", [(1000, 1536, 1536), (512, 13824, 5120), (77, 200, 200)])
def test_linear_w8a8_gelu(M, N, K):
    """BIAS_GELU_TANH: the kernel's tanh is not torch's, so bf16 parity against the fp64 value and fewer than 2 % of the
    outputs off the formula's own rounding (test_gpu_fp8's rule)."""
    from fastvideo_b200 import ops
    x, w, b, _, _ = _case(M, N, K, 1, 0)
    out = ops.linear_any(x, w, b, ops.EPI_BIAS_GELU_TANH)
    exact, rounded = formula(x, w, b, 1, None, None, 0)
    assert_bf16_parity(out, exact, rounded, name="w8a8 gelu")
    mism = (out.float() != rounded.float()).float().mean().item()
    print(f"w8a8 gelu {M}x{N}x{K}: {mism:.4f} of outputs off the formula's rounding")
    assert mism < 0.02


def test_linear_w8a8_sp_options_bit_equal_to_plain_call():
    """x_seg_len / x_seg_stride (the return buffer, quantised through the segmented quantiser) and out_col_offsets (heads
    scattered into a send buffer) give exactly the plain call's outputs, rearranged; the same call twice gives the same bits."""
    from fastvideo_b200 import ops
    torch.manual_seed(7)
    M, K, N, seg = 300, 1024, 768, 256
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = ops.Int8Weight.quantize((torch.randn(N, K, device="cuda") / 32).bfloat16(), int8_activations=True)
    b = torch.randn(N, device="cuda").bfloat16()
    plain = ops.linear_any(x, w, b)
    assert torch.equal(ops.linear_any(x, w, b), plain)
    buf = x.view(M, K // seg, seg).permute(1, 0, 2).contiguous()  # [4, M, 256]
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.linear_sp(buf, M, K, seg, w, b, out, N, x_seg_len=seg, x_seg_stride=M * seg)
    assert torch.equal(out, plain)
    send = torch.zeros(2, M, N // 256, 128, device="cuda", dtype=torch.bfloat16)
    offs = torch.tensor([(j % 2) * M * (N // 2) + (j // 2) * 128 for j in range(N // 128)], device="cuda", dtype=torch.int64)
    ops.linear_sp(x, M, K, K, w, b, send, N // 2, out_col_offsets=offs)
    assert torch.equal(send.permute(1, 2, 0, 3).reshape(M, N), plain)
    # a row slice keeps the mode: the V rows of a fused weight give the plain call's columns
    assert torch.equal(ops.linear_any(x, w[256:512], b[256:512]), plain[:, 256:512])


def test_linear_w8a8_rejects_bad_arguments():
    from fastvideo_b200 import ops
    from fastvideo_b200._lib import lib, ptr
    x, w, b, _, _ = _case(64, 128, 256, 0, 0)
    with pytest.raises(ops.FvbError):
        ops.linear_any(x[:, :128], w)  # K mismatch
    out = torch.empty(64, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(ops.FvbError):  # column-block offsets need N % 128 == 0
        ops.linear_sp(x, 64, 256, 256, w[:64], None, out, 128, out_col_offsets=torch.zeros(1, device="cuda", dtype=torch.int64))
    # K past the s32 bound
    K = 133152
    big = ops.Int8Weight.quantize(torch.ones(8, K, device="cuda").bfloat16(), int8_activations=True)
    with pytest.raises(ops.FvbError, match="133144"):
        ops.linear_any(torch.ones(1, K, device="cuda").bfloat16(), big)
    # missing scales
    xq, xs = ops.quantize_int8_rows(x)
    null = ptr(None)
    rc = lib().fvb_linear_w8a8_sp(ptr(xq), c_int64(xq.stride(0)), null, ptr(w.q), c_int64(w.q.stride(0)), null, null, ptr(out),
                                  c_int64(128), null, null, c_int64(0), null, c_int(0), c_int64(0), c_int(64), c_int(128),
                                  c_int(256), c_int(0), null)
    assert rc != 0


# ------------------------------------------------------------------------------------------------ Wan block / model
def _rope(seq, d):
    return wan_ref.rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)])


def _block_cfg(g, **kw):
    from fastvideo_b200 import wan_dit
    D, H = g["x"].shape[-1], g["heads"]
    return wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                                num_layers=1, **kw)


W8A8 = dict(int8_weights=True, int8_activations=True)
BLOCK_BOUND = 1e-2
MODEL_BOUND = 1e-2
CAUSAL_BOUND = 1e-2


@pytest.mark.parametrize("name", ["wan_block_dense", "wan_block_i2v"])
def test_block_w8a8_against_routed_oracle(golden_dir, name):
    from fastvideo_b200 import ops, wan_dit
    g = torch.load(os.path.join(golden_dir, name + ".pt"))
    D, H = g["x"].shape[-1], g["heads"]
    cfg = _block_cfg(g, **W8A8)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    for n in wan_dit.INT8_LINEARS:
        assert getattr(blk, n) is None or (isinstance(getattr(blk, n), ops.Int8Weight) and getattr(blk, n).int8_activations), n
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    cos, sin = _rope(g["seq"], D // H)
    with torch.no_grad():
        yb = w8a8_ref.wan_block_w8a8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
    e = rel_l2(y, yb[0])
    print(f"w8a8 {name}: relL2 {e:.3e} vs routed bf16 oracle; {rel_l2(y, g['y_fp32'][0]):.3e} from the fp32 oracle")
    assert e < BLOCK_BOUND


def _model(golden_dir, **kw):
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], **kw)
    return g, cfg, wan_dit.WanDiT(cfg, sd)


def test_model_w8a8_against_routed_oracle(golden_dir):
    g, cfg, model = _model(golden_dir, **W8A8)
    y = model.forward(g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    with torch.no_grad():
        yb = w8a8_ref.wan_model_w8a8(g["latents"], g["text"], g["timestep"], g["sd"], g["heads"])
    e = rel_l2(y, yb)
    print(f"w8a8 model: relL2 {e:.3e} vs routed bf16 oracle; {rel_l2(y, g['y_fp32']):.3e} from the fp32 oracle")
    assert e < MODEL_BOUND


def test_block_vsa_w8a8_against_routed_oracle():
    """The VSA block of test_gpu_w8 on W8A8 (the gate rows of w_qkv included): median row relL2 against the routed oracle."""
    from fastvideo_b200 import wan_dit
    from oracle.gen_golden import _rand_block_sd
    g = torch.Generator().manual_seed(5)
    D, H, F_, L = 256, 2, 512, 24
    seq = (5, 6, 7)
    S = int(np.prod(seq))
    sd = _rand_block_sd(D, F_, H, True, g)
    x = torch.randn(1, S, D, generator=g).bfloat16()
    ctx = torch.randn(1, L, D, generator=g).bfloat16()
    temb6 = (torch.randn(1, 6, D, generator=g) * 0.5).bfloat16()
    cos, sin = wan_ref.rotary_tables(seq, [44, 42, 42])
    tile = (4, 4, 4)
    vbs = torch.from_numpy(vsa_index.variable_block_sizes(seq, tile))
    meta = dict(tile_partition=torch.from_numpy(vsa_index.tile_partition_indices(seq, tile)),
                untile_combined=torch.from_numpy(vsa_index.untile_combined_index(seq, tile)),
                non_pad=torch.from_numpy(vsa_index.non_pad_index(vbs.numpy(), 64)), vbs=vbs, s_pad=vbs.numel() * 64,
                topk=vsa_index.compute_topk(0.5, vbs.numel()))
    with torch.no_grad():
        y_ref = w8a8_ref.wan_block_w8a8(x, ctx, temb6, sd, "", H, cos, sin, vsa_meta=meta)
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=F_, num_layers=1, vsa=True, **W8A8)
    blk = wan_dit.WanBlock(cuda_sd(sd), "", cfg)
    lay = wan_dit.make_layout(seq, cfg, "cuda", vsa_sparsity=0.5)
    y = wan_dit.block_forward(x[0].cuda()[lay.perm], blk, ctx[0].cuda(), temb6.cuda(), lay, cfg)[lay.inv_perm]
    err_rows = (y.float().cpu() - y_ref[0].float()).norm(dim=-1) / y_ref[0].float().norm(dim=-1)
    print(f"w8a8 VSA block: median row relL2 {err_rows.median().item():.3e}, whole {rel_l2(y, y_ref[0]):.3e} vs routed oracle")
    assert err_rows.median().item() < BLOCK_BOUND
    assert (err_rows < 3e-2).float().mean().item() > 0.9


def test_block_w8a8_with_attention_8bit(golden_dir):
    """int8_activations + attention_8bit on the dense block, against the oracle with its self-attention on the 8-bit
    restatement and its linears on W8A8."""
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_dense.pt"))
    D, H = g["x"].shape[-1], g["heads"]
    cfg = _block_cfg(g, attention_8bit=True, **W8A8)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    cos, sin = _rope(g["seq"], D // H)
    with torch.no_grad(), w8a8_ref.wan_block_linears_in_w8a8(g["sd"], [""]):
        y_ref = attn8_ref.wan_block_attn8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
    e = rel_l2(y, y_ref[0])
    print(f"w8a8 + attention_8bit block: relL2 {e:.3e} vs routed oracle")
    assert e < BLOCK_BOUND


# ------------------------------------------------------------------------------------------------ causal rollout
@pytest.mark.parametrize("policy", ["absolute", "relativistic"])
def test_causal_block_rollout_w8a8_against_routed_oracle(golden_dir, policy):
    """The golden causal block rollouts (sink frame, eviction, the ring-wrapped QKV write) on W8A8, call by call."""
    from fastvideo_b200 import causal_wan, wan_dit
    from fastvideo_b200.rope import get_rotary_pos_embed
    rel = policy == "relativistic"
    g = torch.load(os.path.join(golden_dir, "wan_causal_block_rel.pt" if rel else "wan_causal_block.pt"))
    D, H = g["sd"]["to_q.weight"].shape[0], g["heads"]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1, **W8A8)
    grid, nf = tuple(g["grid"]), g["frames_per_call"]
    fs = grid[0] * grid[1]
    W, S = g["window_frames"], g["sink_frames"]
    ccfg = causal_wan.CausalConfig(local_attn_size=W, sink_size=S, num_frames_per_block=nf, rope_cache_policy=policy)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    cache = causal_wan.KVCache(W * fs, H, cfg.head_dim, "cuda", S * fs)
    xc = causal_wan.CrossAttnCache()
    ctx = g["ctx"][0].cuda()
    rb, xb = causal_ref.new_kv_cache(1, W * fs, H, 128), {"is_init": False}
    worst = 0.0
    for i, c in enumerate(g["calls"]):
        if rel:
            cos, sin = get_rotary_pos_embed((W, ) + grid, [44, 42, 42], start_frame=0, keep_f64=True)
        else:
            cos, sin = get_rotary_pos_embed((nf, ) + grid, [44, 42, 42], start_frame=c["start_frame"], keep_f64=True)
        cs = c["start_frame"] * fs
        y = causal_wan.causal_block_forward(c["x"][0].cuda(), blk, ctx, c["temb"][0].cuda(), cos.cuda(), sin.cuda(), cache, xc,
                                            cs, cfg, ccfg, frame_seqlen=fs)
        kw = dict(crossattn_cache=xb, rope_cache_policy="relativistic") if rel else dict(crossattn_cache=xb)
        with torch.no_grad():
            yb = w8a8_ref.causal_block_w8a8(c["x"], g["ctx"], c["temb"], g["sd"], "", H, cos, sin, rb, cs, W, S, fs, **kw)
        e = rel_l2(y, yb[0])
        worst = max(worst, e)
        print(f"w8a8 causal block ({policy}) call {i}: relL2 {e:.3e} vs routed oracle")
        assert cache.local_end_index == c["local_end_index"]
    assert cache.head != 0
    assert worst < CAUSAL_BOUND


def _causal_model(golden_dir, policy="absolute", **kw):
    from fastvideo_b200 import causal_wan, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_causal_model_rel.pt" if policy == "relativistic" else "wan_causal_model.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], text_len=g["text_len"],
                               **kw)
    ccfg = causal_wan.CausalConfig(local_attn_size=g["window_frames"], sink_size=g["sink_frames"],
                                   num_frames_per_block=g["frames_per_call"], rope_cache_policy=policy)
    return g, cfg, causal_wan.CausalWanDiT(cfg, sd, ccfg)


@pytest.mark.parametrize("policy", ["absolute", "relativistic"])
def test_causal_model_rollout_w8a8_against_routed_oracle(golden_dir, policy):
    g, cfg, model = _causal_model(golden_dir, policy, **W8A8)
    H, W, S = g["heads"], g["window_frames"], g["sink_frames"]
    c0 = g["calls"][0]["latents"]
    fs = (c0.shape[3] // 2) * (c0.shape[4] // 2)
    kv, xc = model.new_caches(fs, "cuda")
    text = g["text"].cuda()
    kb = [causal_ref.new_kv_cache(1, W * fs, H, 128) for _ in range(2)]
    xb = [{"is_init": False} for _ in range(2)]
    worst = 0.0
    for i, c in enumerate(g["calls"]):
        y = model.forward_inference(c["latents"].cuda(), text, c["timestep"].cuda(), kv, xc, current_start=c["start_frame"] * fs,
                                    start_frame=c["start_frame"])
        kw = dict(current_start=c["start_frame"] * fs, start_frame=c["start_frame"], local_attn_size=W, sink_size=S,
                  text_len=g["text_len"])
        if policy == "relativistic":
            kw["rope_cache_policy"] = "relativistic"
        with torch.no_grad():
            yb = w8a8_ref.causal_model_w8a8(c["latents"], g["text"], c["timestep"], g["sd"], H, kb, xb, **kw)
        e = rel_l2(y, yb)
        worst = max(worst, e)
        print(f"w8a8 causal model ({policy}) call {i}: relL2 {e:.3e} vs routed oracle")
    assert kv[0].head != 0
    assert worst < CAUSAL_BOUND


# ------------------------------------------------------------------------------------------------ graph, memory, SP
def test_denoiser_graph_replay_bit_equal_w8a8(golden_dir):
    from fastvideo_b200.api import WanDenoiser
    g, cfg, model = _model(golden_dir, **W8A8)
    den = WanDenoiser(model, use_graph=True)
    lat = g["latents"].pin_memory()
    txt = g["text"].pin_memory()
    t = float(g["timestep"][0])
    out = den.step(lat, txt, t)
    torch.cuda.synchronize()
    assert den.graph_status == "captured", den.graph_status
    out = out.clone()
    eager = model.forward(g["latents"].cuda(), g["text"].cuda(), torch.full((1,), t, device="cuda"))
    assert torch.equal(out, eager.cpu())
    out2 = den.step(lat, txt, t)
    torch.cuda.synchronize()
    assert torch.equal(out2, out)


def _block_weight_bytes(blk):
    from fastvideo_b200 import ops
    total = 0
    for v in vars(blk).values():
        if isinstance(v, ops.Int8Weight):
            total += v.nbytes
        elif torch.is_tensor(v):
            total += v.numel() * v.element_size()
    return total


def test_weight_bytes_equal_int8_weights():
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(**wan_dit.WAN_14B, vsa=True)
    sd = wan_dit.random_state_dict(wan_dit.WanDiTConfig(**{**cfg.__dict__, "num_layers": 1}), "cuda", layers=1)
    w8 = _block_weight_bytes(wan_dit.WanBlock(sd, "blocks.0.", wan_dit.WanDiTConfig(**wan_dit.WAN_14B, vsa=True,
                                                                                    int8_weights=True)))
    a8 = _block_weight_bytes(wan_dit.WanBlock(sd, "blocks.0.", wan_dit.WanDiTConfig(**wan_dit.WAN_14B, vsa=True, **W8A8)))
    assert a8 == w8


def test_sequence_parallel_and_causal_accept_w8a8(golden_dir):
    """The sequence-parallel and causal classes take a W8A8 model (their fp8 refusals stay)."""
    from fastvideo_b200 import causal_wan, distributed
    g, cfg, model = _model(golden_dir, **W8A8)
    distributed.SPWanDiT(model, 0, 1)
    _, _, cmodel = _causal_model(golden_dir, **W8A8)
    causal_wan.SPCausalWanDiT(cmodel, 0, 1)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_sp_w8a8_equals_single_rank(tmp_path):
    """tests/sp_worker.py w8a8 on 2 ranks: SPWanDiT on W8A8 bit-equal to the single-rank engine (dense and VSA, push and
    NCCL), SPCausalWanDiT on W8A8 within 6e-3 of it."""
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, {torch.cuda.device_count()} visible")
    out = str(tmp_path / f"sp_w8a8_parity_{world}.json")
    env = dict(os.environ, SP_WORKER_OUT=out)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "sp_worker.py"), "w8a8"]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT, env=env)
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    res = json.load(open(out))
    assert any(r.get("causal") and "call" in r for r in res), res
    assert all(r["ok_all_ranks"] for r in res if "skipped" not in r), res
