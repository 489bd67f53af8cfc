"""CPU: the restatements of the Wan block backward kernels (tests/block_bwd_ref.py) against fp64 torch autograd of the
forward formulas, and WanBlock's fused-name -> reference-name mapping."""
import pytest
import torch
import torch.nn.functional as F

import block_bwd_ref as ref


def _g(seed):
    return torch.Generator().manual_seed(seed)


def test_gelu_dgrad_matches_autograd():
    g = _g(1)
    M, N, K = 13, 24, 40
    dy, w, h = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((M, N), (N, K), (M, K)))
    hl = h.clone().requires_grad_(True)
    (F.gelu(hl, approximate="tanh") @ w.t()).backward(dy)
    assert torch.allclose(ref.linear_dgrad_gelu(dy, w, h), hl.grad, rtol=1e-12, atol=1e-12)


def test_resid_gate_bwd_matches_autograd():
    g = _g(2)
    M, N = 29, 48
    resid, y, dout = (torch.randn(M, N, generator=g, dtype=torch.float64) for _ in range(3))
    gate, b = torch.randn(N, generator=g, dtype=torch.float64), torch.randn(N, generator=g, dtype=torch.float64)
    yl, gl, bl, rl = (t.clone().requires_grad_(True) for t in (y, gate, b, resid))
    (rl + (yl + bl) * gl).backward(dout)  # y + b: the projection whose bias gradient is the column sum of dy
    dy, d_gate, db = ref.resid_gate_bwd(dout, y + b, gate)
    assert torch.allclose(dy, yl.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(d_gate, gl.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(db, bl.grad, rtol=1e-12, atol=1e-12)
    assert torch.equal(rl.grad, dout)


@pytest.mark.parametrize("form", ["modulate", "affine", "round_ln"])
def test_layernorm_modulate_bwd_matches_autograd(form):
    g = _g(3)
    M, D = 21, 64
    x = torch.randn(M, D, generator=g, dtype=torch.float64) * 2 + 0.5
    dn, gin = torch.randn(M, D, generator=g, dtype=torch.float64), torch.randn(M, D, generator=g, dtype=torch.float64)
    gain, off = (0.3 * torch.randn(D, generator=g, dtype=torch.float64) for _ in range(2))
    if form == "affine":
        gain = gain + 1
    xl, gl, ol = (t.clone().requires_grad_(True) for t in (x, gain, off))
    t = F.layer_norm(xl, (D,), eps=1e-6)
    if form == "round_ln":  # rounding passes the gradient straight through, as torch's .to(bf16) does
        t = t + (t.detach().float().bfloat16().double() - t.detach())
    n = t * (gl if form == "affine" else 1 + gl) + ol
    (n * dn).sum().backward()
    dx, d_gain, d_off = ref.layernorm_modulate_bwd(x, dn, gain, form != "affine", form == "round_ln", gin=gin)
    assert torch.allclose(dx, xl.grad + gin, rtol=1e-10, atol=1e-10)
    assert torch.allclose(d_gain, gl.grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(d_off, ol.grad, rtol=1e-10, atol=1e-10)


def test_rmsnorm_rope_bwd_matches_autograd():
    from oracle import wan_ref
    g = _g(4)
    seq, H, d = (2, 3, 4), 2, 24
    S, D = 24, H * d
    cos, sin = (t.double() for t in wan_ref.rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)]))
    x, dy = torch.randn(S, D, generator=g, dtype=torch.float64), torch.randn(S, D, generator=g, dtype=torch.float64)
    w = 1 + 0.3 * torch.randn(D, generator=g, dtype=torch.float64)
    xl, wl = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    n = xl * torch.rsqrt(xl.pow(2).mean(-1, keepdim=True) + 1e-6) * wl
    c, s = cos.repeat(1, H), sin.repeat(1, H)  # rotary_embedding.py:124-135 in fp64 (the oracle's version computes in fp32)
    rot = torch.stack([-n[:, 1::2], n[:, 0::2]], dim=-1).flatten(-2)
    o = n * c + rot * s
    o.backward(dy)
    dx, dw = ref.rmsnorm_rope_bwd(x, w, dy, cos.repeat(1, H), sin.repeat(1, H), 1e-6)
    assert torch.allclose(dx, xl.grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(dw, wl.grad, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("golden,vsa", [("wan_block_dense", False), ("wan_block_i2v", False), ("wan_block_dense", True)])
def test_reference_names_round_trip(golden_dir, golden, vsa):
    """WanBlock.tensors() mapped back through WanBlock.to_reference_names gives the reference state_dict bit for bit."""
    import os
    from fastvideo_b200 import wan_dit
    sd = dict(torch.load(os.path.join(golden_dir, f"{golden}.pt"))["sd"])
    D = sd["to_q.weight"].shape[0]
    if vsa:
        sd["to_gate_compress.weight"] = torch.randn(D, D, generator=_g(5)).bfloat16()
        sd["to_gate_compress.bias"] = torch.randn(D, generator=_g(6)).bfloat16()
    sd["self_attn_residual_norm.norm.weight"] = sd["self_attn_residual_norm.norm.weight"].float()
    sd["self_attn_residual_norm.norm.bias"] = sd["self_attn_residual_norm.norm.bias"].float()
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=2, ffn_dim=sd["ffn.fc_in.weight"].shape[0], vsa=vsa)
    blk = wan_dit.WanBlock(sd, "", cfg)
    back = wan_dit.WanBlock.to_reference_names(blk.tensors(), "blocks.3.")
    want = {"blocks.3." + k: v for k, v in sd.items() if k != "attn2.norm_added_q.weight"}
    assert sorted(back) == sorted(want)
    for k, v in want.items():
        assert back[k].dtype == v.dtype and torch.equal(back[k], v), k
