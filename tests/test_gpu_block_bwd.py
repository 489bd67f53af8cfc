"""GPU: the Wan engine block's backward. The new kernels (fvb_linear_bf16_aux, fvb_linear_dgrad_gelu_bf16,
fvb_resid_gate_bwd, fvb_layernorm_modulate_bwd, fvb_rmsnorm_rope_bwd) against their restatements (tests/block_bwd_ref.py),
and wan_dit.block_forward under grad against fp32 torch autograd of oracle.wan_ref.wan_block, with the rule of
tests/test_gpu_linear_bwd.py: relL2(ours, fp32) <= relL2(bf16 torch autograd, fp32) + 2e-3."""
import os

import numpy as np
import pytest
import torch

import block_bwd_ref as ref
from elementwise_ref import ulp_bf16 as _ulp_bf16
from test_gpu_linear_bwd import KEY_BIASES, TOL
from util import rel_l2

pytestmark = pytest.mark.gpu


def _rand(shape, seed, scale=1.0, dtype=torch.bfloat16, shift=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale + shift).to(dtype)


def _within_sum_bound(got, terms, name):
    """An fp32 column sum of `terms` [M, N] (fp64 here): the summation error bound plus one bf16 ulp when got is bf16."""
    t = terms.double()
    exact = t.sum(0)
    bound = t.shape[0] * 2.0 ** -24 * t.abs().sum(0) + 1e-30
    if got.dtype == torch.bfloat16:
        bound = bound + _ulp_bf16(exact)
    err = (got.double() - exact).abs()
    assert (err <= bound).all(), f"{name}: max error {err.max().item():.3e}"


# ---------------------------------------------------------------- kernels
@pytest.mark.parametrize("M,N,K", [(333, 256, 384), (1000, 1536, 1536), (1000, 5120, 13824), (777, 1536, 8960)])
def test_aux_epilogues(M, N, K):
    """out is bit-identical to linear's, aux to linear with EPI_BIAS."""
    from fastvideo_b200 import ops
    x, w = _rand((M, K), 1), _rand((N, K), 2, K ** -0.5)
    b, resid = _rand((N,), 3), _rand((M, N), 4)
    gate = _rand((N,), 5, dtype=torch.float32)
    y = ops.linear(x, w, b)
    for epi in (ops.EPI_BIAS_GELU_TANH, ops.EPI_RESID_GATE_F32, ops.EPI_RESID_GATE_BF16):
        kw = {} if epi == ops.EPI_BIAS_GELU_TANH else dict(resid=resid, gate=gate)
        out, aux = ops.linear_aux(x, w, b, epi, **kw)
        assert torch.equal(out, ops.linear(x, w, b, epi, **kw)), epi
        assert torch.equal(aux, y), epi


@pytest.mark.parametrize("M,N,K", [(333, 1536, 8960), (1000, 5120, 13824), (129, 256, 512)])
def test_dgrad_gelu(M, N, K):
    from fastvideo_b200 import ops
    dy, w, h = _rand((M, N), 6), _rand((N, K), 7, N ** -0.5), _rand((M, K), 8, 2.0)
    got = ops.linear_dgrad_gelu(dy, w, h)
    want = ref.linear_dgrad_gelu(dy, w, h, bf16_points=True)
    # bf16(acc) may differ by the fp32 summation order (one bf16 ulp of acc), then one more rounding
    # plus the fp32 evaluation of gelu' (the hardware exp2 and divide approximations): below 4e-6 absolute, which matters
    # where gelu' crosses zero
    # where |acc| is tiny, the fp32 summation error bound of acc (relative to sum |dy| |w|, not to acc) takes over
    acc = dy.double() @ w.double()
    gp = ref.gelu_tanh_grad(h.double()).abs()
    bound = (2 * _ulp_bf16(want.double()) + 2 * _ulp_bf16(acc) * gp + 4e-6 * acc.abs()
             + 2 * N * 2.0 ** -24 * (dy.double().abs() @ w.double().abs()) * gp)
    err = (got.double() - want.double()).abs()
    assert (err <= bound).all(), f"max error {err.max().item():.3e}"
    assert torch.equal(got, ops.linear_dgrad_gelu(dy, w, h))


@pytest.mark.parametrize("M,N", [(1, 64), (333, 1536), (1000, 5120), (75600 // 8, 5120)])
@pytest.mark.parametrize("f32", [True, False])
def test_resid_gate_bwd(M, N, f32):
    from fastvideo_b200 import ops
    dout = _rand((M, N), 9, dtype=torch.float32 if f32 else torch.bfloat16, shift=0.5)
    y, gate = _rand((M, N), 10, shift=0.5), _rand((N,), 11, dtype=torch.float32)
    dy, d_gate, db = ops.resid_gate_bwd(dout, y, gate)
    rdy, _, _ = ref.resid_gate_bwd(dout, y, gate, bf16_points=True)
    assert torch.equal(dy, rdy)  # one fp32 product, one rounding
    _within_sum_bound(d_gate, dout.double() * y.double(), "d_gate")
    _within_sum_bound(db, dy, "db")
    again = ops.resid_gate_bwd(dout, y, gate)
    assert all(torch.equal(a, b) for a, b in zip((dy, d_gate, db), again))


def _ln_case(M, D, form, seed):
    x = _rand((M, D), seed, 2.0, torch.float32 if form == "affine" else torch.bfloat16, 0.3)
    dn = _rand((M, D), seed + 1, shift=0.5)
    gain = _rand((D,), seed + 2, 0.2, torch.float32, 1.0 if form == "affine" else 0.0)
    gin = _rand((M, D), seed + 3, dtype=torch.float32 if form != "round_ln" else torch.bfloat16)
    return x, dn, gain, gin


@pytest.mark.parametrize("M,D", [(333, 1536), (1000, 5120), (3, 256)])
@pytest.mark.parametrize("form", ["modulate", "affine", "round_ln"])
def test_layernorm_modulate_bwd(M, D, form):
    from fastvideo_b200 import ops
    x, dn, gain, gin = _ln_case(M, D, form, M + D)
    kw = dict(weight=gain) if form == "affine" else dict(scale=gain)
    dx, d_gain, d_off = ops.layernorm_modulate_bwd(x, dn, round_ln=form == "round_ln", gin=gin, **kw)
    rdx, _, _ = ref.layernorm_modulate_bwd(x, dn, gain, form != "affine", form == "round_ln", gin=gin, bf16_points=True)
    assert dx.dtype == x.dtype
    # fp32 row statistics in another order than fp64: relative error far below a bf16 ulp, then (bf16 x) one rounding
    e = rel_l2(dx, rdx)
    assert e < (4e-3 if dx.dtype == torch.bfloat16 else 1e-5), e
    if dx.dtype == torch.bfloat16:
        assert ((dx.float() - rdx.float()).abs() <= 2 * _ulp_bf16(rdx.double()).float() + 1e-6).float().mean() > 0.999
    xf = x.double()
    t = (xf - xf.mean(-1, keepdim=True)) / torch.sqrt(xf.var(-1, unbiased=False, keepdim=True) + 1e-6)
    if form == "round_ln":
        t = t.float().bfloat16().double()
    # round_ln: an fp32 t and an fp64 t can round to neighbouring bf16 values at a rounding boundary
    assert rel_l2(d_gain, (dn.double() * t).sum(0)) < (1e-4 if form == "round_ln" else 1e-5)
    _within_sum_bound(d_off, dn, "d_offset")
    again = ops.layernorm_modulate_bwd(x, dn, round_ln=form == "round_ln", gin=gin, **kw)
    assert all(torch.equal(a, b) for a, b in zip((dx, d_gain, d_off), again))


@pytest.mark.parametrize("M,D,H", [(333, 1536, 12), (1000, 5120, 40), (77, 256, 2)])
def test_rmsnorm_rope_bwd_into_fused_buffer(M, D, H):
    """q and k in one launch, x read from and dx written to column slices of fused [M, 4D] buffers; the other columns keep
    their sentinel."""
    from fastvideo_b200 import ops, wan_dit
    d = D // H
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H)
    lay = wan_dit.make_layout((1, 1, M), cfg, "cuda")
    qkv = _rand((M, 4 * D), M, 2.0)
    dy = _rand((M, 2 * D), M + 1)
    w0, w1 = _rand((D,), M + 2, 0.2, shift=1.0), _rand((D,), M + 3, 0.2, shift=1.0)
    rope_row = torch.arange(M, device="cuda", dtype=torch.int32).flip(0).contiguous()
    sentinel = -7.0
    dqkv = torch.full((M, 4 * D), sentinel, dtype=torch.bfloat16, device="cuda")
    dw0, dw1 = ops.rmsnorm_rope_bwd(qkv[:, :D], w0, dy[:, :D], dqkv[:, :D], qkv[:, D:2 * D], w1, dy[:, D:], dqkv[:, D:2 * D],
                                    lay.cos, lay.sin, rope_row, head_dim=d)
    assert (dqkv[:, 2 * D:] == sentinel).all()
    cos, sin = lay.cos[rope_row.long()].repeat(1, H), lay.sin[rope_row.long()].repeat(1, H)
    for i, (w, dw) in enumerate(((w0, dw0), (w1, dw1))):
        x = qkv[:, i * D:(i + 1) * D]
        rdx, rdw = ref.rmsnorm_rope_bwd(x, w, dy[:, i * D:(i + 1) * D], cos, sin, 1e-6, bf16_points=True)
        got = dqkv[:, i * D:(i + 1) * D]
        assert rel_l2(got, rdx) < 4e-3
        assert ((got.float() - rdx.float()).abs() <= 2 * _ulp_bf16(rdx.double()).float() + 1e-6).float().mean() > 0.999
        assert rel_l2(dw, rdw) < 4e-3
    again = torch.full_like(dqkv, sentinel)
    dw0b, dw1b = ops.rmsnorm_rope_bwd(qkv[:, :D], w0, dy[:, :D], again[:, :D], qkv[:, D:2 * D], w1, dy[:, D:],
                                      again[:, D:2 * D], lay.cos, lay.sin, rope_row, head_dim=d)
    assert torch.equal(again, dqkv) and torch.equal(dw0b, dw0) and torch.equal(dw1b, dw1)


# ---------------------------------------------------------------- the block end to end
def _oracle_grads(g, dtype, dy, vsa_meta=None, block_map=None, device="cuda"):
    """x / ctx / temb6 / parameter gradients (+ "out:<bias>" for KEY_BIASES) of oracle.wan_ref.wan_block in `dtype`.
    block_map: the VSA block selection to use instead of the oracle's own top-k (which has no gradient): the engine's,
    so that the three evaluations differentiate the same sparse attention."""
    from oracle import wan_ref
    D, H = g["x"].shape[-1], g["heads"]
    d = D // H
    sd = {k: v.to(device, dtype).requires_grad_(True) for k, v in g["sd"].items()}
    ins = {k: g[k].to(device, dtype).requires_grad_(True) for k in ("x", "ctx", "temb6")}
    cos, sin = (t.to(device) for t in wan_ref.rotary_tables(g["seq"], [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)]))
    outs, lin = {}, wan_ref.linear

    def keep_key_outputs(x, w, b):
        y = lin(x, w, b)
        for k in KEY_BIASES:
            if k in sd and b is sd[k]:
                y.retain_grad()
                outs["out:" + k] = y
        return y

    wan_ref.linear = keep_key_outputs
    topk_mask = wan_ref.topk_mask
    if block_map is not None:
        wan_ref.topk_mask = lambda scores, topk: block_map.to(scores.device).view(scores.shape)
    try:
        with torch.device(device):
            y = wan_ref.wan_block(ins["x"], ins["ctx"], ins["temb6"], sd, "", H, cos, sin, vsa_meta=vsa_meta)
    finally:
        wan_ref.linear, wan_ref.topk_mask = lin, topk_mask
    y.backward(dy.to(y.device, y.dtype))
    return {**{k: t.grad for k, t in ins.items()}, **{k: t.grad for k, t in sd.items()},
            **{k: t.grad for k, t in outs.items()}}


def _engine(g, vsa=False, sparsity=None):
    from fastvideo_b200 import wan_dit
    D, H = g["x"].shape[-1], g["heads"]
    sd = {k: v.cuda() for k, v in g["sd"].items()}
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=sd["ffn.fc_in.weight"].shape[0], num_layers=1,
                               vsa=vsa)
    blk = wan_dit.WanBlock(sd, "", cfg)
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda", vsa_sparsity=sparsity)
    return cfg, blk, lay


def _engine_grads(g, dy, vsa=False, sparsity=None):
    """block_forward under grad: (output in raster order, {reference name or x / ctx / temb6: gradient}, the VSA block
    map or None)."""
    from fastvideo_b200 import wan_dit
    cfg, blk, lay = _engine(g, vsa, sparsity)
    for n, t in blk.tensors().items():
        setattr(blk, n, t.detach().clone().requires_grad_(True))
    perm = (lambda t: t[lay.perm]) if lay.perm is not None else (lambda t: t)
    unperm = (lambda t: t[lay.inv_perm]) if lay.inv_perm is not None else (lambda t: t)
    ins = {k: g[k][0].cuda().requires_grad_(True) for k in ("x", "ctx")}
    ins["temb6"] = g["temb6"].cuda().requires_grad_(True)
    y = wan_dit.block_forward(perm(ins["x"]), blk, ins["ctx"], ins["temb6"], lay, cfg)
    assert y.grad_fn is not None
    # the VSA forward's saved tensors follow the block's own; index 14 of them is the block map
    block_map = y.grad_fn.saved_tensors[6 + len(y.grad_fn.names) + 14].clone() if vsa else None
    y.backward(perm(dy[0]))
    grads = wan_dit.WanBlock.to_reference_names({n: t.grad for n, t in blk.tensors().items()})
    grads.update({k: t.grad.unsqueeze(0) if k != "temb6" else t.grad for k, t in ins.items()})
    return unperm(y.detach()), grads, block_map


def _check_block(g, vsa_meta=None, sparsity=None, seed=0):
    dy = torch.randn(g["x"].shape, generator=torch.Generator().manual_seed(seed)).bfloat16().cuda()
    y, ours, block_map = _engine_grads(g, dy, vsa_meta is not None, sparsity)
    # the oracle's VSA restatement keeps its tile tables on the host: that block runs on the CPU
    dev = "cuda" if vsa_meta is None else "cpu"
    truth = _oracle_grads(g, torch.float32, dy, vsa_meta, block_map, dev)
    floor = _oracle_grads(g, torch.bfloat16, dy, vsa_meta, block_map, dev)
    checked, bad = 0, []
    for k, t in truth.items():
        if k.startswith("out:"):
            continue
        if t is None:  # a parameter the block does not use (attn2.norm_added_q)
            assert k not in ours, k
            continue
        got = ours[k]
        assert got is not None and torch.isfinite(got.float()).all(), k
        assert got.shape == t.shape, (k, got.shape, t.shape)
        if k in KEY_BIASES:
            # softmax cancels a bias shared by all keys up to what the QK RMSNorm lets through (see KEY_BIASES in
            # test_gpu_linear_bwd): the exact gradient is a small remainder of a sum of large per-token terms, and two
            # equally accurate bf16 pipelines land a few e-3 apart there in either direction. test_gpu_linear_bwd holds the
            # key projection's output gradient instead; the engine keeps that gradient inside its fused d(qkv) buffer,
            # whose key columns also feed the key weight gradient (to_k.weight), which is held to the strict rule above.
            # The bias itself is held to three times the larger bf16-autograd distance (bias or output gradient) + TOL.
            up = "out:" + k
            e, fl = rel_l2(got, t), rel_l2(floor[k], t)
            if not e <= max(fl, rel_l2(floor[up], truth[up])) * 3 + TOL:
                bad.append(f"{k}: relL2 {e:.3e} (bf16 autograd {fl:.3e})")
        else:
            e, fl = rel_l2(got, t), rel_l2(floor[k], t)
            if not e <= fl + TOL:
                bad.append(f"{k}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + {TOL}")
        checked += 1
    assert not bad, "; ".join(bad)
    assert checked == sum(1 for t in truth.values() if t is not None) - sum(1 for k in truth if k.startswith("out:"))
    return y


@pytest.mark.parametrize("name", ["wan_block_dense", "wan_block_i2v"])
def test_block_gradients_against_fp32_autograd(golden_dir, name):
    _check_block(torch.load(os.path.join(golden_dir, f"{name}.pt")))


def _vsa_case():
    from oracle import vsa_index
    from oracle.gen_golden import _rand_block_sd
    g = torch.Generator().manual_seed(5)
    D, H, F_, L = 256, 2, 512, 24
    seq = (5, 6, 7)
    S = int(np.prod(seq))
    sd = _rand_block_sd(D, F_, H, True, g)
    case = dict(sd=sd, x=torch.randn(1, S, D, generator=g).bfloat16(), ctx=torch.randn(1, L, D, generator=g).bfloat16(),
                temb6=(torch.randn(1, 6, D, generator=g) * 0.5).bfloat16(), seq=seq, heads=H)
    tile = (4, 4, 4)
    vbs = torch.from_numpy(vsa_index.variable_block_sizes(seq, tile))
    meta = dict(tile_partition=torch.from_numpy(vsa_index.tile_partition_indices(seq, tile)),
                untile_combined=torch.from_numpy(vsa_index.untile_combined_index(seq, tile)),
                non_pad=torch.from_numpy(vsa_index.non_pad_index(vbs.numpy(), 64)), vbs=vbs, s_pad=vbs.numel() * 64,
                topk=vsa_index.compute_topk(0.5, vbs.numel()))
    return case, meta


def test_vsa_block_gradients_against_fp32_autograd():
    case, meta = _vsa_case()
    _check_block(case, meta, sparsity=0.5)


def test_14b_width_block_gradients():
    """One block at Wan 14B width (D = 5120, 40 heads, ffn 13824), 256 tokens, 512 text tokens."""
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_14B, "num_layers": 1})
    sd = {k[len("blocks.0."):]: v for k, v in wan_dit.random_state_dict(cfg, "cuda", 11, layers=1).items()
          if k.startswith("blocks.0.")}
    gen = torch.Generator(device="cuda").manual_seed(3)
    for k in list(sd):  # non-trivial norm weights and biases
        if k.endswith(".bias") or "norm" in k:
            sd[k] = (sd[k].float() + 0.1 * torch.randn(sd[k].shape, device="cuda", generator=gen)).bfloat16()
    case = dict(sd={k: v.cpu() for k, v in sd.items()}, x=torch.randn(1, 256, 5120).bfloat16(),
                ctx=torch.randn(1, 512, 5120).bfloat16(), temb6=(torch.randn(1, 6, 5120) * 0.5).bfloat16(), seq=(1, 16, 16),
                heads=40)
    _check_block(case)


@pytest.mark.parametrize("kind", ["dense", "i2v", "vsa"])
def test_output_bits_and_determinism(golden_dir, kind):
    """The block output under grad is the no-grad block_forward's, bit for bit; two backward passes give the same bits."""
    from fastvideo_b200 import wan_dit
    if kind == "vsa":
        g, _ = _vsa_case()
        args = dict(vsa=True, sparsity=0.5)
    else:
        g, args = torch.load(os.path.join(golden_dir, f"wan_block_{kind}.pt")), {}
    cfg, blk, lay = _engine(g, **args)
    x = g["x"][0].cuda()
    if lay.perm is not None:
        x = x[lay.perm]
    with torch.no_grad():
        plain = wan_dit.block_forward(x, blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    dy = torch.randn(g["x"].shape, generator=torch.Generator().manual_seed(1)).bfloat16().cuda()
    y1, g1, _ = _engine_grads(g, dy, **args)
    y2, g2, _ = _engine_grads(g, dy, **args)
    if lay.inv_perm is not None:
        plain = plain[lay.inv_perm]
    assert torch.equal(y1, plain) and torch.equal(y2, plain)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_no_grad_path_unchanged_when_nothing_requires_grad(golden_dir):
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_dense.pt"))
    cfg, blk, lay = _engine(g)
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    assert y.grad_fn is None


@pytest.mark.parametrize("fmt", ["fp8_linears", "int8_weights", "w8a8", "attention_8bit", "fp32_rmsnorm"])
def test_refusals(golden_dir, fmt):
    """Configurations without a backward raise FvbError under grad and run as before without it."""
    from fastvideo_b200 import ops, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_dense.pt"))
    D = g["x"].shape[-1]
    sd = {k: v.cuda() for k, v in g["sd"].items()}
    opts = {"fp8_linears": dict(fp8_linears=True), "int8_weights": dict(int8_weights=True),
            "w8a8": dict(int8_weights=True, int8_activations=True), "attention_8bit": dict(attention_8bit=True),
            "fp32_rmsnorm": {}}[fmt]
    if fmt == "fp32_rmsnorm":  # q and k share one launch, so they share the weight dtype
        sd["norm_q.weight"], sd["norm_k.weight"] = sd["norm_q.weight"].float(), sd["norm_k.weight"].float()
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=sd["ffn.fc_in.weight"].shape[0],
                               num_layers=1, **opts)
    blk = wan_dit.WanBlock(sd, "", cfg)
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    x, ctx, temb6 = g["x"][0].cuda(), g["ctx"][0].cuda(), g["temb6"].cuda()
    with torch.no_grad():
        ref_y = wan_dit.block_forward(x, blk, ctx, temb6, lay, cfg)
    with pytest.raises(ops.FvbError):
        wan_dit.block_forward(x.clone().requires_grad_(True), blk, ctx, temb6, lay, cfg)
    assert torch.equal(wan_dit.block_forward(x, blk, ctx, temb6, lay, cfg), ref_y)  # nothing requires grad


def test_sequence_parallel_refuses_grad(golden_dir):
    from fastvideo_b200 import distributed, ops, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = {k: v.cuda() for k, v in g["sd"].items()}
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1])
    model = wan_dit.WanDiT(cfg, sd)
    sp = distributed.SPWanDiT(model, 0, 1)
    args = (g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    y = sp.forward(*args)
    blk = model.blocks[0]
    blk.w_o = blk.w_o.clone().requires_grad_(True)
    with pytest.raises(ops.FvbError):
        with torch.enable_grad():
            sp.forward.__wrapped__(sp, *args)
    assert torch.equal(sp.forward(*args), y)


# ---------------------------------------------------------------- outputs stay inside their shapes
def test_new_entry_points_write_only_their_outputs():
    """Every output written through a row stride wider than its width, with sentinels around it, gives the bits of the
    contiguous call and leaves the sentinels untouched."""
    from ctypes import c_float, c_int, c_int64
    from fastvideo_b200 import ops
    from fastvideo_b200._lib import check, lib, ptr, stream_ptr
    L = lib()
    M, N, K, pad = 333, 256, 384, 40
    sentinel = -12345.0
    x, w = _rand((M, K), 21), _rand((N, K), 22, K ** -0.5)
    b, resid, gate = _rand((N,), 23), _rand((M, N), 24), _rand((N,), 25, dtype=torch.float32)

    def padded(rows, cols, dtype=torch.bfloat16):
        return torch.full((rows + pad, cols + pad), sentinel, dtype=dtype, device="cuda")

    def clean(buf, ref, rows, cols):
        assert torch.equal(buf[:rows, :cols], ref)
        assert (buf[rows:] == sentinel).all() and (buf[:, cols:] == sentinel).all()

    # fvb_linear_bf16_aux
    ref_out, ref_aux = ops.linear_aux(x, w, b, ops.EPI_RESID_GATE_BF16, resid=resid, gate=gate)
    out, aux = padded(M, N), padded(M, N)
    check(L.fvb_linear_bf16_aux(ptr(x), c_int64(K), ptr(w), c_int64(K), ptr(b), ptr(out), c_int64(N + pad), ptr(resid),
                                c_int64(N), ops._f32p(gate), c_int(0), c_int64(0), ptr(aux), c_int64(N + pad), c_int(M), c_int(N),
                                c_int(K), c_int(ops.EPI_RESID_GATE_BF16), stream_ptr()))
    clean(out, ref_out, M, N)
    clean(aux, ref_aux, M, N)
    # fvb_linear_dgrad_gelu_bf16: dy [M, N], w [N, K], h [M, K]
    dy, h = _rand((M, N), 26), _rand((M, K), 27)
    ref_dh = ops.linear_dgrad_gelu(dy, w, h)
    dh = padded(M, K)
    check(L.fvb_linear_dgrad_gelu_bf16(ptr(dy), c_int64(N), ptr(w), c_int64(K), ptr(h), c_int64(K), ptr(dh), c_int64(K + pad),
                                       c_int(M), c_int(N), c_int(K), stream_ptr()))
    clean(dh, ref_dh, M, K)
    # fvb_resid_gate_bwd
    dout, y = _rand((M, N), 28, dtype=torch.float32), _rand((M, N), 29)
    r_dy, r_dg, r_db = ops.resid_gate_bwd(dout, y, gate)
    g_dy, g_dg, g_db = padded(M, N), torch.full((N + pad,), sentinel, device="cuda"), torch.full(
        (N + pad,), sentinel, dtype=torch.bfloat16, device="cuda")
    ws = torch.empty(int(L.fvb_resid_gate_bwd_workspace_bytes(c_int(M), c_int(N))) // 4, device="cuda")
    check(L.fvb_resid_gate_bwd(ptr(dout), c_int(1), c_int64(N), ptr(y), c_int64(N), ops._f32p(gate), ptr(g_dy),
                               c_int64(N + pad), ops._f32p(g_dg), ptr(g_db), ops._f32p(ws), c_int64(ws.numel() * 4), c_int(M),
                               c_int(N), stream_ptr()))
    clean(g_dy, r_dy, M, N)
    for got, want in ((g_dg, r_dg), (g_db, r_db)):
        assert torch.equal(got[:N], want) and (got[N:] == sentinel).all()
    # fvb_layernorm_modulate_bwd (bf16 x, modulation, fp32 incoming gradient)
    xl, dn, scale, gin = _rand((M, N), 30), _rand((M, N), 31), _rand((N,), 32, 0.2, torch.float32), _rand((M, N), 33,
                                                                                                          dtype=torch.float32)
    r_dx, r_ds, r_dh = ops.layernorm_modulate_bwd(xl, dn, scale=scale, gin=gin)
    g_dx = padded(M, N)
    g_ds, g_dh = torch.full((N + pad,), sentinel, device="cuda"), torch.full((N + pad,), sentinel, device="cuda")
    ws = torch.empty(int(L.fvb_layernorm_modulate_bwd_workspace_bytes(c_int(M), c_int(N))) // 4, device="cuda")
    check(L.fvb_layernorm_modulate_bwd(ptr(xl), c_int(0), c_int64(N), ptr(dn), c_int64(N), ops._f32p(scale), c_int(1), c_int(0),
                                       ptr(gin), c_int(1), c_int64(N), ptr(g_dx), c_int64(N + pad), ops._f32p(g_ds),
                                       ops._f32p(g_dh), ops._f32p(ws), c_int64(ws.numel() * 4), c_int(M), c_int(N),
                                       c_float(1e-6), stream_ptr()))
    clean(g_dx, r_dx, M, N)
    for got, want in ((g_ds, r_ds), (g_dh, r_dh)):
        assert torch.equal(got[:N], want) and (got[N:] == sentinel).all()


def test_rmsnorm_rope_bwd_one_tensor_without_dw():
    from fastvideo_b200 import ops, wan_dit
    M, D, H = 300, 1536, 12
    lay = wan_dit.make_layout((1, 1, M), wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H), "cuda")
    x, dy, w = _rand((M, D), 40), _rand((M, D), 41), _rand((D,), 42, 0.2, shift=1.0)
    dx = torch.empty_like(x)
    assert ops.rmsnorm_rope_bwd(x, w, dy, dx, None, None, None, None, lay.cos, lay.sin, want_dw=False) == (None, None)
    dx2 = torch.empty_like(x)
    dw, _ = ops.rmsnorm_rope_bwd(x, w, dy, dx2, None, None, None, None, lay.cos, lay.sin)
    assert torch.equal(dx, dx2) and dw is not None


def test_affine_layernorm_backward_refuses_round_ln():
    from fastvideo_b200 import ops
    x, dn, w = _rand((64, 256), 50, dtype=torch.float32), _rand((64, 256), 51), _rand((256,), 52, dtype=torch.float32)
    with pytest.raises(ops.FvbError):
        ops.layernorm_modulate_bwd(x, dn, weight=w, round_ln=True)


def test_i2v_block_without_text_tokens_refuses_grad(golden_dir):
    """An I2V context of only the 257 image tokens runs without grad (the image branch alone) and is refused under grad."""
    from fastvideo_b200 import ops, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_i2v.pt"))
    cfg, blk, lay = _engine(g)
    x, ctx, temb6 = g["x"][0].cuda(), g["ctx"][0, :257].cuda(), g["temb6"].cuda()
    with torch.no_grad():
        y = wan_dit.block_forward(x, blk, ctx, temb6, lay, cfg)
    assert torch.isfinite(y.float()).all()
    with pytest.raises(ops.FvbError):
        wan_dit.block_forward(x.clone().requires_grad_(True), blk, ctx, temb6, lay, cfg)


def test_causal_block_refuses_grad(golden_dir):
    """The causal block (per-frame bf16 modulation) raises under grad and runs as before without it."""
    from fastvideo_b200 import causal_wan, ops, wan_dit
    from fastvideo_b200.rope import get_rotary_pos_embed
    g = torch.load(os.path.join(golden_dir, "wan_causal_block.pt"))
    D = g["calls"][0]["x"].shape[-1]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1)
    grid, nf = tuple(g["grid"]), g["frames_per_call"]
    fs = grid[0] * grid[1]
    ccfg = causal_wan.CausalConfig(local_attn_size=g["window_frames"], sink_size=g["sink_frames"], num_frames_per_block=nf)
    blk = wan_dit.WanBlock({k: v.cuda() for k, v in g["sd"].items()}, "", cfg)
    c = g["calls"][0]
    cos, sin = get_rotary_pos_embed((nf, ) + grid, [44, 42, 42], start_frame=c["start_frame"], keep_f64=True)

    def run(x):
        cache = causal_wan.KVCache(g["window_frames"] * fs, cfg.num_attention_heads, cfg.head_dim, "cuda", g["sink_frames"] * fs)
        return causal_wan.causal_block_forward(x, blk, g["ctx"][0].cuda(), c["temb"][0].cuda(), cos.cuda(), sin.cuda(), cache,
                                               causal_wan.CrossAttnCache(), c["start_frame"] * fs, cfg, ccfg, frame_seqlen=fs)
    x = c["x"][0].cuda()
    with torch.no_grad():
        y = run(x)
    with pytest.raises(ops.FvbError):
        run(x.clone().requires_grad_(True))
    assert torch.equal(run(x), y)  # grad enabled, nothing requires grad
