"""GPU: the causal Wan model's training forward (CausalWanDiT.forward_train) and its backward -- the per-frame bf16
modulation kernels against restatements of their formulas, the aux GEMM's rounded per-frame gate epilogue, forward parity
with the CPU training oracle (tests/causal_train_ref.py) and with the engine's own KV-cache rollout, gradients against fp32
torch autograd with the rule of tests/test_gpu_model_bwd.py, bits with and without checkpointing, and the memory a
checkpointed causal block keeps."""
import os

import pytest
import torch

import causal_train_ref
from causal_train_ref import block_causal_mask, causal_model_train
from test_gpu_linear_bwd import KEY_BIASES, TOL
from test_gpu_model_bwd import _perturb
from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16).float()


def _sum_close(got, want, abs_sum, tol=1e-5):
    """fp32 group sums: relative error to 1e-5 of the summed magnitudes (sum |term|), the bound fp32 accumulation in any
    order meets; relative to the sum itself it would not hold where the terms cancel."""
    return float((got.double() - want).norm() / abs_sum.norm()) < tol


def _ulp_close(got, want):
    """|got - want| <= 1 bf16 ulp, the ulp taken at the larger of |got|, |want| and 2^-6 of the row's RMS: an output of the
    LayerNorm backward that cancels to far below its row's scale carries the fp32 statistics' absolute error, which no
    restatement with another summation order reproduces below that scale."""
    g, w = got.float(), want.float()
    mag = torch.maximum(torch.maximum(g.abs(), w.abs()), w.pow(2).mean(-1, keepdim=True).sqrt() / 64)
    ulp = torch.ldexp(torch.ones_like(w), (torch.frexp(mag)[1] - 8).clamp_min(-126))
    return bool(((g - w).abs() <= ulp).all())


@pytest.mark.parametrize("D,G,R,gin", [(1536, 3, 40, None), (1536, 5, 37, "f32"), (5120, 4, 24, "bf16"), (256, 21, 24, "bf16")])
def test_layernorm_modulate_grouped_bwd_against_formulas(D, G, R, gin):
    from fastvideo_b200 import ops
    torch.manual_seed(D + G)
    M = G * R - 5  # the last group is shorter
    x = (torch.randn(M, D, device="cuda") * 2 + 0.3).bfloat16()
    dn = torch.randn(M, D, device="cuda").bfloat16()
    e = (torch.randn(G, 6, D, device="cuda") * 0.5).bfloat16().float()
    scale = e[:, 1]
    gi = None if gin is None else torch.randn(M, D, device="cuda").to(torch.float32 if gin == "f32" else torch.bfloat16)
    dx, ds, dsh = ops.layernorm_modulate_grouped_bwd(x, dn, scale, R, gin=gi)
    # restatement at the rounding points: t = bf16(LN(x)), G = bf16(1 + scale), dt = bf16(dn G)
    xf = x.float().double()
    mean = xf.mean(1, keepdim=True)
    rstd = 1 / torch.sqrt(((xf - mean) ** 2).mean(1, keepdim=True) + 1e-6)
    xh = (xf - mean) * rstd
    grp = torch.arange(M, device="cuda") // R
    Gv = _bf(1 + scale)[grp].double()
    dt = _bf(dn.float() * Gv.float()).double()
    want = rstd * (dt - dt.mean(1, keepdim=True) - xh * (dt * xh).mean(1, keepdim=True))
    if gi is not None:
        want = want + gi.double()
    assert _ulp_close(dx, want.to(torch.bfloat16)), (dx.float() - want.float()).abs().max()
    t = _bf(xh.float()).double()
    z = lambda v: torch.zeros(G, D, dtype=torch.float64, device="cuda").index_add_(0, grp, v)
    ws, wh = z(dn.double() * t), z(dn.double())
    assert _sum_close(ds, ws, z((dn.double() * t).abs())) and _sum_close(dsh, wh, z(dn.double().abs()))
    # deterministic: a second call gives the same bits
    dx2, ds2, dsh2 = ops.layernorm_modulate_grouped_bwd(x, dn, scale, R, gin=gi)
    assert torch.equal(dx, dx2) and torch.equal(ds, ds2) and torch.equal(dsh, dsh2)


@pytest.mark.parametrize("N,G,R", [(1536, 3, 40), (5120, 4, 24), (1536, 21, 77)])
def test_resid_gate_grouped_bwd_against_formulas(N, G, R):
    from fastvideo_b200 import ops
    torch.manual_seed(N + G)
    M = G * R - 3
    dout = torch.randn(M, N, device="cuda").bfloat16()
    y = torch.randn(M, N, device="cuda").bfloat16()
    gate = (torch.randn(G, 6, N, device="cuda")).bfloat16().float()[:, 2]
    dy, dg, db = ops.resid_gate_grouped_bwd(dout, y, gate, R)
    grp = torch.arange(M, device="cuda") // R
    want_dy = (dout.float() * gate[grp]).bfloat16()
    assert torch.equal(dy, want_dy)
    z = lambda v: torch.zeros(G, N, dtype=torch.float64, device="cuda").index_add_(0, grp, v)
    prod = dout.double() * y.double()
    assert _sum_close(dg, z(prod), z(prod.abs()))
    assert rel_l2(db, want_dy.double().sum(0)) < 4e-3  # one bf16 rounding of an fp32 sum
    dy2, dg2, db2 = ops.resid_gate_grouped_bwd(dout, y, gate, R)
    assert torch.equal(dy, dy2) and torch.equal(dg, dg2) and torch.equal(db, db2)


@pytest.mark.parametrize("N", [1536, 256, 64])
def test_linear_aux_rounded_per_frame_gate_bit_equal(N):
    from fastvideo_b200 import ops
    torch.manual_seed(N)
    F_, tpf, K = 3, 50, 256
    x = torch.randn(F_ * tpf, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    resid = torch.randn(F_ * tpf, N, device="cuda").bfloat16()
    gate = torch.randn(F_, 6, N, device="cuda").bfloat16().float()[:, 2]
    out, aux = ops.linear_aux(x, w, b, ops.EPI_RESID_GATE_BF16R, resid=resid, gate=gate, gate_rows=tpf)
    assert torch.equal(out, ops.linear(x, w, b, ops.EPI_RESID_GATE_BF16R, resid=resid, gate=gate, gate_rows=tpf))
    assert torch.equal(aux, ops.linear(x, w, b))


@pytest.mark.parametrize("frames,fs,n,local", [(5, 24, 2, -1), (7, 40, 3, 4), (21, 1560, 3, -1)])
def test_device_lists_select_the_token_mask(frames, fs, n, local):
    from fastvideo_b200 import wan_dit
    c = wan_dit.block_causal_tiles(frames, fs, n, local, "cuda")
    nqb, nkb = c.q_off.numel() - 1, c.nkb
    m = torch.zeros(nqb, nkb, dtype=torch.bool)
    for i, (cnt, row) in enumerate(zip(c.q2k_num[0, 0].cpu(), c.q2k_idx[0, 0].cpu())):
        m[i, row[:cnt].long()] = True
        assert (row[:cnt].diff() > 0).all()
    mt = torch.zeros(nkb, nqb, dtype=torch.bool)
    for j, (cnt, row) in enumerate(zip(c.k2q_num[0, 0].cpu(), c.k2q_idx[0, 0].cpu())):
        mt[j, row[:cnt].long()] = True
    assert torch.equal(m, c.tile_map[0, 0].cpu()) and torch.equal(mt, m.T)
    qo, ko = c.q_off.cpu(), c.kv_off.cpu()
    qt = torch.repeat_interleave(torch.arange(nqb), (qo[1:] - qo[:-1]).long())
    kt = torch.repeat_interleave(torch.arange(nkb), (ko[1:] - ko[:-1]).long())
    assert torch.equal(m[qt][:, kt], block_causal_mask(frames, fs, n, local))


# ---------------------------------------------------------------------------------------------------------------- model
def _case(kind, golden_dir):
    """dict(sd (CPU, reference names), latents, text, timestep [B, F], heads, text_len, n, local)."""
    from fastvideo_b200 import wan_dit
    gen = torch.Generator().manual_seed(11)
    if kind == "wide":  # Wan 1.3B width, 2 layers, a small grid
        cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_1_3B, "num_layers": 2})
        sd = _perturb(wan_dit.random_state_dict(cfg, "cpu", 31, layers=2), 6)
        return dict(sd=sd, latents=torch.randn(1, 16, 4, 8, 8, generator=gen).bfloat16(),
                    text=torch.randn(1, 40, cfg.text_dim, generator=gen).bfloat16(), timestep=torch.tensor([[900, 700, 500, 300]]),
                    heads=cfg.num_attention_heads, text_len=64, n=3, local=-1)
    g = torch.load(os.path.join(golden_dir, "wan_causal_model.pt"))
    B = 2 if kind == "batch2" else 1
    F_ = 5 if kind in ("golden_n2", "batch2") else 7
    t = torch.randint(0, 1000, (B, F_), generator=gen)
    return dict(sd=dict(g["sd"]), latents=torch.randn(B, 16, F_, 8, 12, generator=gen).bfloat16(),
                text=torch.randn(B, g["text"].shape[1], g["text"].shape[2], generator=gen).bfloat16(), timestep=t,
                heads=g["heads"], text_len=g["text_len"], n=3 if kind == "golden_n3" else 2,
                local=4 if kind == "local" else -1)


def _model(case, train=True, layers=None):
    from fastvideo_b200 import causal_wan, wan_dit
    sd = case["sd"]
    D = sd["proj_out.weight"].shape[1]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=case["heads"], ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0],
                               num_layers=2, text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1],
                               text_len=case["text_len"])
    model = causal_wan.CausalWanDiT(cfg, {k: v.cuda() for k, v in sd.items()},
                                    causal_wan.CausalConfig(local_attn_size=case["local"], num_frames_per_block=case["n"]))
    if train:
        for t in model.tensors().values():
            t.requires_grad_(True)
    return model


def _oracle(case, dtype, device="cpu"):
    sd = {k: v.to(device, dtype) for k, v in case["sd"].items()}
    with torch.no_grad():
        return causal_model_train(case["latents"].to(device, dtype), case["text"].to(device, dtype), case["timestep"].to(device),
                                  sd, case["heads"], case["n"], local_attn_size=case["local"], text_len=case["text_len"])


@pytest.mark.parametrize("kind", ["golden_n2", "golden_n3", "wide", "batch2", "local"])
def test_forward_train_parity(golden_dir, kind):
    case = _case(kind, golden_dir)
    model = _model(case, train=False)
    with torch.no_grad():
        y = model.forward_train(case["latents"].cuda(), case["text"].cuda(), case["timestep"].cuda())
    assert y.shape == case["latents"].shape and y.dtype == torch.bfloat16
    assert_bf16_parity(y, _oracle(case, torch.float32), _oracle(case, torch.bfloat16), name=kind)


def test_forward_train_matches_the_engine_rollout(golden_dir):
    """Frame block b of forward_train against the engine's own forward_inference rollout over blocks 0..b (same latents and
    timesteps): within the bf16 parity bound of the fp32 training oracle."""
    case = _case("golden_n2", golden_dir)
    model = _model(case, train=False)
    lat, text, t = case["latents"].cuda(), case["text"].cuda(), case["timestep"].cuda()
    fs = (lat.shape[3] // 2) * (lat.shape[4] // 2)
    ref32, ref16 = _oracle(case, torch.float32), _oracle(case, torch.bfloat16)
    with torch.no_grad():
        y = model.forward_train(lat, text, t)
        kv, xc = model.new_caches(fs, "cuda")
        for f0 in range(0, lat.shape[2], case["n"]):
            f1 = min(f0 + case["n"], lat.shape[2])
            r = model.forward_inference(lat[:, :, f0:f1].contiguous(), text, t[:, f0:f1], kv, xc, current_start=f0 * fs,
                                        start_frame=f0)
            blk = (slice(None), slice(None), slice(f0, f1))
            e, floor = assert_bf16_parity(r, ref32[blk], ref16[blk], name=f"rollout block at frame {f0}")
            assert_bf16_parity(y[blk], ref32[blk], ref16[blk], name=f"training forward block at frame {f0}")
            assert rel_l2(y[:, :, f0:f1], r) <= 2 * floor + 5e-3


def _run(model, case, dy, checkpoint):
    lat = case["latents"].cuda().requires_grad_(True)
    text = case["text"].cuda().requires_grad_(True)
    y = model.forward_train(lat, text, case["timestep"].cuda(), checkpoint=checkpoint)
    assert y.grad_fn is not None
    y.backward(dy)
    grads = model.to_reference_names({n: t.grad for n, t in model.tensors().items()})
    grads.update(latents=lat.grad, text=text.grad)
    for t in model.tensors().values():
        t.grad = None
    return y.detach(), grads


def _oracle_grads(case, dtype, dy, device):
    """Gradients of every parameter, latents and text (+ "out:<bias>" for the key biases' projection outputs)."""
    sd = {k: v.to(device, dtype).requires_grad_(True) for k, v in case["sd"].items()}
    ins = {k: case[k].to(device, dtype).requires_grad_(True) for k in ("latents", "text")}
    outs, lin = {}, causal_train_ref.linear
    key_biases = [k for k in sd if k.endswith(KEY_BIASES)]

    def keep_key_outputs(x, w, b):
        y = lin(x, w, b)
        for k in key_biases:
            if b is sd[k]:
                y.retain_grad()
                outs["out:" + k] = y
        return y

    causal_train_ref.linear = keep_key_outputs
    try:
        with torch.device(device):
            y = causal_model_train(ins["latents"], ins["text"], case["timestep"].to(device), sd, case["heads"], case["n"],
                                   local_attn_size=case["local"], text_len=case["text_len"])
    finally:
        causal_train_ref.linear = lin
    y.backward(dy.to(device, y.dtype))
    return {**{k: t.grad for k, t in ins.items()}, **{k: t.grad for k, t in sd.items()},
            **{k: t.grad for k, t in outs.items()}}


@pytest.mark.parametrize("kind", ["golden_n3", "wide", "batch2", "local"])
def test_gradients_against_fp32_autograd(golden_dir, kind):
    case = _case(kind, golden_dir)
    if kind != "wide":
        case["sd"] = _perturb(case["sd"], 3)
    dy = torch.randn(case["latents"].shape, generator=torch.Generator().manual_seed(1)).bfloat16().cuda()
    _, ours = _run(_model(case), case, dy, checkpoint=True)
    truth = _oracle_grads(case, torch.float32, dy, "cuda")
    floor = _oracle_grads(case, torch.bfloat16, dy, "cuda")
    # Named exceptions, the rule of test_model_gradients_against_fp32_autograd (tests/test_gpu_model_bwd.py): gradients that
    # are mostly rounding noise, where two bf16 torch pipelines (SDPA's default and its math backend) sit about as far apart
    # as each is from fp32. They are held to the default pipeline's distance plus the two pipelines' spread, and the test
    # checks that the spread is there (more than half that distance). At the 1.3B width: the last block's self-attention q /
    # k gradients, as in the bidirectional model. With the 4-frame window: the first block's norm2 bias and cross-attention
    # query bias, column sums over every token of the same cross-attention query gradient.
    noisy = {"wide": {"blocks.1." + n for n in ("to_q.weight", "to_q.bias", "to_k.weight", "norm_q.weight", "norm_k.weight")},
             "local": {"blocks.0.attn2.to_q.bias", "blocks.0.self_attn_residual_norm.norm.bias"}}.get(kind, set())
    if noisy:
        from torch.nn.attention import SDPBackend, sdpa_kernel
        with sdpa_kernel(SDPBackend.MATH):
            other = _oracle_grads(case, torch.bfloat16, dy, "cuda")
    bad, checked = [], 0
    for k, t in truth.items():
        if k.startswith("out:"):
            continue
        got = ours[k]
        assert got is not None and torch.isfinite(got.float()).all(), k
        assert got.shape == t.shape, (k, got.shape, t.shape)
        e, fl = rel_l2(got, t), rel_l2(floor[k], t)
        if k.endswith(KEY_BIASES):  # the key biases' gradient is ~0 in exact arithmetic: see test_gpu_block_bwd.py
            up = "out:" + k
            if not e <= max(fl, rel_l2(floor[up], truth[up])) * 3 + TOL:
                bad.append(f"{k}: relL2 {e:.3e} (bf16 autograd {fl:.3e})")
        elif k in noisy:
            spread = rel_l2(other[k], floor[k])
            assert spread > fl / 2, f"{k}: the two bf16 pipelines agree ({spread:.3e}, fp32 distance {fl:.3e})"
            if not e <= fl + spread:
                bad.append(f"{k}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + pipeline spread {spread:.3e}")
        elif not e <= fl + TOL:
            bad.append(f"{k}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + {TOL}")
        checked += 1
    assert not bad, "; ".join(bad)
    assert checked == len(case["sd"]) + 2


def test_bits_checkpoint_and_determinism(golden_dir):
    """Forward under grad (checkpoint off and on) = the no-grad forward; checkpointed gradients = the others; a second
    backward gives the same bits; the checkpointed backward launches no self-attention (cross-attention once per block)."""
    from fastvideo_b200 import ops
    case = _case("golden_n3", golden_dir)
    args = (case["latents"].cuda(), case["text"].cuda(), case["timestep"].cuda())
    with torch.no_grad():
        plain = _model(case, train=False).forward_train(*args)
    dy = torch.randn(plain.shape, generator=torch.Generator().manual_seed(2)).bfloat16().cuda()
    model = _model(case)
    y0, g0 = _run(model, case, dy, checkpoint=False)
    y1, g1 = _run(model, case, dy, checkpoint=True)
    y2, g2 = _run(model, case, dy, checkpoint=True)
    for y_ in (y0, y1, y2):
        assert torch.equal(y_, plain)
    assert sorted(g0) == sorted(g1) == sorted(g2)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
        assert torch.equal(g1[k], g2[k]), k
    calls = dict(blocklist=0, cross=0)
    blocklist, attention = ops.attention_blocklist, ops.attention

    def counted_blocklist(*a, **kw):
        calls["blocklist"] += 1
        return blocklist(*a, **kw)

    def counted_attention(*a, **kw):
        calls["cross"] += 1
        return attention(*a, **kw)

    ops.attention_blocklist, ops.attention = counted_blocklist, counted_attention
    try:
        lat = args[0].clone().requires_grad_(True)
        y = model.forward_train(lat, *args[1:], checkpoint=True)
        assert calls == dict(blocklist=2, cross=2)
        calls.update(blocklist=0, cross=0)
        y.backward(dy)
    finally:
        ops.attention_blocklist, ops.attention = blocklist, attention
    assert calls == dict(blocklist=0, cross=2), calls


def test_memory_kept_per_causal_block():
    """memory_allocated() held between forward and backward at D 1536, 7 frames of 384 tokens (n = 3): per checkpointed
    block at most checkpoint_bytes_per_block(..., frames=7) + 1 MiB."""
    from fastvideo_b200 import causal_wan, wan_dit
    F_, fs, L = 7, 384, 128
    S = F_ * fs
    gen = torch.Generator(device="cuda").manual_seed(0)
    lat = torch.randn(1, 16, F_, 32, 48, device="cuda", generator=gen).bfloat16()
    text = torch.randn(1, L, 256, device="cuda", generator=gen).bfloat16()
    t = torch.randint(0, 1000, (1, F_), device="cuda", generator=gen)
    held = {}
    for layers in (2, 6):
        cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_1_3B, "num_layers": layers, "text_dim": 256, "text_len": L})
        model = causal_wan.CausalWanDiT.random(cfg, causal_wan.CausalConfig(num_frames_per_block=3), "cuda", 3)
        for p in model.tensors().values():
            p.requires_grad_(True)
        dy = torch.randn(lat.shape, device="cuda", generator=gen).bfloat16()
        model.forward_train(lat, text, t, checkpoint=True).backward(dy)  # warm-up
        for p in model.tensors().values():
            p.grad = None
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        y = model.forward_train(lat, text, t, checkpoint=True)
        torch.cuda.synchronize()
        held[layers] = torch.cuda.memory_allocated() - base
        del y, model
        torch.cuda.empty_cache()
    formula = wan_dit.checkpoint_bytes_per_block(S, 1536, 12, frames=F_)
    per_block = (held[6] - held[2]) / 4
    assert formula - 2 ** 20 <= per_block <= formula + 2 ** 20, (per_block, formula)
