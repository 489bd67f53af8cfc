"""CPU: the W8A8 INT8 restatement (tests/w8a8_ref.py) -- the activation quantiser's rounding, zero rows and clamp, the exact
integer accumulation and the epilogue's rounding order, and how far W8A8 moves the oracle from fp32 next to bf16, INT8 weights
and FP8 linears -- plus the host-side pieces of the option: the int8-activation mark on ops.Int8Weight, WanDiTConfig's
validation and the plug-in config.

Distance (relative L2) of each bf16 restatement from the fp32 oracle, measured on the golden fixtures (causal rows: the worst
call of the rollout). The bounds below leave about 30 % above the measured W8A8 values. The activations of the random
fixtures have no outlier channels, so these say nothing about real checkpoints.

| case                  | bf16    | INT8 weights | W8A8    | FP8 linears |
|-----------------------|---------|--------------|---------|-------------|
| block                 | 3.5e-3  | 6.5e-3       | 9.2e-3  | 2.7e-2      |
| I2V block             | 3.6e-3  | 7.1e-3       | 9.8e-3  | 2.7e-2      |
| 2-layer model         | 5.6e-3  | 7.6e-3       | 9.0e-3  | 2.1e-2      |
| causal block rollout  | 4.1e-3  | 7.1e-3       | 9.9e-3  | --          |
| causal model rollout  | 6.3e-3  | 8.2e-3       | 9.4e-3  | --          |
"""
import os

import pytest
import torch

import fp8_ref
import w8_ref
import w8a8_ref
from oracle import causal_ref, ref_shim, wan_ref
from util import rel_l2

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


# ------------------------------------------------------------------------------------------------ restatement
def test_activation_rows_ties_to_even_clamp_and_zero_rows():
    # amax 127 -> inv = 1 exactly: ties go to the even integer, the amax element to 127
    x = torch.tensor([[127.0, 0.5, 1.5, 2.5, -0.5, -1.5, 126.5, -126.5],
                      [0.0] * 8,
                      [-3.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]]).bfloat16()
    q, s = w8a8_ref.quantize_rows(x.view(1, 3, 8))  # leading dimensions are kept
    q, s = q[0], s[0]
    assert q.dtype == torch.int8 and s.dtype == torch.float32 and s.shape == (3,)
    assert s[0].item() == 1.0 and q[0].tolist() == [127, 0, 2, 2, 0, -2, 126, -126]
    assert s[1].item() == 1.0 and (q[1] == 0).all()
    assert q[2, 0].item() == -127 and q[2, 7].item() == 42  # 1 * (127 / 3) = 42.33
    assert s[2] == torch.tensor(3.0) / torch.tensor(127.0)
    # amaxes where amax * (127 / amax) rounds above 127 in fp32 still give +-127, never 128
    for a in torch.linspace(1.0, 1000.0, 2001).bfloat16().float().unique().tolist():
        qa, _ = w8a8_ref.quantize_rows(torch.tensor([[a, -a]]))
        assert qa[0].tolist() == [127, -127], a


def test_accumulator_is_exact_and_bounded():
    assert 127 ** 2 * w8a8_ref.MAX_K < 2 ** 31 <= 127 ** 2 * (w8a8_ref.MAX_K + 1)
    K = 13824
    xq = torch.full((2, K), 127, dtype=torch.int8)
    xq[1] = -127
    q = torch.full((3, K), -127, dtype=torch.int8)
    acc = w8a8_ref.w8a8_acc(xq, q)
    assert acc.dtype == torch.int64 and acc[0, 0].item() == -127 * 127 * K and acc[1, 2].item() == 127 * 127 * K


def test_linear_rounding_order():
    torch.manual_seed(3)
    x = torch.randn(5, 96).bfloat16()
    w = (torch.randn(24, 96) / 10).bfloat16()
    b = torch.randn(24).bfloat16()
    q, s = w8_ref.quantize_int8_rows(w)
    y, acc, xs = w8a8_ref.w8a8_linear_f32(x, q, s, b)
    xq, xs2 = w8a8_ref.quantize_rows(x)
    assert torch.equal(xs, xs2)
    for m in range(5):
        for n in range(24):
            a = float(sum(int(xq[m, k]) * int(q[n, k]) for k in range(96)))
            v = torch.tensor(a, dtype=torch.float32)
            v = (v * xs[m]) * s[n]
            v = v + b[n].float()
            assert v.item() == y[m, n].item()
    assert w8a8_ref.linear_w8a8(x, q, s, b).dtype == torch.bfloat16


# ------------------------------------------------------------------------------------------------ host side
def test_int8_weight_activation_mark_survives_row_slices():
    from fastvideo_b200 import ops
    w = (torch.randn(96, 64) / 8).bfloat16()
    plain, marked = ops.Int8Weight.quantize(w), ops.Int8Weight.quantize(w, int8_activations=True)
    assert not plain.int8_activations and marked.int8_activations
    assert torch.equal(plain.q, marked.q) and torch.equal(plain.scale, marked.scale) and plain.nbytes == marked.nbytes
    assert marked[32:64].int8_activations and marked[64:].int8_activations and not plain[:32].int8_activations
    assert ops.Int8Weight(marked.q, marked.scale, int8_activations=True)[0:8].int8_activations


def test_config_int8_activations_needs_int8_weights():
    from fastvideo_b200 import ops, wan_dit
    with pytest.raises(ops.FvbError):
        wan_dit.WanDiTConfig(int8_activations=True)
    with pytest.raises(ops.FvbError):
        wan_dit.WanDiTConfig(int8_activations=True, fp8_linears=True)
    with pytest.raises(ops.FvbError):
        wan_dit.WanDiTConfig(int8_activations=True, int8_weights=True, fp8_linears=True)
    cfg = wan_dit.WanDiTConfig(int8_weights=True, int8_activations=True, vsa=True, attention_8bit=True)
    assert cfg.int8_weights and cfg.int8_activations and not cfg.fp8_linears
    assert not wan_dit.WanDiTConfig(int8_weights=True).int8_activations


def test_block_marks_every_int8_linear():
    from fastvideo_b200 import ops, wan_dit
    g = torch.load(os.path.join(GOLDEN, "wan_block_i2v.pt"))
    D = g["x"].shape[-1]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1, int8_weights=True, int8_activations=True)
    blk = wan_dit.WanBlock(g["sd"], "", cfg)
    for n in wan_dit.INT8_LINEARS:
        w = getattr(blk, n)
        assert isinstance(w, ops.Int8Weight) and w.int8_activations, n


# ------------------------------------------------------------------------------------------------ oracle routing
def test_block_routing_touches_exactly_the_block_linears(monkeypatch):
    g = torch.load(os.path.join(GOLDEN, "wan_block_i2v.pt"))
    seen = []
    orig = w8a8_ref.linear_w8a8
    monkeypatch.setattr(w8a8_ref, "linear_w8a8", lambda x, q, s, b: seen.append(q.shape) or orig(x, q, s, b))
    cos, sin = wan_ref.rotary_tables(g["seq"], [44, 42, 42])
    with torch.no_grad():
        w8a8_ref.wan_block_w8a8(g["x"], g["ctx"], g["temb6"], g["sd"], "", g["heads"], cos, sin)
    want = sorted(tuple(g["sd"][n + ".weight"].shape) for n in w8_ref.BLOCK_LINEARS if n + ".weight" in g["sd"])
    assert sorted(seen) == want and len(seen) == 12
    assert wan_ref.linear.__name__ == "linear"  # restored


# ------------------------------------------------------------------------------------------------ distance from fp32
@pytest.mark.parametrize("name,bound", [("wan_block_dense", 1.2e-2), ("wan_block_i2v", 1.3e-2)])
def test_block_distance_from_fp32(name, bound):
    g = torch.load(os.path.join(GOLDEN, name + ".pt"))
    cos, sin = wan_ref.rotary_tables(g["seq"], [44, 42, 42])
    H, ref = g["heads"], g["y_fp32"]
    with torch.no_grad():
        a = w8a8_ref.wan_block_w8a8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
        w = w8_ref.wan_block_w8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
        f8 = fp8_ref.wan_block_fp8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
    e_bf16, e_w8, e_a8, e_f8 = (rel_l2(t, ref) for t in (g["y_ref_bf16"], w, a, f8))
    print(f"{name} relL2 from fp32: bf16 {e_bf16:.2e}, int8 weights {e_w8:.2e}, w8a8 {e_a8:.2e}, fp8 {e_f8:.2e}")
    assert e_w8 < e_a8 < bound and e_a8 < e_f8 / 2


def test_model_distance_from_fp32():
    g = torch.load(os.path.join(GOLDEN, "wan_model_dense.pt"))
    with torch.no_grad():
        a = w8a8_ref.wan_model_w8a8(g["latents"], g["text"], g["timestep"], g["sd"], g["heads"])
    e = rel_l2(a, g["y_fp32"])
    print(f"wan_model_dense relL2 from fp32: bf16 {rel_l2(g['y_ref_bf16'], g['y_fp32']):.2e}, w8a8 {e:.2e}")
    assert e < 1.2e-2


def test_causal_block_distance_from_fp32():
    g = torch.load(os.path.join(GOLDEN, "wan_causal_block.pt"))
    H, grid, nf = g["heads"], tuple(g["grid"]), g["frames_per_call"]
    fs = grid[0] * grid[1]
    caches = {k: causal_ref.new_kv_cache(1, g["window_frames"] * fs, H, 128) for k in ("w8", "w8a8")}
    xcs = {k: {"is_init": False} for k in caches}
    fns = {"w8": w8_ref.causal_block_w8, "w8a8": w8a8_ref.causal_block_w8a8}
    worst = {"bf16": 0.0, "w8": 0.0, "w8a8": 0.0}
    for c in g["calls"]:
        cos, sin = wan_ref.rotary_tables((nf, ) + grid, [44, 42, 42], start_frame=c["start_frame"], keep_f64=True)
        worst["bf16"] = max(worst["bf16"], rel_l2(c["y_ref_bf16"], c["y_fp32"]))
        for k, fn in fns.items():
            with torch.no_grad():
                y = fn(c["x"], g["ctx"], c["temb"], g["sd"], "", H, cos, sin, caches[k], c["start_frame"] * fs,
                       g["window_frames"], g["sink_frames"], fs, crossattn_cache=xcs[k])
            worst[k] = max(worst[k], rel_l2(y, c["y_fp32"]))
    print("causal block rollout, worst call relL2 from fp32: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert worst["w8"] < worst["w8a8"] < 1.3e-2


def test_causal_model_distance_from_fp32():
    g = torch.load(os.path.join(GOLDEN, "wan_causal_model.pt"))
    H, window, sink = g["heads"], g["window_frames"], g["sink_frames"]
    c0 = g["calls"][0]["latents"]
    fs = (c0.shape[3] // 2) * (c0.shape[4] // 2)
    fns = {"w8": w8_ref.causal_model_w8, "w8a8": w8a8_ref.causal_model_w8a8}
    kvs = {k: [causal_ref.new_kv_cache(1, window * fs, H, 128) for _ in range(2)] for k in fns}
    xcs = {k: [{"is_init": False} for _ in range(2)] for k in fns}
    worst = {"bf16": 0.0, "w8": 0.0, "w8a8": 0.0}
    for c in g["calls"]:
        worst["bf16"] = max(worst["bf16"], rel_l2(c["y_ref_bf16"], c["y_fp32"]))
        for k, fn in fns.items():
            with torch.no_grad():
                y = fn(c["latents"], g["text"], c["timestep"], g["sd"], H, kvs[k], xcs[k], current_start=c["start_frame"] * fs,
                       start_frame=c["start_frame"], local_attn_size=window, sink_size=sink, text_len=g["text_len"])
            worst[k] = max(worst[k], rel_l2(y, c["y_fp32"]))
    print("causal model rollout, worst call relL2 from fp32: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))
    assert worst["w8"] < worst["w8a8"] < 1.3e-2


# ------------------------------------------------------------------------------------------------ plug-in
@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present (set FVB_REFERENCE_ROOT or stage oracle/_ref/reference_py)")
def test_plugin_w8a8_config_resolves_on_sm90(monkeypatch):
    ref_shim.install()
    from fastvideo_b200 import plugin as p
    p.install(force=True)
    try:
        monkeypatch.setattr(torch.cuda, "get_device_capability", lambda *a, **k: (9, 0))
        from fastvideo.layers.linear import LinearMethodBase, ReplicatedLinear
        from fastvideo.layers.quantization import get_quantization_config
        from fastvideo_b200._lib import FvbError
        cfg_cls = get_quantization_config(p.QUANT_NAME_W8A8)
        assert cfg_cls.__name__ == "Fvb200W8A8Config" and cfg_cls.get_min_capability() == 90
        assert cfg_cls().get_name() == "fvb200_w8a8"
        lin = ReplicatedLinear(256, 384, bias=True, params_dtype=torch.bfloat16, quant_config=cfg_cls(), prefix="blocks.0.to_q")
        assert type(lin.quant_method).__name__ == "Fvb200W8A8LinearMethod"
        assert isinstance(lin.quant_method, LinearMethodBase) and lin.quant_method.int8_activations
        assert tuple(lin.weight.shape) == (384, 256) and lin.weight.dtype == torch.bfloat16
        with pytest.raises(FvbError):
            lin.quant_method.process_weights_after_loading(lin)  # CPU weights: quantised on the GPU only
        with pytest.raises(FvbError):
            lin(torch.zeros(2, 5, 256, dtype=torch.bfloat16))
    finally:
        p.uninstall()
