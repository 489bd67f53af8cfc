"""CPU: the INT8 weight-only restatement (tests/w8_ref.py) -- the quantiser's rounding, zero rows and clamp, which linears of the
block restatements it routes, and how far INT8 weights move the oracle from fp32 compared with bf16 and FP8 -- plus the
host-side pieces of the option: ops.Int8Weight, WanDiTConfig's exclusivity with fp8_linears and the plug-in config."""
import os

import pytest
import torch

import fp8_ref
import w8_ref
from oracle import causal_ref, ref_shim, wan_ref
from util import rel_l2

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


# ------------------------------------------------------------------------------------------------ quantiser
def test_round_trip_within_half_a_step():
    torch.manual_seed(0)
    w = (torch.randn(64, 320) * torch.logspace(-3, 2, 64)[:, None]).bfloat16()
    q, s = w8_ref.quantize_int8_rows(w)
    assert q.dtype == torch.int8 and s.dtype == torch.float32 and s.shape == (64,)
    err = (q.double() * s.double()[:, None] - w.double()).abs()
    # half a step, plus the fp32 rounding of scale and of w * (127 / amax): a few ulps of 127 steps
    assert (err <= s.double()[:, None] * (0.5 + 127 * 2.0 ** -21)).all()
    assert (err > 0.49 * s.double()[:, None]).any()  # and the bound is not loose
    assert (q.abs().amax(dim=1) == 127).all()  # each row's amax element maps to +-127


def test_rint_ties_to_even_and_clamp():
    # amax 127 -> inv = 1 exactly, so the elements are rounded unscaled: ties go to the even integer
    w = torch.tensor([[127.0, 0.5, 1.5, 2.5, -0.5, -1.5, 126.5]])
    q, s = w8_ref.quantize_int8_rows(w)
    assert s.item() == 1.0 and q[0].tolist() == [127, 0, 2, 2, 0, -2, 126]
    # amaxes where amax * (127 / amax) rounds above 127 in fp32: the element equal to amax must still give +-127
    found = 0
    for a in torch.linspace(1.0, 1000.0, 4001).bfloat16().float().unique().tolist():
        if float(torch.tensor(a) * (torch.tensor(127.0) / torch.tensor(a))) > 127.0:
            q, _ = w8_ref.quantize_int8_rows(torch.tensor([[a, -a, a / 3]]))
            assert q[0, :2].tolist() == [127, -127], a
            found += 1
    assert found > 0


def test_zero_rows():
    w = torch.zeros(3, 48, dtype=torch.bfloat16)
    w[1, 7] = -0.25
    q, s = w8_ref.quantize_int8_rows(w)
    assert s[0] == 1.0 and s[2] == 1.0 and (q[0] == 0).all() and (q[2] == 0).all()
    assert s[1] == torch.tensor(0.25) / torch.tensor(127.0) and q[1, 7] == -127


def test_int8_weight_quantize_matches_restatement():
    from fastvideo_b200 import ops
    torch.manual_seed(1)
    w = (torch.randn(40, 200) * 0.02).bfloat16()
    w[3] = 0
    iw = ops.Int8Weight.quantize(w)
    q, s = w8_ref.quantize_int8_rows(w)
    assert iw.q.shape == (40, 200) and iw.q.stride(0) % 16 == 0  # 200 is padded to 16-byte rows
    assert torch.equal(iw.q, q) and torch.equal(iw.scale.view(torch.int32), s.view(torch.int32))
    assert iw.nbytes == 40 * 200 + 40 * 4


def test_int8_weight_validation_and_row_slices():
    from fastvideo_b200 import ops
    q = torch.zeros(96, 64, dtype=torch.int8)
    s = torch.arange(96, dtype=torch.float32)
    w = ops.Int8Weight(q, s)
    part = w[32:64]
    assert part.shape == (32, 64) and torch.equal(part.scale, s[32:64]) and part.q.data_ptr() == q[32].data_ptr()
    assert w[64:].shape == (32, 64) and w[:32].scale[0] == 0.0
    with pytest.raises(ops.FvbError):
        w[::2]
    with pytest.raises(ops.FvbError):
        ops.Int8Weight(q.float(), s)                       # not int8
    with pytest.raises(ops.FvbError):
        ops.Int8Weight(torch.zeros(8, 40, dtype=torch.int8)[:, :20], s[:8])  # 40-byte rows: not 16-byte aligned
    with pytest.raises(ops.FvbError):
        ops.Int8Weight(q, s[:95])                          # one scale per row
    with pytest.raises(ops.FvbError):
        ops.Int8Weight(q, s.double())


def test_config_int8_weights_and_fp8_linears_exclusive():
    from fastvideo_b200 import ops, wan_dit
    with pytest.raises(ops.FvbError):
        wan_dit.WanDiTConfig(int8_weights=True, fp8_linears=True)
    cfg = wan_dit.WanDiTConfig(int8_weights=True, vsa=True, attention_8bit=True)
    assert cfg.int8_weights and not cfg.fp8_linears


# ------------------------------------------------------------------------------------------------ oracle routing
def _record(monkeypatch):
    seen = []
    orig = w8_ref.linear_w8

    def spy(x, q, s, b):
        seen.append(q.shape)
        return orig(x, q, s, b)
    monkeypatch.setattr(w8_ref, "linear_w8", spy)
    return seen


def _expected(sd, prefix):
    return sorted(tuple(sd[prefix + n + ".weight"].shape) for n in w8_ref.BLOCK_LINEARS if prefix + n + ".weight" in sd)


@pytest.mark.parametrize("name", ["wan_block_dense", "wan_block_i2v"])
def test_block_routing_touches_exactly_the_block_linears(monkeypatch, name):
    g = torch.load(os.path.join(GOLDEN, name + ".pt"))
    seen = _record(monkeypatch)
    cos, sin = wan_ref.rotary_tables(g["seq"], [44, 42, 42])
    with torch.no_grad():
        y = w8_ref.wan_block_w8(g["x"], g["ctx"], g["temb6"], g["sd"], "", g["heads"], cos, sin)
    assert sorted(seen) == _expected(g["sd"], "")
    assert len(seen) == (12 if name == "wan_block_i2v" else 10)
    assert wan_ref.linear is not None and wan_ref.linear.__name__ == "linear"  # restored
    assert 0 < rel_l2(y, g["y_ref_bf16"]) < 2e-2


def test_causal_block_routing_touches_exactly_the_block_linears(monkeypatch):
    g = torch.load(os.path.join(GOLDEN, "wan_causal_block.pt"))
    grid, nf = tuple(g["grid"]), g["frames_per_call"]
    fs = grid[0] * grid[1]
    c = g["calls"][0]
    seen = _record(monkeypatch)
    cache = causal_ref.new_kv_cache(1, g["window_frames"] * fs, g["heads"], 128)
    cos, sin = wan_ref.rotary_tables((nf, ) + grid, [44, 42, 42], start_frame=c["start_frame"], keep_f64=True)
    with torch.no_grad():
        y = w8_ref.causal_block_w8(c["x"], g["ctx"], c["temb"], g["sd"], "", g["heads"], cos, sin, cache,
                                   c["start_frame"] * fs, g["window_frames"], g["sink_frames"], fs, crossattn_cache=None)
    assert sorted(seen) == _expected(g["sd"], "") and len(seen) == 10
    assert causal_ref._lin.__name__ == "_lin"  # restored
    assert 0 < rel_l2(y, c["y_ref_bf16"]) < 2e-2


# ------------------------------------------------------------------------------------------------ distance from fp32
def test_int8_weights_are_closer_to_fp32_than_fp8_linears():
    """On the golden fixtures (bf16 restatements, distance from the fp32 oracle): bf16 3.5e-3 / 5.6e-3, INT8 weights
    6.5e-3 / 7.6e-3, FP8 linears 2.7e-2 / 2.1e-2 for the dense block / 2-layer model. The int8 step (amax / 127) is
    about 10x finer than e4m3's 3-bit mantissa, and the activations stay bf16."""
    f32 = lambda sd: {k: v.float() for k, v in sd.items()}
    g = torch.load(os.path.join(GOLDEN, "wan_block_dense.pt"))
    cos, sin = wan_ref.rotary_tables(g["seq"], [44, 42, 42])
    H, ref = g["heads"], g["y_fp32"]
    with torch.no_grad():
        w8 = w8_ref.wan_block_w8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
        f8 = fp8_ref.wan_block_fp8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
        w8_32 = w8_ref.wan_block_w8(g["x"].float(), g["ctx"].float(), g["temb6"].float(), f32(g["sd"]), "", H, cos, sin,
                                    attn_fn=lambda q, k, v: wan_ref.attention_fp32(q, k, v)[0])
    e_bf16, e_w8, e_f8, e_w8_32 = (rel_l2(t, ref) for t in (g["y_ref_bf16"], w8, f8, w8_32))
    print(f"block relL2 from fp32: bf16 {e_bf16:.2e}, int8 weights {e_w8:.2e} (fp32 activations {e_w8_32:.2e}), fp8 {e_f8:.2e}")
    assert e_bf16 < e_w8 < 1e-2 and e_w8_32 < 1e-2
    assert e_f8 > 3 * e_w8


# ------------------------------------------------------------------------------------------------ plug-in
@pytest.mark.skipif(not ref_shim.available(), reason="reference tree not present (set FVB_REFERENCE_ROOT or stage oracle/_ref/reference_py)")
def test_plugin_int8w_config_resolves_on_sm90(monkeypatch):
    ref_shim.install()
    from fastvideo_b200 import plugin as p
    ns = p.install(force=True)
    try:
        monkeypatch.setattr(torch.cuda, "get_device_capability", lambda *a, **k: (9, 0))
        from fastvideo.layers.linear import LinearMethodBase, ReplicatedLinear
        from fastvideo.layers.quantization import get_quantization_config
        from fastvideo_b200._lib import FvbError
        cfg_cls = get_quantization_config(p.QUANT_NAME_INT8W)
        assert cfg_cls.__name__ == "Fvb200Int8WeightConfig" and cfg_cls.get_min_capability() == 90
        assert cfg_cls().get_name() == "fvb200_int8w"
        lin = ReplicatedLinear(256, 384, bias=True, params_dtype=torch.bfloat16, quant_config=cfg_cls(), prefix="blocks.0.to_q")
        assert type(lin.quant_method).__name__ == "Fvb200Int8WeightLinearMethod"
        assert isinstance(lin.quant_method, LinearMethodBase)
        assert tuple(lin.weight.shape) == (384, 256) and lin.weight.dtype == torch.bfloat16
        src = torch.nn.Linear(256, 384).to(torch.bfloat16)
        lin.load_state_dict(src.state_dict())
        assert torch.equal(lin.weight, src.weight)
        with pytest.raises(FvbError):
            lin.quant_method.process_weights_after_loading(lin)  # CPU weights: quantised on the GPU only
        with pytest.raises(FvbError):
            lin(torch.zeros(2, 5, 256, dtype=torch.bfloat16))
    finally:
        p.uninstall()
