"""CPU: the FP8 configuration's guards -- no CPU fallback, and the paths that read bf16 weights directly refuse an FP8
model with FvbError instead of failing on a missing attribute."""
import types

import pytest
import torch


def test_fp8_ops_have_no_cpu_fallback():
    from fastvideo_b200 import ops
    x = torch.zeros(8, 64, dtype=torch.bfloat16)
    with pytest.raises(ops.FvbError):
        ops.quantize_fp8_rows(x)
    with pytest.raises(ops.FvbError):
        ops.linear_fp8(x, x)


def test_fp8_weight_validates_its_layout():
    from fastvideo_b200 import ops
    q = torch.zeros(4, 32, dtype=torch.float8_e4m3fn)
    w = ops.Fp8Weight(q, torch.ones(4))
    assert tuple(w.shape) == (4, 32)
    with pytest.raises(ops.FvbError):
        ops.Fp8Weight(q.view(torch.uint8), torch.ones(4))
    with pytest.raises(ops.FvbError):
        ops.Fp8Weight(torch.zeros(4, 40, dtype=torch.float8_e4m3fn), torch.ones(4))  # 40-byte rows: not 16-byte aligned
    with pytest.raises(ops.FvbError):
        ops.Fp8Weight(q, torch.ones(5))


def test_sequence_parallel_and_causal_refuse_fp8_config():
    from fastvideo_b200 import causal_wan, distributed, ops, wan_dit
    cfg = wan_dit.WanDiTConfig(hidden_size=256, num_attention_heads=2, ffn_dim=512, num_layers=1, fp8_linears=True)
    model = types.SimpleNamespace(cfg=cfg)
    with pytest.raises(ops.FvbError):
        distributed.SPWanDiT(model, 0, 1)
    with pytest.raises(ops.FvbError):
        causal_wan.CausalWanDiT(cfg, {}, causal_wan.CausalConfig())
    with pytest.raises(ops.FvbError):
        causal_wan.CausalWanDiT.random(cfg, causal_wan.CausalConfig(), device="cpu")
    with pytest.raises(ops.FvbError):
        causal_wan.SPCausalWanDiT(model, 0, 1)
    assert wan_dit.WanDiTConfig().fp8_linears is False
