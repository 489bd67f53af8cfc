"""CPU: the arithmetic of the FP8 residual-block convolutions of the Wan VAE decoder (tests/vae_fp8_ref.py) -- the static
activation bound, the routing of the oracle decoder, the FP8 decoder's distance from the fp32 one -- and the guards of the
WanVAEConfig.fp8_convs flag."""
import os

import pytest
import torch

import vae_fp8_ref as ref
from oracle import vae_ref
from util import rel_l2


@pytest.mark.parametrize("C", [96, 192, 384])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_bound_is_attained_by_a_one_hot_pixel(C, sign):
    """A pixel whose whole energy sits in the channel of the largest |gamma| normalises to exactly sqrt(C) * gamma_k: the
    bound itself, quantised to +-448 (and not beyond)."""
    g = torch.Generator().manual_seed(C)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).bfloat16().float()
    k = int(gamma.abs().argmax())
    gamma[k] = sign * gamma[k].abs()
    bound = ref.norm_bound(gamma)
    y = torch.zeros(3, C)
    y[:, k] = torch.tensor([1e-3, 1.0, 37.0])
    q = ref.norm_e4m3(y, gamma, bound, silu=False)
    assert torch.equal(q[:, k].float(), torch.full((3,), sign * 448.0))
    assert float(q.float().abs().max()) == 448.0


@pytest.mark.parametrize("silu", [True, False])
def test_bound_holds_for_random_gamma_and_inputs(silu):
    g = torch.Generator().manual_seed(3)
    for C in (16, 96, 384):
        gamma = torch.randn(C, generator=g) * 2
        bound = ref.norm_bound(gamma)
        y = torch.randn(4096, C, generator=g) * torch.rand(4096, 1, generator=g) * 100
        y[:64] = 0
        y[64:128, : C // 2] = 0
        v = ref.rms_norm_silu(y, gamma, silu)
        assert float(v.abs().max()) <= bound * (1 + 2e-7)
        q = ref.quantize_static(v, bound)
        assert not torch.isnan(q.float()).any() and float(q.float().abs().max()) <= 448.0
        # the dequantised values sit within e4m3's half-step of v (relative 2^-4) or its subnormal step
        deq = q.float() * ref.x_scale(bound)
        assert bool(((deq - v).abs() <= v.abs() * 2 ** -4 + ref.x_scale(bound) * 2 ** -9 * 1.01).all())


def test_zero_bound_quantises_to_zero():
    q = ref.quantize_static(torch.randn(8, 16), 0.0)
    assert q.float().abs().max() == 0 and float(ref.x_scale(0.0)) == 1.0


def test_routing_hits_exactly_the_28_res_block_convs(golden_dir):
    """The default structure (4 stages x 3 residual blocks + 2 mid blocks): 14 blocks x (conv1, conv2), each called once
    by the one-pass oracle, and no other convolution."""
    g = torch.load(os.path.join(golden_dir, "wan_vae_decode.pt"))
    sd = {k: v.float() for k, v in g["sd"].items()}
    assert len(ref.res_conv_bounds(sd)) == 28
    with ref.route_res_convs(sd) as hits:
        vae_ref.decode(g["z"][:, :, :2].float(), sd, g["dim_mult"], g["num_res_blocks"], g["temperal_downsample"])
    assert len(hits) == 28 and len(set(hits)) == 28
    assert vae_ref.causal_conv3d.__name__ == "causal_conv3d"  # restored


def test_fp8_decoder_restatement_real_widths():
    """Real widths (384 / 192 / 96 channels), random weights: the FP8 decode is 5.3e-2 (relative L2) from the fp32 one;
    rounding the same 28 convolutions' operands to bf16 instead gives 2.4e-3."""
    sd, g = ref.real_width_state_dict()
    z = torch.randn(1, 16, 3, 4, 6, generator=g).bfloat16().float()
    with torch.no_grad():
        y32 = vae_ref.decode(z, sd)
        y8 = ref.decode_fp8(z, sd)
    e = rel_l2(y8, y32)
    assert y8.shape == y32.shape == (1, 3, 9, 32, 48)
    assert 1e-2 < e < 8e-2, e


def test_fp8_ops_have_no_cpu_fallback():
    from fastvideo_b200 import ops
    x = torch.zeros(1, 4, 4, 32, dtype=torch.float8_e4m3fn)
    w = torch.zeros(32, 27 * 32, dtype=torch.float8_e4m3fn)
    with pytest.raises(ops.FvbError):
        ops.conv3d_cl_fp8(x, w, torch.ones(32), 32, (3, 3, 3), 1.0)
    with pytest.raises(ops.FvbError):
        ops.rmsnorm_silu_cl_e4m3(torch.zeros(4, 32, dtype=torch.bfloat16), torch.ones(32), 1.0)


def test_encoder_refuses_fp8_convs():
    from fastvideo_b200 import ops, wan_vae
    with pytest.raises(ops.FvbError):
        wan_vae.WanVAEEncoder(wan_vae.WanVAEConfig(fp8_convs=True), {})
    assert wan_vae.WanVAEConfig().fp8_convs is False
