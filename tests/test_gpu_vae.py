"""GPU: Wan VAE decode. (1) golden output of the reference's AutoencoderKLWan.decode (feature-cache loop, fp32 CPU,
small decoder); (2) the real channel widths (base_dim 96: 384/192/96) against the oracle's single-pass causal
restatement; (3) the implicit-GEMM conv kernel alone against F.conv3d, including cache / t_off handling."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import vae_ref
from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu


def bf16_floor(y):
    return rel_l2(y.bfloat16(), y)


@pytest.mark.parametrize("Cin,Cout,kt,k,T,H,W,t_off", [(64, 64, 3, 3, 3, 9, 20, 0), (64, 128, 3, 3, 3, 16, 16, 2), (96, 96, 3, 3, 2, 10, 33, 1),
                                                      (16, 64, 3, 3, 1, 8, 8, 0), (192, 96, 1, 3, 2, 12, 17, 0), (96, 3, 3, 3, 2, 24, 40, 2),
                                                      (384, 384, 3, 3, 1, 8, 16, 2), (128, 256, 3, 1, 2, 6, 10, 1),
                                                      (96, 96, 3, 3, 1, 40, 50, 2), (192, 192, 3, 3, 1, 20, 30, 2)])
@pytest.mark.parametrize("seed", [0, 1])
def test_conv3d_cl_matches_torch(Cin, Cout, kt, k, T, H, W, t_off, seed):
    """Two seeded inputs per shape, each held to F.conv3d."""
    from fastvideo_b200 import ops
    torch.manual_seed(Cin + Cout + T + 1000 * seed)
    Tn = T
    x = torch.randn(t_off + Tn, H, W, Cin, device="cuda").bfloat16()
    w = (torch.randn(Cout, Cin, kt, k, k, device="cuda") / (Cin * kt * k * k) ** 0.5).bfloat16()
    b = torch.randn(Cout, device="cuda").bfloat16()
    resid = torch.randn(Tn, H, W, Cout, device="cuda").bfloat16() if Cout % 8 == 0 else None
    wp, cin_pad, kk = ops.pack_conv_weight(w)
    out = ops.conv3d_cl(x, wp, cin_pad, kk, b, resid, T_out=Tn, t_off=t_off)
    # reference: causal conv over [cache | new] with zeros before the buffer start
    xn = x.permute(3, 0, 1, 2)[None].float()  # [1, C, T, H, W]
    pad_t = (kt - 1) - t_off if kt > 1 else 0
    xp = F.pad(xn, (k // 2, k // 2, k // 2, k // 2, max(pad_t, 0), 0))
    y = F.conv3d(xp, w.float(), b.float())[0]  # [Cout, T', H, W]
    y = y[:, -Tn:].permute(1, 2, 3, 0)
    ref_round = y.bfloat16()
    if resid is not None:
        y = ref_round.float() + resid.float()
    assert out.shape == (Tn, H, W, Cout)
    assert_bf16_parity(out, y, name="conv3d")


@pytest.mark.parametrize("Cin,Cout,kt,T,H,W,t_off,resid,raw", [(96, 96, 3, 2, 10, 33, 1, True, True), (192, 192, 3, 1, 9, 20, 2, True, False),
                                                               (64, 32, 3, 2, 8, 16, 0, False, False), (384, 192, 1, 2, 12, 17, 0, False, True),
                                                               (128, 128, 3, 1, 16, 16, 2, True, True)])
@pytest.mark.parametrize("seed", [0, 1])
def test_conv3d_fused_consumer_norm_equals_separate_pass(Cin, Cout, kt, T, H, W, t_off, resid, raw, seed):
    """fvb_conv3d_cl_norm == fvb_rmsnorm_silu_cl(fvb_conv3d_cl(...)): the same bf16 row, the same fp32 norm expression; only
    the order of the sum of squares differs (thread-serial vs warp tree)."""
    from fastvideo_b200 import ops
    torch.manual_seed(Cin + Cout + 1000 * seed)
    x = torch.randn(t_off + T, H, W, Cin, device="cuda").bfloat16()
    w = (torch.randn(Cout, Cin, kt, 3, 3, device="cuda") / (Cin * kt * 9) ** 0.5).bfloat16()
    b = torch.randn(Cout, device="cuda").bfloat16()
    r = torch.randn(T, H, W, Cout, device="cuda").bfloat16() if resid else None
    gamma = (1 + 0.2 * torch.randn(Cout, device="cuda")).float()
    wp, cin_pad, kk = ops.pack_conv_weight(w)
    y = ops.conv3d_cl(x, wp, cin_pad, kk, b, r, T_out=T, t_off=t_off)
    for silu in (True, False):
        want = ops.rmsnorm_silu_cl(y, gamma, silu=silu)
        got_raw, got = ops.conv3d_cl_norm(x, wp, cin_pad, kk, gamma, b, r, want_raw=raw, silu=silu, T_out=T, t_off=t_off)
        assert (got_raw is None) == (not raw)
        if raw:
            assert torch.equal(got_raw, y)
        # (one multiplier per pixel instead of a division per element: an occasional last-bit difference in bf16)
        assert (got != want).float().mean() < 2e-2 and rel_l2(got, want) < 1e-3
    with pytest.raises(ops.FvbError):  # more than one N tile: the caller has to take the separate pass
        w2 = (torch.randn(384, Cin, kt, 3, 3, device="cuda") / (Cin * kt * 9) ** 0.5).bfloat16()
        wp2, cp2, kk2 = ops.pack_conv_weight(w2)
        ops.conv3d_cl_norm(x, wp2, cp2, kk2, torch.ones(384, device="cuda"), T_out=T, t_off=t_off)


def test_vae_decode_fused_and_separate_norm_agree(golden_dir, monkeypatch):
    from fastvideo_b200 import wan_vae
    g = torch.load(os.path.join(golden_dir, "wan_vae_decode.pt"))
    dec = _decoder(g["sd"], g["base_dim"], g["dim_mult"], g["num_res_blocks"], g["temperal_downsample"])
    monkeypatch.setattr(wan_vae, "FUSE_NORM", True)
    y1 = dec.decode(g["z"].cuda())
    monkeypatch.setattr(wan_vae, "FUSE_NORM", False)
    y0 = dec.decode(g["z"].cuda())
    # The two flows differ only in the order of a sum of squares, but one flipped last bit re-randomises every later bf16
    # rounding of the ~50-layer decoder: they end up as two independent bf16 evaluations (measured 1.2e-2 apart = the
    # reference-bf16 floor). Both are held to the stated rule against the fp32 evaluation.
    assert_bf16_parity(y1, g["y_fp32"], ref_bf16=g["y_ref_bf16"], name="VAE decode, fused consumer norm")
    assert_bf16_parity(y0, g["y_fp32"], ref_bf16=g["y_ref_bf16"], name="VAE decode, separate norm pass")
    assert rel_l2(y1, y0) < 2.5 * rel_l2(g["y_ref_bf16"], g["y_fp32"])


def test_conv_time_interleave():
    from fastvideo_b200 import ops
    torch.manual_seed(0)
    C, T, H, W = 64, 2, 6, 9
    x = torch.randn(T, H, W, C, device="cuda").bfloat16()
    w = (torch.randn(2 * C, C, 3, 1, 1, device="cuda") / (3 * C) ** 0.5).bfloat16()
    b = torch.randn(2 * C, device="cuda").bfloat16()
    wp, cp, kk = ops.pack_conv_weight(w)
    out = ops.conv3d_cl(x, wp, cp, kk, b, T_out=T, t_off=0, interleave_c=C)
    y = F.conv3d(F.pad(x.permute(3, 0, 1, 2)[None].float(), (0, 0, 0, 0, 2, 0)), w.float(), b.float())  # [1, 2C, T, H, W]
    y = y.reshape(1, 2, C, T, H, W)
    y = torch.stack((y[:, 0], y[:, 1]), 3).reshape(1, C, 2 * T, H, W)[0].permute(1, 2, 3, 0)
    assert_bf16_parity(out, y, name="interleave")


def _decoder(sd, base_dim, dim_mult, nrb, tds):
    from fastvideo_b200 import wan_vae
    cfg = wan_vae.WanVAEConfig(base_dim=base_dim, dim_mult=tuple(dim_mult), num_res_blocks=nrb, temperal_downsample=tuple(tds))
    return wan_vae.WanVAEDecoder(cfg, {k: v.cuda() for k, v in sd.items()})


def test_vae_decode_against_reference_golden(golden_dir):
    g = torch.load(os.path.join(golden_dir, "wan_vae_decode.pt"))
    dec = _decoder(g["sd"], g["base_dim"], g["dim_mult"], g["num_res_blocks"], g["temperal_downsample"])
    y = dec.decode(g["z"].cuda())
    assert y.shape == g["y_fp32"].shape and y.dtype == torch.float32
    assert float(y.abs().max()) <= 1.0
    # the reference itself runs this decoder under bf16 autocast (configs/pipelines/wan.py:59): dozens of chained bf16
    # roundings. Stated tolerance (tests/util.py): no further from the fp32 evaluation than the reference's own bf16-autocast
    # decode of the same z (golden `y_ref_bf16`, relL2 1.2e-2 on this fixture) + 1e-3.
    assert_bf16_parity(y, g["y_fp32"], ref_bf16=g["y_ref_bf16"], name="VAE decode (feature cache)")
    # decoding twice gives bitwise the same result (cache reset works)
    assert torch.equal(y, dec.decode(g["z"].cuda()))


def test_vae_decode_real_widths_against_oracle():
    """base_dim 96 -> 384/192/96-channel stages (the 32-channel k-block / SWIZZLE_64B path), tiny frames."""
    torch.manual_seed(1)
    g = torch.Generator().manual_seed(1)
    base, mult, nrb, tds = 96, (1, 2, 4, 4), 2, (False, True, True)
    dims = [base * u for u in [mult[-1]] + list(mult[::-1])]
    sd = {}

    def conv(name, co, ci, k):
        fan = ci * k[0] * k[1] * k[2]
        sd[name + ".weight"] = (torch.randn(co, ci, *k, generator=g) * (1.5 / fan ** 0.5)).bfloat16().float()
        sd[name + ".bias"] = (0.1 * torch.randn(co, generator=g)).bfloat16().float()

    def res(p, ci, co):
        sd[p + "norm1.gamma"] = (1 + 0.2 * torch.randn(ci, 1, 1, 1, generator=g)).bfloat16().float()
        sd[p + "norm2.gamma"] = (1 + 0.2 * torch.randn(co, 1, 1, 1, generator=g)).bfloat16().float()
        conv(p + "conv1", co, ci, (3, 3, 3)); conv(p + "conv2", co, co, (3, 3, 3))
        if ci != co: conv(p + "conv_shortcut", co, ci, (1, 1, 1))

    conv("post_quant_conv", 16, 16, (1, 1, 1)); conv("decoder.conv_in", dims[0], 16, (3, 3, 3))
    res("decoder.mid_block.resnets.0.", dims[0], dims[0]); res("decoder.mid_block.resnets.1.", dims[0], dims[0])
    sd["decoder.mid_block.attentions.0.norm.gamma"] = (1 + 0.2 * torch.randn(dims[0], 1, 1, generator=g)).bfloat16().float()
    for n, co in (("to_qkv", 3 * dims[0]), ("proj", dims[0])):
        sd[f"decoder.mid_block.attentions.0.{n}.weight"] = (torch.randn(co, dims[0], 1, 1, generator=g) / dims[0] ** 0.5).bfloat16().float()
        sd[f"decoder.mid_block.attentions.0.{n}.bias"] = (0.1 * torch.randn(co, generator=g)).bfloat16().float()
    t_up = list(tds)[::-1]
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        if i > 0: ci = ci // 2
        cur = ci
        for j in range(nrb + 1):
            res(f"decoder.up_blocks.{i}.resnets.{j}.", cur, co); cur = co
        if i != len(mult) - 1:
            p = f"decoder.up_blocks.{i}.upsamplers.0."
            sd[p + "resample.1.weight"] = (torch.randn(co // 2, co, 3, 3, generator=g) * (1.5 / (9 * co) ** 0.5)).bfloat16().float()
            sd[p + "resample.1.bias"] = (0.1 * torch.randn(co // 2, generator=g)).bfloat16().float()
            if t_up[i]: conv(p + "time_conv", 2 * co, co, (3, 1, 1))
    sd["decoder.norm_out.gamma"] = (1 + 0.2 * torch.randn(dims[-1], 1, 1, 1, generator=g)).bfloat16().float()
    conv("decoder.conv_out", 3, dims[-1], (3, 3, 3))
    z = torch.randn(1, 16, 3, 4, 6, generator=g).bfloat16().float()
    with torch.no_grad():
        ref = vae_ref.decode(z, sd, mult, nrb, tds)
    y = _decoder({k: v.bfloat16() for k, v in sd.items()}, base, mult, nrb, tds).decode(z.cuda())
    assert y.shape == ref.shape == (1, 3, 9, 32, 48)
    e = rel_l2(y, ref)
    assert e < 2e-2, e


def test_vae_cacheless_decode_and_wan_tiled_wrappers_against_reference_golden(golden_dir):
    """AutoencoderKLWan._decode (feature cache off) and AutoencoderKLWan.decode over ParallelTiledVAE's temporal / spatial
    tiling with Wan's wrappers (wanvae.py:1218-1247; models/vaes/common.py:77-92, 266-374), same weights as the cached
    fixture, goldens from the reference on CPU (fp32 + its own bf16-autocast run as the floor)."""
    from fastvideo_b200 import vae_tiling
    g = torch.load(os.path.join(golden_dir, "wan_vae_decode.pt"))
    c = torch.load(os.path.join(golden_dir, "wan_vae_cacheless.pt"))
    dec = _decoder(g["sd"], g["base_dim"], g["dim_mult"], g["num_res_blocks"], g["temperal_downsample"])
    for case in c["cases"]:
        z = case["z"].cuda()
        if case["cfg"] is None:
            y = dec.decode_tile(z)
        else:
            cfg = vae_tiling.TilingConfig(use_parallel_tiling=False, **case["cfg"])
            y = dec.decode_tiled(z, cfg)
        assert tuple(y.shape) == tuple(case["y_fp32"].shape), (case["name"], y.shape, case["y_fp32"].shape)
        assert_bf16_parity(y, case["y_fp32"], ref_bf16=case["y_ref_bf16"], name="VAE " + case["name"])
    # the cached decoder still works after cache-less calls (mode flag restored)
    y = dec.decode(g["z"].cuda())
    assert_bf16_parity(y, g["y_fp32"], ref_bf16=g["y_ref_bf16"], name="VAE decode after cache-less calls")


def test_vae_encoder_against_reference_golden(golden_dir):
    """AutoencoderKLWan.encode (feature-cache loop: first frame, then 4-frame chunks; wanvae.py:1128-1151) -- golden from the
    reference on CPU in fp32, floor from its own bf16-autocast run."""
    from fastvideo_b200 import wan_vae
    g = torch.load(os.path.join(golden_dir, "wan_vae_encode.pt"))
    cfg = wan_vae.WanVAEConfig(base_dim=g["base_dim"], dim_mult=tuple(g["dim_mult"]), num_res_blocks=g["num_res_blocks"],
                               temperal_downsample=tuple(g["temperal_downsample"]))
    enc = wan_vae.WanVAEEncoder(cfg, {k: v.cuda() for k, v in g["sd"].items()})
    mean, logvar = enc.encode(g["x"].cuda())
    y = torch.cat([mean, logvar], 1)
    assert y.shape == g["y_fp32"].shape and y.dtype == torch.float32
    assert_bf16_parity(y, g["y_fp32"], ref_bf16=g["y_ref_bf16"], name="VAE encode")
    m2, l2 = enc.encode(g["x"].cuda())
    assert torch.equal(mean, m2) and torch.equal(logvar, l2)
