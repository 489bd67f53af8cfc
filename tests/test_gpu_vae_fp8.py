"""GPU: the FP8 (e4m3) residual-block convolutions of the Wan VAE decoder against their CPU restatement (tests/vae_fp8_ref.py):
the FP8 implicit-GEMM conv (fvb_conv3d_cl_fp8), the e4m3 norm outputs (fused epilogue and separate row pass), the argument
checks, and the whole decoder with WanVAEConfig(fp8_convs=True)."""
import os

import pytest
import torch

import vae_fp8_ref as ref
from oracle import vae_ref
from util import rel_l2

pytestmark = pytest.mark.gpu


def e4m3_steps(a, b):
    """Per-element distance between two e4m3 tensors in representable steps (signed ordinal of the code)."""
    def ordinal(t):
        c = t.view(torch.uint8).int().cpu()
        return torch.where(c >= 128, -(c - 128), c)
    return (ordinal(a) - ordinal(b)).abs()


def _conv_case(Cin, Cout, kt, k, T, H, W, t_off, seed, resid=True):
    """Seeded e4m3 input (a normalised activation quantised against its bound), weights, bias, residual; returns the GPU
    operands and the fp64 restatement (before the bf16 rounding)."""
    torch.manual_seed(Cin + Cout + T + 1000 * seed)
    x = torch.randn(t_off + T, H, W, Cin)
    bound = float(x.abs().max()) * 1.05
    xq = ref.quantize_static(x, bound)
    w = (torch.randn(Cout, Cin, kt, k, k) / (Cin * kt * k * k) ** 0.5).bfloat16()
    b = torch.randn(Cout).bfloat16()
    r = torch.randn(T, H, W, Cout).bfloat16() if resid and Cout % 8 == 0 else None
    wq_ref, ws_ref = ref.quantize_conv_weight(w.float())
    pad_t = max((kt - 1) - t_off, 0) if kt > 1 else 0
    y64 = ref.fp8_conv3d_exact(xq.permute(3, 0, 1, 2)[None], ref.x_scale(bound), wq_ref, ws_ref, b.float(), t_pad=pad_t)
    y64 = y64[0, :, -T:].permute(1, 2, 3, 0)
    return dict(x=xq.cuda(), w=w.cuda(), b=b.cuda(), r=r.cuda() if r is not None else None, x_scale=float(ref.x_scale(bound)),
                y64=y64, wq_ref=wq_ref, ws_ref=ws_ref)


def _want(c):
    """bf16(y) (+ resid, rounded again): the kernel's epilogue applied to the exact value."""
    y = c["y64"].float().bfloat16()
    if c["r"] is not None:
        y = (y.float() + c["r"].cpu().float()).bfloat16()
    return y


# The MMAs accumulate straight into the fp32 accumulators, and the tensor core sums e4m3 products with fewer bits than fp32.
# Measured on an H100 80GB against exact accumulation: relative L2 7e-4 (K = 3 x 128) to 2.25e-3 (K = 27 x 384), growing with
# K; the e4m3 rounding of the operands themselves costs 3.7e-2 per convolution (CPU, Gaussian inputs).
CONV_TOL = 3e-3


@pytest.mark.parametrize("Cin,Cout,kt,k,T,H,W,t_off", [(64, 64, 3, 3, 3, 9, 20, 0), (64, 128, 3, 3, 3, 16, 16, 2), (96, 96, 3, 3, 2, 10, 33, 1),
                                                      (192, 96, 1, 3, 2, 12, 17, 0), (96, 3, 3, 3, 2, 24, 40, 2), (96, 40, 3, 3, 1, 9, 18, 1),
                                                      (384, 384, 3, 3, 1, 8, 16, 2), (128, 256, 3, 1, 2, 6, 10, 1), (384, 200, 3, 3, 1, 8, 16, 1),
                                                      (96, 96, 3, 3, 1, 40, 50, 2), (192, 192, 3, 3, 1, 20, 30, 2), (192, 384, 3, 3, 1, 10, 20, 2)])
@pytest.mark.parametrize("seed", [0, 1])
def test_conv3d_fp8_matches_restatement(Cin, Cout, kt, k, T, H, W, t_off, seed):
    """fvb_conv3d_cl_fp8 against the fp64 conv of the dequantised operands: cache / t_off, residual, Couts that are not a
    multiple of the N tile, every k-block width (32 / 64 / 128 bytes)."""
    from fastvideo_b200 import ops
    c = _conv_case(Cin, Cout, kt, k, T, H, W, t_off, seed)
    wq, ws, cin_pad, kk = ops.pack_conv_weight_fp8(c["w"])
    # the weight quantiser is the row quantiser: bit-equal to its restatement
    ntaps = kk[0] * kk[1] * kk[2]
    assert torch.equal(wq.view(Cout, ntaps, cin_pad)[:, :, :Cin].cpu().view(torch.uint8),
                       c["wq_ref"].permute(0, 2, 3, 4, 1).reshape(Cout, ntaps, Cin).view(torch.uint8))
    assert torch.equal(ws.cpu(), c["ws_ref"])
    out = ops.conv3d_cl_fp8(c["x"], wq, ws, cin_pad, kk, c["x_scale"], c["b"], c["r"], T_out=T, t_off=t_off)
    assert out.shape == (T, H, W, Cout) and out.dtype == torch.bfloat16
    want = _want(c)
    e = rel_l2(out, want)
    print(f"conv fp8 {Cin}->{Cout} k{kt}x{k} seed {seed}: relL2 {e:.2e}")
    assert e < CONV_TOL, e


@pytest.mark.parametrize("Cin,Cout,kt,T,H,W,t_off,resid,raw", [(96, 96, 3, 2, 10, 33, 1, True, True), (192, 192, 3, 1, 9, 20, 2, True, False),
                                                               (64, 32, 3, 2, 8, 16, 0, False, False), (384, 192, 1, 2, 12, 17, 0, False, True),
                                                               (128, 128, 3, 1, 16, 16, 2, True, True)])
@pytest.mark.parametrize("seed", [0, 1])
def test_fused_e4m3_norm_output_equals_row_pass(Cin, Cout, kt, T, H, W, t_off, resid, raw, seed):
    """The e4m3 normalised output of the fused epilogue (FP8 and bf16 convolutions) against the separate e4m3 row pass on
    the same raw output: at most one e4m3 step apart (the epilogue's one multiplier per pixel vs a division per element),
    rarely; the bf16 normalised output of the FP8 conv against the bf16 row pass; the row pass against its restatement."""
    from fastvideo_b200 import ops
    c = _conv_case(Cin, Cout, kt, 3, T, H, W, t_off, seed, resid)
    gamma = (1 + 0.2 * torch.randn(Cout)).float().cuda()
    bound = ref.norm_bound(gamma.cpu())
    wq, ws, cin_pad, kk = ops.pack_conv_weight_fp8(c["w"])
    y = ops.conv3d_cl_fp8(c["x"], wq, ws, cin_pad, kk, c["x_scale"], c["b"], c["r"], T_out=T, t_off=t_off)
    wp, cp, kk2 = ops.pack_conv_weight(c["w"])
    xb = (c["x"].float() * c["x_scale"]).bfloat16()  # a bf16 input for the bf16 conv
    yb = ops.conv3d_cl(xb, wp, cp, kk2, c["b"], c["r"], T_out=T, t_off=t_off)
    for silu in (True, False):
        want = ops.rmsnorm_silu_cl_e4m3(y, gamma, bound, silu=silu)
        # row pass vs restatement
        st = e4m3_steps(want, ref.norm_e4m3(y.cpu(), gamma.cpu(), bound, silu))
        assert int(st.max()) <= 1 and float((st > 0).float().mean()) < 1e-3
        got_raw, got = ops.conv3d_cl_fp8_norm(c["x"], wq, ws, cin_pad, kk, c["x_scale"], gamma, c["b"], c["r"], want_raw=raw,
                                              silu=silu, T_out=T, t_off=t_off, norm_bound=bound)
        assert got.dtype == torch.float8_e4m3fn and (got_raw is None) == (not raw)
        if raw:
            assert torch.equal(got_raw, y)
        st = e4m3_steps(got, want)
        rate = float((st > 0).float().mean())
        print(f"fused e4m3 norm {Cin}->{Cout} silu={silu}: one-step flips {rate:.2e}")
        assert int(st.max()) <= 1 and rate < 1e-2, rate
        _, gotb = ops.conv3d_cl_fp8_norm(c["x"], wq, ws, cin_pad, kk, c["x_scale"], gamma, c["b"], c["r"], want_raw=False,
                                         silu=silu, T_out=T, t_off=t_off)
        assert gotb.dtype == torch.bfloat16
        wantb = ops.rmsnorm_silu_cl(y, gamma, silu=silu)
        assert (gotb != wantb).float().mean() < 2e-2 and rel_l2(gotb, wantb) < 1e-3
        # bf16 operands, e4m3 normalised output (the upsampler convolution feeding a residual block)
        _, got8 = ops.conv3d_cl_norm_e4m3(xb, wp, cp, kk2, gamma, bound, c["b"], c["r"], want_raw=False, silu=silu, T_out=T,
                                          t_off=t_off)
        st = e4m3_steps(got8, ops.rmsnorm_silu_cl_e4m3(yb, gamma, bound, silu=silu))
        assert int(st.max()) <= 1 and float((st > 0).float().mean()) < 1e-2


def test_fp8_conv_bad_arguments_raise():
    from fastvideo_b200 import ops
    torch.manual_seed(0)
    w = (torch.randn(64, 24, 3, 3, 3) / 25).bfloat16().cuda()
    wq, ws, cp, kk = ops.pack_conv_weight_fp8(w)
    x = torch.zeros(1, 8, 16, 24, dtype=torch.float8_e4m3fn, device="cuda")
    with pytest.raises(ops.FvbError):  # Cin % 16 != 0
        ops.conv3d_cl_fp8(x, wq, ws, cp, kk, 1.0)
    w = (torch.randn(64, 32, 3, 3, 3) / 25).bfloat16().cuda()
    wq, ws, cp, kk = ops.pack_conv_weight_fp8(w)
    x = torch.zeros(1, 8, 16, 32, dtype=torch.float8_e4m3fn, device="cuda")
    with pytest.raises(ops.FvbError):  # missing weight scales
        ops.conv3d_cl_fp8(x, wq, None, cp, kk, 1.0)
    with pytest.raises(ops.FvbError):  # bf16 input
        ops.conv3d_cl_fp8(x.float().bfloat16(), wq, ws, cp, kk, 1.0)
    w = (torch.randn(384, 32, 3, 3, 3) / 25).bfloat16().cuda()
    wq, ws, cp, kk = ops.pack_conv_weight_fp8(w)
    with pytest.raises(ops.FvbError):  # fused norm needs one N tile
        ops.conv3d_cl_fp8_norm(x, wq, ws, cp, kk, 1.0, torch.ones(384, device="cuda"), norm_bound=1.0)
    ops.conv3d_cl_fp8(x, wq, ws, cp, kk, 1.0)  # the same convolution without the norm is fine
    torch.cuda.synchronize()


def _decoder(sd, base_dim, dim_mult, nrb, tds, fp8):
    from fastvideo_b200 import wan_vae
    cfg = wan_vae.WanVAEConfig(base_dim=base_dim, dim_mult=tuple(dim_mult), num_res_blocks=nrb, temperal_downsample=tuple(tds),
                               fp8_convs=fp8)
    return wan_vae.WanVAEDecoder(cfg, {k: v.cuda() for k, v in sd.items()})


# The decoder and its restatement are two independent FP8 evaluations: bf16 rounding elsewhere in the decoder moves some
# inputs of the e4m3 roundings across a rounding boundary, and each such element then lands a whole e4m3 step (6 %) away.
# So the decode is held to the restatement's own statistics: no further from the restatement than the restatement is from
# fp32, and no more than 15 % further from fp32 than the restatement. Measured on an H100 80GB (relative L2): golden fixture
# 7.3e-2 from the restatement, 7.9e-2 from fp32 (restatement 7.9e-2, bf16 decode 9.4e-3); real widths 4.4e-2 and 5.5e-2
# (restatement 5.3e-2).
def _check_decode(y, want, y32, name):
    e_ref, e32, e_rs = rel_l2(y, want), rel_l2(y, y32), rel_l2(want, y32)
    print(f"{name}: relL2 {e_ref:.2e} from the restatement, {e32:.2e} from fp32 (restatement {e_rs:.2e})")
    assert e_ref < e_rs and e32 < 1.15 * e_rs, (e_ref, e32, e_rs)
    return e_rs


def test_fp8_decode_golden(golden_dir):
    from fastvideo_b200 import vae_tiling
    g = torch.load(os.path.join(golden_dir, "wan_vae_decode.pt"))
    args = (g["base_dim"], g["dim_mult"], g["num_res_blocks"], g["temperal_downsample"])
    sd32 = {k: v.float() for k, v in g["sd"].items()}
    dec_b = _decoder(g["sd"], *args, fp8=False)
    yb = dec_b.decode(g["z"].cuda())
    dec = _decoder(g["sd"], *args, fp8=True)
    y = dec.decode(g["z"].cuda())
    with torch.no_grad():
        want = ref.decode_fp8(g["z"].float(), sd32, g["dim_mult"], g["num_res_blocks"], g["temperal_downsample"])
    assert y.shape == g["y_fp32"].shape and float(y.abs().max()) <= 1.0
    e_rs = _check_decode(y, want, g["y_fp32"], "golden fp8 decode")
    print(f"golden bf16 decode: relL2 {rel_l2(yb, g['y_fp32']):.2e} from fp32")
    assert torch.equal(y, dec.decode(g["z"].cuda()))  # decoding twice: bit-equal
    # the bf16 decoder of the same state dict is untouched
    assert torch.equal(yb, _decoder(g["sd"], *args, fp8=False).decode(g["z"].cuda()))
    # cache-less tile and one temporal-tiled case against the reference's fp32 goldens
    c = torch.load(os.path.join(golden_dir, "wan_vae_cacheless.pt"))
    done = set()
    for case in c["cases"]:
        kind = "tile" if case["cfg"] is None else ("temporal" if case["name"].startswith("temporal") else None)
        if kind is None or kind in done:
            continue
        z = case["z"].cuda()
        if kind == "tile":
            yt = dec.decode_tile(z)
        else:
            yt = dec.decode_tiled(z, vae_tiling.TilingConfig(use_parallel_tiling=False, **case["cfg"]))
        assert tuple(yt.shape) == tuple(case["y_fp32"].shape)
        e = rel_l2(yt, case["y_fp32"])
        print(f"golden fp8 {case['name']}: relL2 {e:.2e} from fp32")
        assert e < 1.25 * e_rs, (case["name"], e)  # no cache-less restatement: the cached decode's FP8 error + 25 %
        done.add(kind)
    assert done == {"tile", "temporal"}
    assert torch.equal(y, dec.decode(g["z"].cuda()))  # the cached decoder still works after cache-less calls


def test_fp8_decode_real_widths():
    sd, g = ref.real_width_state_dict()
    z = torch.randn(1, 16, 3, 4, 6, generator=g).bfloat16().float()
    args = (96, (1, 2, 4, 4), 2, (False, True, True))
    with torch.no_grad():
        y32 = vae_ref.decode(z, sd)
        want = ref.decode_fp8(z, sd)
    dec = _decoder({k: v.bfloat16() for k, v in sd.items()}, *args, fp8=True)
    y = dec.decode(z.cuda())
    assert y.shape == (1, 3, 9, 32, 48)
    _check_decode(y, want, y32, "real-width fp8 decode")
    assert torch.equal(y, dec.decode(z.cuda()))
    yt = dec.decode_tile(z.cuda())
    assert yt.shape == (1, 3, 12, 32, 48) and torch.isfinite(yt).all()
