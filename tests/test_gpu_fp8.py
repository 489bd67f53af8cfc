"""GPU: FP8 (e4m3) linear layers -- the row quantiser, fvb_linear_fp8 with every epilogue, and the Wan block / model / denoiser
with WanDiTConfig.fp8_linears -- against the FP8 restatement (tests/fp8_ref.py: quantize_fp8_rows, fp8_linear_f32, wan_block_fp8,
wan_model_fp8)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fp8_ref
from oracle import vsa_index, wan_ref
from util import assert_bf16_parity, assert_two_bf16_paths_close, rel_l2

pytestmark = pytest.mark.gpu


def cuda_sd(sd):
    return {k: v.cuda() for k, v in sd.items()}


# ------------------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("K", [208, 5120, 13824, 20480])
def test_quantize_rows_bit_exact(K):
    """q and scale bit-equal to the oracle on strided rows, with zero rows and single-outlier rows mixed in (20480 also
    runs the part of the kernel that re-reads rows longer than its register cache)."""
    from fastvideo_b200 import ops
    torch.manual_seed(K)
    M, ld = 67, K + 24
    buf = torch.randn(M, ld, device="cuda").bfloat16() * 3
    buf[5] = 0
    buf[9, 7] = 4.0e4     # outliers: the rest of the row falls into e4m3's subnormal / zero range
    buf[11, K - 1] = -1.5e3
    buf[13, :K] = torch.randn(K, device="cuda").bfloat16() * 1e-6
    x = buf[:, 8:8 + K]  # row stride ld, start 16 bytes into the row
    q, s = ops.quantize_fp8_rows(x)
    q_ref, s_ref = fp8_ref.quantize_fp8_rows(x.cpu())
    assert q.shape == (M, K) and q.dtype == torch.float8_e4m3fn
    assert torch.equal(q.cpu().view(torch.uint8), q_ref.view(torch.uint8))
    assert torch.equal(s.cpu().view(torch.int32), s_ref.view(torch.int32))
    assert s[5].item() == 1.0 and (q[5].view(torch.uint8) == 0).all()


# ------------------------------------------------------------------------------------------------ fvb_linear_fp8
def ref_linear_fp8(x, wq, ws, b, epi, resid, gate, gate_rows):
    """(fp64 value of the formula, the formula with its fp32 / bf16 rounding points) for fvb_linear_fp8. The e4m3 products
    and their sums are exact in fp64, so the fp64 GEMM (run on the GPU for speed) is the exact accumulator."""
    xq, xs = fp8_ref.quantize_fp8_rows(x.cpu())
    xq, xs = xq.cuda(), xs.cuda()
    acc = xq.double() @ wq.double().t()
    exact = acc * xs.double()[:, None] * ws.double()[None, :]
    y32 = (acc.float() * xs[:, None]) * ws[None, :]
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


CASES = [(256, 512, 512, 0, 0), (1, 1536, 256, 0, 0), (333, 384, 200, 0, 0), (300, 64, 512, 0, 0), (300, 200, 640, 0, 0),
         (1000, 1536, 1536, 1, 0), (1000, 1536, 1536, 2, 0), (777, 1536, 1536, 3, 0), (777, 1536, 1536, 7, 128),
         (777, 1536, 1536, 4, 0), (9450, 5120, 5120, 0, 0), (2048, 5120, 13824, 0, 0), (512, 13824, 5120, 1, 0)]


def _case(M, N, K, epi, gate_rows):
    from fastvideo_b200 import ops
    torch.manual_seed(M + N + K + epi)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    resid = torch.randn(M, N, device="cuda").bfloat16() if epi >= 2 else None
    gate = None
    if epi in (2, 3, 7):
        gate = torch.randn(N, device="cuda") if gate_rows == 0 else torch.randn((M + gate_rows - 1) // gate_rows, N, device="cuda")
    wf = ops.Fp8Weight.quantize(w)
    return x, wf, b, resid, gate


@pytest.mark.parametrize("M,N,K,epi,gate_rows", CASES)
def test_linear_fp8_matches_formula(M, N, K, epi, gate_rows):
    """Against the fp64 value of the formula in include/fvb200.h (bf16 parity), and against the formula's own rounding
    points. Inside a 128-element k-block the tensor core accumulates e4m3 products with fewer bits than fp32, so the fp32
    value before the bf16 rounding is off by about 1e-4 relative and a few per cent of the outputs land on the
    neighbouring bf16 value: measured on an H100, 3.1 % (M = 1) to 5.3 % of the bf16 outputs, the same at K = 13 824 as
    at K = 5120 -- the partial sums leave the tensor core every 128 elements, so the error does not grow with K. The
    bound is 8 %; a wrong scale or a missing k-block is O(1) and fails the parity check."""
    from fastvideo_b200 import ops
    x, wf, b, resid, gate = _case(M, N, K, epi, gate_rows)
    out = ops.linear_fp8(x, wf, b, epi, resid, gate, gate_rows=gate_rows)
    exact, rounded = ref_linear_fp8(x, wf.q, wf.scale, b, epi, resid, gate, gate_rows)
    if epi == 2:  # fp32 output
        assert out.dtype == torch.float32
        assert rel_l2(out, rounded) < 1e-3
    else:
        assert_bf16_parity(out, exact, rounded, name=f"linear_fp8 epi{epi}")
        mism = (out.float() != rounded.float()).float().mean().item()
        print(f"linear_fp8 {M}x{N}x{K} epi{epi}: {mism:.4f} of outputs off the formula's rounding")
        assert mism < 0.08


def test_linear_fp8_repeatable_and_matches_scaled_mm():
    from fastvideo_b200 import ops
    x, wf, b, _, _ = _case(1000, 1536, 1536, 0, 0)
    a = ops.linear_fp8(x, wf, b)
    for _ in range(3):
        assert torch.equal(ops.linear_fp8(x, wf, b), a)
    xq, xs = ops.quantize_fp8_rows(x)
    try:
        ref = torch._scaled_mm(xq, wf.q.t(), scale_a=xs[:, None].contiguous(), scale_b=wf.scale[None, :].contiguous(),
                               bias=b, out_dtype=torch.bfloat16)
    except (RuntimeError, AttributeError, TypeError) as e:
        pytest.skip(f"torch._scaled_mm with row-wise scales is not available in this torch build ({e})")
    assert_two_bf16_paths_close(a, ref, name="linear_fp8 vs torch._scaled_mm")


def test_linear_fp8_rejects_bad_arguments():
    from fastvideo_b200 import ops
    x, wf, b, _, _ = _case(64, 128, 256, 0, 0)
    with pytest.raises(ops.FvbError):
        ops.linear_fp8(x, x)  # not an Fp8Weight
    with pytest.raises(ops.FvbError):
        ops.linear_fp8(x[:, :128], wf)  # K mismatch


# ------------------------------------------------------------------------------------------------ Wan block / model
def _rope(seq, d):
    return wan_ref.rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)])


def test_block_dense_fp8_against_oracle(golden_dir):
    """FP8 WanBlock vs the oracle block with the FP8 linear restatement (CPU, bf16). Measured on an H100: relL2 1.5e-2
    (2.8e-2 from the bf16 reference's output). Activations that differ in their last bf16 bit can quantise to neighbouring
    e4m3 values (a 1/16 relative step), which is what this distance is made of; a wrong scale would be O(1)."""
    from fastvideo_b200 import ops, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_dense.pt"))
    D, H = g["x"].shape[-1], g["heads"]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1, fp8_linears=True)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    for n in wan_dit.FP8_LINEARS:
        assert isinstance(getattr(blk, n), ops.Fp8Weight)
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    cos, sin = _rope(g["seq"], D // H)
    with torch.no_grad():
        y_ref = fp8_ref.wan_block_fp8(g["x"], g["ctx"], g["temb6"], g["sd"], "", H, cos, sin)
    e = rel_l2(y, y_ref[0])
    print(f"fp8 block relL2 vs oracle {e:.3e}, vs bf16 reference {rel_l2(y, g['y_ref_bf16'][0]):.3e}")
    assert e <= 3e-2


def _fp8_model(golden_dir, fp8=True):
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], fp8_linears=fp8)
    return g, cfg, wan_dit.WanDiT(cfg, sd)


def test_model_dense_fp8_against_oracle(golden_dir):
    """2-layer FP8 WanDiT vs the oracle model with the FP8 linear restatement. Measured on an H100: relL2 1.2e-2
    (2.2e-2 from the bf16 reference's output)."""
    from fastvideo_b200 import ops, wan_dit
    g, cfg, model = _fp8_model(golden_dir)
    y = model.forward(g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    with torch.no_grad():
        y_ref = fp8_ref.wan_model_fp8(g["latents"], g["text"], g["timestep"], g["sd"], g["heads"])
    e = rel_l2(y, y_ref)
    print(f"fp8 model relL2 vs oracle {e:.3e}, vs bf16 reference {rel_l2(y, g['y_ref_bf16']):.3e}")
    assert e <= 2e-2
    # the six token-stream weights are e4m3 only: no bf16 tensor of theirs is left on the block
    for blk in model.blocks:
        for n in wan_dit.FP8_LINEARS:
            w = getattr(blk, n)
            assert isinstance(w, ops.Fp8Weight) and w.q.dtype == torch.float8_e4m3fn
        shapes = {tuple(getattr(blk, n).shape) for n in wan_dit.FP8_LINEARS}
        left = [k for k, v in vars(blk).items() if torch.is_tensor(v) and v.dtype == torch.bfloat16 and v.dim() == 2
                and tuple(v.shape) in shapes and k not in ("w_kv2", "w_kv_img")]
        assert not left, left


def test_block_vsa_fp8_against_oracle():
    """WanTransformerBlock_VSA with FP8 linears, on the row criteria of test_gpu_wan.test_block_vsa_against_oracle with the
    median bound raised from 1e-2 to 3e-2 for the e4m3 quantisation flips (see test_block_dense_fp8_against_oracle).
    Measured on an H100: median row relL2 1.5e-2, every row below 3e-2."""
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
        y_ref = fp8_ref.wan_block_fp8(x, ctx, temb6, sd, "", H, cos, sin, vsa_meta=meta)
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=F_, num_layers=1, vsa=True, fp8_linears=True)
    blk = wan_dit.WanBlock(cuda_sd(sd), "", cfg)
    lay = wan_dit.make_layout(seq, cfg, "cuda", vsa_sparsity=0.5)
    y = wan_dit.block_forward(x[0].cuda()[lay.perm], blk, ctx[0].cuda(), temb6.cuda(), lay, cfg)[lay.inv_perm]
    err_rows = (y.float().cpu() - y_ref[0].float()).norm(dim=-1) / y_ref[0].float().norm(dim=-1)
    print(f"fp8 VSA block: median row relL2 {err_rows.median().item():.3e}, rows < 3e-2: {(err_rows < 3e-2).float().mean().item():.3f}")
    assert err_rows.median().item() < 3e-2
    assert (err_rows < 6e-2).float().mean().item() > 0.9


def test_denoiser_graph_replay_bit_equal_fp8(golden_dir):
    from fastvideo_b200.api import WanDenoiser
    g, cfg, model = _fp8_model(golden_dir)
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


def test_sequence_parallel_and_causal_reject_fp8(golden_dir):
    from fastvideo_b200 import causal_wan, distributed, ops
    g, cfg, model = _fp8_model(golden_dir)
    with pytest.raises(ops.FvbError):
        distributed.SPWanDiT(model, 0, 1)
    with pytest.raises(ops.FvbError):
        causal_wan.CausalWanDiT(cfg, cuda_sd(g["sd"]), causal_wan.CausalConfig())
    with pytest.raises(ops.FvbError):
        causal_wan.SPCausalWanDiT(model, 0, 1)
