"""GPU: the Wan transformer block and the whole DiT forward against golden outputs produced by the reference's own
WanTransformerBlock / WanTransformer3DModel (torch-SDPA backend, bf16, CPU; oracle/gen_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import vsa_index, wan_ref
from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu


def cuda_sd(sd):
    return {k: v.cuda() for k, v in sd.items()}


def test_block_dense_against_reference_golden(golden_dir):
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_dense.pt"))
    D = g["x"].shape[-1]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    e, floor = assert_bf16_parity(y, g["y_fp32"][0], g["y_ref_bf16"][0], name="wan block")
    # direct distance to the reference's bf16 output: two bf16 paths sharing rounding points
    assert rel_l2(y, g["y_ref_bf16"][0]) < 2 * floor


def test_block_i2v_cross_attention_against_reference_golden(golden_dir):
    """WanTransformerBlock with WanI2VCrossAttention (257 CLIP image tokens + text, wanvideo.py:225-280)."""
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_block_i2v.pt"))
    D = g["x"].shape[-1]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=g["sd"]["ffn.fc_in.weight"].shape[0],
                               num_layers=1)
    blk = wan_dit.WanBlock(cuda_sd(g["sd"]), "", cfg)
    assert blk.w_kv_img is not None
    lay = wan_dit.make_layout(g["seq"], cfg, "cuda")
    y = wan_dit.block_forward(g["x"][0].cuda(), blk, g["ctx"][0].cuda(), g["temb6"].cuda(), lay, cfg)
    e, floor = assert_bf16_parity(y, g["y_fp32"][0], g["y_ref_bf16"][0], name="wan i2v block")
    assert rel_l2(y, g["y_ref_bf16"][0]) < 2 * floor


def test_model_dense_against_reference_golden(golden_dir):
    from fastvideo_b200 import wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = cuda_sd(g["sd"])
    D = sd["proj_out.weight"].shape[1]
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0],
                               num_layers=2, text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1])
    model = wan_dit.WanDiT(cfg, sd)
    y = model.forward(g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    assert y.shape == g["y_ref_bf16"].shape
    e, floor = assert_bf16_parity(y, g["y_fp32"], g["y_ref_bf16"], name="wan model")
    assert rel_l2(y, g["y_ref_bf16"]) < 2 * floor


def test_block_vsa_against_oracle():
    """WanTransformerBlock_VSA: the reference's sparse kernels are Triton-only (no CPU run), so the checker is the
    oracle restatement (tile -> video_sparse_attn -> untile, wanvideo.py:520-582). Our engine runs the block in
    compact tile-major order; results are compared in raster order on rows whose block lists agree."""
    from fastvideo_b200 import wan_dit
    torch.manual_seed(0)
    from oracle.gen_golden import _rand_block_sd  # seeded synthetic weights only; no reference import
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
    sd32 = {k: v.float() for k, v in sd.items()}
    with torch.no_grad():
        y_ref = wan_ref.wan_block(x, ctx, temb6, sd, "", H, cos, sin, vsa_meta=meta)
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=H, ffn_dim=F_, num_layers=1, vsa=True)
    blk = wan_dit.WanBlock(cuda_sd(sd), "", cfg)
    lay = wan_dit.make_layout(seq, cfg, "cuda", vsa_sparsity=0.5)
    assert lay.topk == meta["topk"]
    xp = x[0].cuda()[lay.perm]
    y = wan_dit.block_forward(xp, blk, ctx[0].cuda(), temb6.cuda(), lay, cfg)[lay.inv_perm]
    # bf16-vs-bf16 with a discontinuous block selection: compare in relative L2 over all rows, loosely, and
    # tightly over the bulk (rows whose selection did not flip)
    err_rows = (y.float().cpu() - y_ref[0].float()).norm(dim=-1) / y_ref[0].float().norm(dim=-1)
    assert err_rows.median().item() < 1e-2
    assert (err_rows < 3e-2).float().mean().item() > 0.9


def test_sequence_parallel_code_path_world1_matches_single_rank(golden_dir):
    """SPWanDiT at world size 1 exercises the head-scattered GEMM epilogue, the offset-aware RMSNorm/RoPE pass, the
    strided attention reads and the K-segmented out-projection -- with identity all-to-alls."""
    from fastvideo_b200 import wan_dit, distributed
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1])
    model = wan_dit.WanDiT(cfg, sd)
    args = (g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    y1 = model.forward(*args)
    y2 = distributed.SPWanDiT(model, 0, 1).forward(*args)
    assert torch.equal(y1, y2)


@pytest.mark.parametrize("vsa, weights", [(False, "int8_weights"), (False, "w8a8"), (True, "bf16"), (True, "int8_weights"),
                                          (True, "w8a8")], ids=lambda v: {False: "dense", True: "vsa"}.get(v, v))
def test_sequence_parallel_world1_matches_single_rank_vsa_and_int8(golden_dir, vsa, weights):
    """The world-1 check above with VSA attention and with int8 weights (weight-only and W8A8): the sequence-parallel
    out-projection and block tail match the single-rank forward bit for bit in every weight format."""
    from fastvideo_b200 import wan_dit, distributed
    fmt = {"bf16": {}, "int8_weights": dict(int8_weights=True), "w8a8": dict(int8_weights=True, int8_activations=True)}[weights]
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    sd = cuda_sd(g["sd"])
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], vsa=vsa, **fmt)
    if vsa:  # the checkpoint is a dense one: add the VSA gate projections
        gen = torch.Generator(device="cuda").manual_seed(0)
        for i in range(2):
            sd[f"blocks.{i}.to_gate_compress.weight"] = (torch.randn(cfg.hidden_size, cfg.hidden_size, device="cuda", generator=gen) / 16).bfloat16()
            sd[f"blocks.{i}.to_gate_compress.bias"] = torch.zeros(cfg.hidden_size, device="cuda").bfloat16()
    model = wan_dit.WanDiT(cfg, sd)
    args = (g["latents"].cuda(), g["text"].cuda(), g["timestep"].cuda())
    sparsity = 0.5 if vsa else None
    y1 = model.forward(*args, vsa_sparsity=sparsity)
    y2 = distributed.SPWanDiT(model, 0, 1).forward(*args, vsa_sparsity=sparsity)
    assert torch.equal(y1, y2)
