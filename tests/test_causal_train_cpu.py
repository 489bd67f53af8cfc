"""CPU: the causal model's training forward -- block-causal tile tables against the token mask, the training oracle
(tests/causal_train_ref.py) against the golden-pinned rollout oracle, and CausalWanDiT.forward_train's refusals under grad."""
import os

import pytest
import torch

from causal_train_ref import block_causal_mask, causal_model_train
from oracle import causal_ref
from util import rel_l2


def _expand(q_off, kv_off, tile_map):
    """[nqb, nkb] tile map -> [S, S] token mask through the tile tables."""
    qt = torch.repeat_interleave(torch.arange(q_off.numel() - 1), (q_off[1:] - q_off[:-1]).long())
    kt = torch.repeat_interleave(torch.arange(kv_off.numel() - 1), (kv_off[1:] - kv_off[:-1]).long())
    return tile_map[qt][:, kt]


# (frames, frame_seqlen, frames_per_block, local_attn_size): n fs not a multiple of 64, F not a multiple of n, a window
# that is not a multiple of n (its starts cut inside blocks), and the 480p x 81-frame shape
CASES = [(4, 24, 2, -1), (5, 24, 2, -1), (7, 40, 3, -1), (7, 40, 3, 4), (8, 30, 3, 2), (21, 1560, 3, -1), (21, 1560, 3, 7)]


@pytest.mark.parametrize("frames,fs,n,local", CASES)
def test_tile_tables_expand_to_the_token_mask(frames, fs, n, local):
    from fastvideo_b200 import wan_dit
    q_off, kv_off, tile_map = wan_dit.block_causal_tile_map(frames, fs, n, local)
    S = frames * fs
    for off in (q_off, kv_off):
        sizes = off[1:] - off[:-1]
        assert off[0] == 0 and off[-1] == S and (sizes > 0).all() and (sizes <= 64).all()
    mask = block_causal_mask(frames, fs, n, local)
    assert torch.equal(_expand(q_off, kv_off, tile_map), mask)
    # batch 2: the [1, 1, nqb, nkb] map broadcasts over batch and heads, every sample gets the same mask
    assert torch.equal(_expand(q_off, kv_off, tile_map[None, None].expand(2, 1, -1, -1)[1, 0]), mask)
    # the q -> k lists (ascending, as ops.map_to_index writes them) and the transposed map's k -> q lists select the mask
    lists = [row.nonzero().flatten() for row in tile_map]
    rebuilt = torch.zeros_like(tile_map)
    for i, ks in enumerate(lists):
        rebuilt[i, ks] = True
    assert torch.equal(rebuilt, tile_map) and torch.equal(rebuilt.T.contiguous(), tile_map.T)


def test_block_causal_tile_count_at_480p():
    """480p x 81 frames (S = 32 760, fs = 1560, n = 3): the cuts at block ends add about 1 % more tiles than dense, and the
    mask keeps 28/49 of dense attention's (q, k) pairs."""
    from fastvideo_b200 import wan_dit
    q_off, kv_off, tile_map = wan_dit.block_causal_tile_map(21, 1560, 3)
    dense = -(-32760 // 64)
    assert q_off.numel() - 1 == kv_off.numel() - 1 == 7 * 74 and (q_off.numel() - 1) / dense < 1.02
    assert block_causal_mask(21, 1560, 3).float().mean().item() == pytest.approx(28 / 49)


def _rollout_case(golden_dir, frames=5, seed=0):
    g = torch.load(os.path.join(golden_dir, "wan_causal_model.pt"))
    sd = {k: v.float() for k, v in g["sd"].items()}
    gen = torch.Generator().manual_seed(seed)
    lat = torch.randn(1, 16, frames, 8, 12, generator=gen)
    t = torch.randint(0, 1000, (1, frames), generator=gen)
    return g, sd, lat, g["text"].float(), t


def test_training_oracle_equals_the_rollout_oracle(golden_dir):
    """local_attn_size = -1, no sink, absolute RoPE: frame block b of causal_model_train equals a causal_model_inference
    rollout fed blocks 0..b with the same latents and timesteps (fp32 on the CPU: summation order only). 5 frames in
    2-frame blocks, so the last block is shorter."""
    g, sd, lat, text, t = _rollout_case(golden_dir)
    H, n, frames = g["heads"], 2, lat.shape[2]
    fs = (lat.shape[3] // 2) * (lat.shape[4] // 2)
    with torch.no_grad():
        train = causal_model_train(lat, text, t, sd, H, n, text_len=g["text_len"])
        kv = [causal_ref.new_kv_cache(1, 21 * fs, H, 128, torch.float32) for _ in range(2)]
        xc = [{"is_init": False} for _ in range(2)]
        for f0 in range(0, frames, n):
            f1 = min(f0 + n, frames)
            y = causal_ref.causal_model_inference(lat[:, :, f0:f1], text, t[:, f0:f1], sd, H, kv, xc, current_start=f0 * fs,
                                                  start_frame=f0, text_len=g["text_len"])
            assert rel_l2(train[:, :, f0:f1], y) < 1e-5, f"frame block starting at {f0}"
    # and the mask matters: the first block differs from a forward in which it sees every frame
    full = causal_model_train(lat, text, t, sd, H, frames, text_len=g["text_len"])
    assert rel_l2(full[:, :, :n], train[:, :, :n]) > 1e-3


def _model(golden_dir, **cfg_kw):
    from fastvideo_b200 import causal_wan, wan_dit
    g = torch.load(os.path.join(golden_dir, "wan_causal_model.pt"))
    sd = dict(g["sd"])
    D = sd["proj_out.weight"].shape[1]
    if cfg_kw.get("vsa"):
        for i in range(2):
            sd[f"blocks.{i}.to_gate_compress.weight"] = torch.zeros(D, D, dtype=torch.bfloat16)
            sd[f"blocks.{i}.to_gate_compress.bias"] = torch.zeros(D, dtype=torch.bfloat16)
    if cfg_kw.pop("fp32_norms", False):
        sd["blocks.1.norm_k.weight"] = sd["blocks.1.norm_k.weight"].float()
    cfg = wan_dit.WanDiTConfig(hidden_size=D, num_attention_heads=g["heads"], ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0],
                               num_layers=2, text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1],
                               text_len=g["text_len"], **cfg_kw)
    return causal_wan.CausalWanDiT(cfg, sd, causal_wan.CausalConfig(num_frames_per_block=2)), g


@pytest.mark.parametrize("kind", ["fp32_rmsnorm_weights", "vsa"])
def test_forward_train_refusals_under_grad(golden_dir, kind):
    """An fp32-RMSNorm-weight model or a VSA-configured one raises FvbError under grad, before anything runs (here: before
    the CPU tensors are refused); without grad the same call gets as far as the CUDA check."""
    from fastvideo_b200 import ops
    model, g = _model(golden_dir, **({"vsa": True} if kind == "vsa" else {"fp32_norms": True}))
    lat, text, t = g["calls"][0]["latents"], g["text"], g["calls"][0]["timestep"]
    model.w_out.requires_grad_(True)
    with pytest.raises(ops.FvbError, match="vsa=False" if kind == "vsa" else "RMSNorm"):
        model.forward_train(lat, text, t)
    model.w_out.requires_grad_(False)
    with pytest.raises(ops.FvbError, match="CUDA"):
        model.forward_train(lat, text, t)


def test_causal_forwards_keep_refusing_grad(golden_dir):
    """forward and forward_inference stay inference-only."""
    from fastvideo_b200 import ops
    model, g = _model(golden_dir)
    lat = g["calls"][0]["latents"].clone().requires_grad_(True)
    with pytest.raises(ops.FvbError, match="no backward"):
        model.forward(lat, g["text"], g["calls"][0]["timestep"][:, 0])
    with pytest.raises(ops.FvbError, match="no backward"):
        model.forward_inference(lat, g["text"], g["calls"][0]["timestep"], None, None)


def test_checkpoint_bytes_per_frame_modulation():
    from fastvideo_b200 import wan_dit
    S, D, H = 32760, 1536, 12
    assert wan_dit.checkpoint_bytes_per_block(S, D, H, frames=21) - wan_dit.checkpoint_bytes_per_block(S, D, H) == 24 * 20 * D
