"""CPU: the causal-rollout oracle against the golden fixture produced by the reference's own CausalWanTransformerBlock,
and the host-side KV-cache bookkeeping (ring eviction) against the oracle's reference-style shifting cache."""
import os
import random

import torch

from oracle import causal_ref, wan_ref
from util import assert_equal_or_host_rounding


def test_oracle_reproduces_reference_causal_rollout(golden_dir):
    g = torch.load(os.path.join(golden_dir, "wan_causal_block.pt"))
    H, grid, nf = g["heads"], tuple(g["grid"]), g["frames_per_call"]
    fs = grid[0] * grid[1]
    cache = causal_ref.new_kv_cache(1, g["window_frames"] * fs, H, 128)
    xc = {"is_init": False}
    for c in g["calls"]:
        cos, sin = wan_ref.rotary_tables((nf, ) + grid, [44, 42, 42], start_frame=c["start_frame"], keep_f64=True)
        with torch.no_grad():
            y = causal_ref.causal_block(c["x"], g["ctx"], c["temb"], g["sd"], "", H, cos, sin, cache, c["start_frame"] * fs,
                                        g["window_frames"], g["sink_frames"], fs, crossattn_cache=xc)
        assert_equal_or_host_rounding(y, c["y_ref_bf16"], name="causal block")
        assert int(cache["local_end_index"]) == c["local_end_index"]
        assert_equal_or_host_rounding(cache["k"][:, :c["local_end_index"]], c["k_window"], name="cache window")


def test_ring_cache_matches_reference_shift():
    """KVCache.advance (ring head instead of a memory shift) attends the same key set, keeps the same counters and
    the same logical order as causal_wanvideo.py:122-176 on random rollouts, including windows shorter than the cache
    (which force the ordered layout) and rings whose size is not a multiple of the block."""
    from fastvideo_b200.causal_wan import KVCache
    rnd = random.Random(0)
    checked = 0
    for _ in range(150):
        fs, nf = rnd.choice([4, 6]), rnd.choice([1, 2, 3])
        window, sink = rnd.choice([3, 4, 5, 6, 7]), rnd.choice([0, 1, 2])
        cache_frames = rnd.choice([window, window, window + 1])
        if sink + nf > cache_frames:
            continue
        ref = causal_ref.new_kv_cache(1, cache_frames * fs, 1, 8, torch.float32)
        mine = KVCache(cache_frames * fs, 1, 8, "cpu", sink * fs)
        mine.k, mine.v = mine.k.float(), mine.v.float()
        for step in range(12):
            start = (step // 2) * nf * fs
            new = torch.randn(1, nf * fs, 1, 8)
            w0, w1 = causal_ref.cache_update(ref, new, new * 2, start, window, sink, fs)
            segs, (k0, k1) = mine.advance(start, nf * fs, window, fs)
            r = 0
            for a, b in segs:
                mine.k[a:b], mine.v[a:b] = new[0, r:r + b - a], new[0, r:r + b - a] * 2
                r += b - a
            assert r == nf * fs
            want = sorted(map(tuple, ref["k"][0, w0:w1].reshape(w1 - w0, -1).tolist()))
            got = sorted(map(tuple, mine.k[k0:k1].reshape(k1 - k0, -1).tolist()))
            assert want == got
            assert mine.local_end_index == ref["local_end_index"] and mine.global_end_index == ref["global_end_index"]
            assert torch.equal(mine.logical(mine.k, 0, mine.local_end_index), ref["k"][0, :ref["local_end_index"]])
            assert torch.equal(mine.logical(mine.v, 0, mine.local_end_index), ref["v"][0, :ref["local_end_index"]])
            checked += 1
    assert checked > 1000


def test_local_attn_minus_one_rejects_rollouts_past_21_frames():
    from fastvideo_b200.causal_wan import KVCache
    import pytest
    c = KVCache(21 * 4, 1, 8, "cpu")
    for f in range(0, 21, 3):
        c.advance(f * 4, 12, -1, 4)
    with pytest.raises(ValueError):
        c.advance(21 * 4, 12, -1, 4)


def test_oracle_reproduces_reference_causal_model_rollout(golden_dir):
    g = torch.load(os.path.join(golden_dir, "wan_causal_model.pt"))
    H, window, sink = g["heads"], g["window_frames"], g["sink_frames"]
    c0 = g["calls"][0]["latents"]
    fs = (c0.shape[3] // 2) * (c0.shape[4] // 2)
    kv = [causal_ref.new_kv_cache(1, window * fs, H, 128) for _ in range(2)]
    xc = [{"is_init": False} for _ in range(2)]
    for c in g["calls"]:
        with torch.no_grad():
            y = causal_ref.causal_model_inference(c["latents"], g["text"], c["timestep"], g["sd"], H, kv, xc,
                                                  current_start=c["start_frame"] * fs, start_frame=c["start_frame"],
                                                  local_attn_size=window, sink_size=sink, text_len=g["text_len"])
        assert_equal_or_host_rounding(y, c["y_ref_bf16"], tol=6e-3, name="causal model")  # 2 blocks + head: the flips compound


def test_oracle_reproduces_reference_relativistic_rollouts(golden_dir):
    """rope_cache_policy == "relativistic": block and 2-layer model rollouts of the reference (oracle/gen_golden.py
    `causal_rel`, `causal_model_rel`)."""
    g = torch.load(os.path.join(golden_dir, "wan_causal_block_rel.pt"))
    H, grid, nf, window = g["heads"], tuple(g["grid"]), g["frames_per_call"], g["window_frames"]
    fs = grid[0] * grid[1]
    cache = causal_ref.new_kv_cache(1, window * fs, H, 128)
    xc = {"is_init": False}
    cos, sin = wan_ref.rotary_tables((window, ) + grid, [44, 42, 42], start_frame=0, keep_f64=True)
    for c in g["calls"]:
        with torch.no_grad():
            y = causal_ref.causal_block(c["x"], g["ctx"], c["temb"], g["sd"], "", H, cos, sin, cache, c["start_frame"] * fs,
                                        window, g["sink_frames"], fs, crossattn_cache=xc, rope_cache_policy="relativistic")
        assert_equal_or_host_rounding(y, c["y_ref_bf16"], name="relativistic block")
        assert int(cache["local_end_index"]) == c["local_end_index"]
    g = torch.load(os.path.join(golden_dir, "wan_causal_model_rel.pt"))
    H, window, sink = g["heads"], g["window_frames"], g["sink_frames"]
    c0 = g["calls"][0]["latents"]
    fs = (c0.shape[3] // 2) * (c0.shape[4] // 2)
    kv = [causal_ref.new_kv_cache(1, window * fs, H, 128) for _ in range(2)]
    xc = [{"is_init": False} for _ in range(2)]
    for c in g["calls"]:
        with torch.no_grad():
            y = causal_ref.causal_model_inference(c["latents"], g["text"], c["timestep"], g["sd"], H, kv, xc,
                                                  current_start=c["start_frame"] * fs, start_frame=c["start_frame"],
                                                  local_attn_size=window, sink_size=sink, text_len=g["text_len"],
                                                  rope_cache_policy="relativistic")
        assert_equal_or_host_rounding(y, c["y_ref_bf16"], tol=6e-3, name="relativistic model")


def test_causal_model_refuses_i2v_blocks():
    """The causal rollout's cross-attention is text-only (WanT2VCrossAttention): a checkpoint whose blocks carry the I2V
    image-token projections is refused at load instead of running an image branch the causal reference does not have."""
    import pytest
    from fastvideo_b200 import causal_wan, ops, wan_dit
    cfg = wan_dit.WanDiTConfig(hidden_size=64, num_attention_heads=1, ffn_dim=128, num_layers=1, text_dim=32, freq_dim=16)
    sd = wan_dit.random_state_dict(cfg, device="cpu")
    causal_wan.CausalWanDiT(cfg, sd, causal_wan.CausalConfig())  # the text-to-video checkpoint loads
    D = cfg.hidden_size
    for n in ("add_k_proj", "add_v_proj"):
        sd[f"blocks.0.attn2.{n}.weight"] = torch.zeros(D, D, dtype=torch.bfloat16)
        sd[f"blocks.0.attn2.{n}.bias"] = torch.zeros(D, dtype=torch.bfloat16)
    sd["blocks.0.attn2.norm_added_k.weight"] = torch.ones(D, dtype=torch.bfloat16)
    with pytest.raises(ops.FvbError, match="text-only"):
        causal_wan.CausalWanDiT(cfg, sd, causal_wan.CausalConfig())


def test_window_positions_follow_the_reference_order():
    """KVCache.window_positions: the position the relativistic policy gives a physical row equals the row's index in the
    reference's shifted (logical) window, for every ring state of random rollouts."""
    from fastvideo_b200.causal_wan import KVCache
    rnd = random.Random(1)
    checked = 0
    for _ in range(60):
        fs, nf = rnd.choice([4, 6]), rnd.choice([1, 2, 3])
        window, sink = rnd.choice([4, 5, 6, 7]), rnd.choice([0, 1, 2])
        if sink + nf > window:
            continue
        ref = causal_ref.new_kv_cache(1, window * fs, 1, 8, torch.float32)
        mine = KVCache(window * fs, 1, 8, "cpu", sink * fs)
        mine.k, mine.v = mine.k.float(), mine.v.float()
        for step in range(10):
            start = step * nf * fs
            new = torch.randn(1, nf * fs, 1, 8)
            w0, w1 = causal_ref.cache_update(ref, new, new, start, window, sink, fs)
            segs, (k0, k1) = mine.advance(start, nf * fs, window, fs)
            r = 0
            for a, b in segs:
                mine.k[a:b] = new[0, r:r + b - a]
                r += b - a
            pos = mine.window_positions(k0, k1).long()
            assert sorted(pos.tolist()) == list(range(w1 - w0))
            assert torch.equal(mine.k[k0:k1], ref["k"][0, w0:w1][pos])
            checked += 1
    assert checked > 300
