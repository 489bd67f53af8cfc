"""CPU: WanDiT.tensors() / WanDiT.to_reference_names -- the engine's trainable tensors map back to the reference state dict
(names, shapes, values) as views, and the mapped dict rebuilds the same model."""
import os

import pytest
import torch


def _golden_sd(golden_dir):
    return dict(torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))["sd"])


def _vsa_sd():
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(hidden_size=256, num_attention_heads=2, ffn_dim=512, num_layers=2, text_dim=64, vsa=True)
    return wan_dit.random_state_dict(cfg, "cpu", 17)


def _cfg(sd):
    from fastvideo_b200 import wan_dit
    return wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=2,
                                ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                                text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1],
                                vsa="blocks.0.to_gate_compress.weight" in sd)


@pytest.mark.parametrize("kind", ["dense_golden", "vsa_random"])
def test_reference_names_round_trip(golden_dir, kind):
    from fastvideo_b200 import wan_dit
    sd = _golden_sd(golden_dir) if kind == "dense_golden" else _vsa_sd()
    cfg = _cfg(sd)
    model = wan_dit.WanDiT(cfg, sd)
    own = model.tensors()
    assert len(own) == 15 + 2 * 21  # model tensors + two blocks (the VSA gate rows live in w_qkv / b_qkv)
    back = model.to_reference_names(own)
    assert sorted(back) == sorted(sd)
    storages = {t.untyped_storage().data_ptr() for t in own.values()}
    for k, v in sd.items():
        got = back[k]
        assert got.shape == v.shape, k
        # the engine keeps the residual LayerNorm's affine parameters in fp32 (exact for bf16 values)
        assert got.dtype == (torch.float32 if "self_attn_residual_norm" in k else v.dtype), k
        assert torch.equal(got.to(v.dtype), v), k
        assert got.untyped_storage().data_ptr() in storages, f"{k} is not a view of an engine tensor"
    rebuilt = wan_dit.WanDiT(cfg, back)
    for n, t in rebuilt.tensors().items():
        assert t.dtype == own[n].dtype and torch.equal(t, own[n]), n


def test_reference_names_of_gradients(golden_dir):
    """The same keys holding gradient-shaped tensors map the same way (what an optimizer or a checkpoint writer reads)."""
    from fastvideo_b200 import wan_dit
    sd = _golden_sd(golden_dir)
    model = wan_dit.WanDiT(_cfg(sd), sd)
    g = torch.Generator().manual_seed(0)
    grads = {n: torch.randn(t.shape, generator=g).to(t.dtype) for n, t in model.tensors().items()}
    back = model.to_reference_names(grads)
    assert torch.equal(back["patch_embedding.proj.weight"].reshape(grads["w_patch"].shape), grads["w_patch"])
    assert torch.equal(back["blocks.1.to_v.weight"], grads["blocks.1.w_qkv"][512:768])
    assert torch.equal(back["blocks.0.attn2.to_v.bias"], grads["blocks.0.b_kv2"][256:])
    assert all(back[k].shape == v.shape for k, v in sd.items())


def test_reference_names_of_partial_gradients():
    """A partly frozen model's .grads (None for the tensors not trained) map to None under the same names; the patch
    embedding takes the model's own patch size."""
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(hidden_size=256, num_attention_heads=2, ffn_dim=512, num_layers=2, text_dim=64,
                               patch_size=(2, 2, 2))
    sd = wan_dit.random_state_dict(cfg, "cpu", 5)
    model = wan_dit.WanDiT(cfg, sd)
    g = torch.Generator().manual_seed(1)
    frozen = lambda n: n.startswith("blocks.0.") or n in ("w_patch", "b_t1") or n.endswith("w_qkv")
    grads = {n: None if frozen(n) else torch.randn(t.shape, generator=g).to(t.dtype) for n, t in model.tensors().items()}
    back = model.to_reference_names(grads)
    assert sorted(back) == sorted(sd)
    for k in sd:
        want_none = (k.startswith("blocks.0.") or k in ("patch_embedding.proj.weight",
                                                         "condition_embedder.time_embedder.mlp.fc_in.bias")
                     or k.endswith(("to_q.weight", "to_k.weight", "to_v.weight")) and "attn2" not in k)
        assert (back[k] is None) == want_none, k
        if back[k] is not None:
            assert back[k].shape == sd[k].shape, k
    grads["w_patch"] = torch.zeros_like(model.w_patch)
    assert model.to_reference_names(grads)["patch_embedding.proj.weight"].shape == (256, 16, 2, 2, 2)


def test_checkpoint_bytes_formula():
    """The per-block checkpoint of DESIGN.md ("Wan model backward"), at Wan 1.3B, 480p x 81 frames."""
    from fastvideo_b200 import wan_dit
    S, D, H = 32760, 1536, 12
    dense = wan_dit.checkpoint_bytes_per_block(S, D, H)
    assert dense == 4 * S * D + 4 * S * H + 24 * D
    assert 0.2e9 < dense < 0.205e9
    n = 6 * 8 * 13  # 4 x 4 x 4 tiles over the (21, 30, 52) token grid
    n8 = (n + 7) // 8 * 8
    vsa = wan_dit.checkpoint_bytes_per_block(S, D, H, n)
    assert vsa - dense == H * (512 * n8 + 512 * n + 2 * n * n8 + 5 * n * n + 4 * n)


def test_causal_model_refuses_grad(golden_dir):
    """The causal model has no backward: its forward and forward_inference raise FvbError under grad with an input or a
    model tensor requiring grad, before anything runs."""
    from fastvideo_b200 import causal_wan, ops
    sd = _golden_sd(golden_dir)
    model = causal_wan.CausalWanDiT(_cfg(sd), sd, causal_wan.CausalConfig())
    g = torch.load(os.path.join(golden_dir, "wan_model_dense.pt"))
    lat, text, t = g["latents"], g["text"], g["timestep"]
    for train in ("latents", "w_out"):
        x = lat.clone().requires_grad_(train == "latents")
        model.w_out.requires_grad_(train == "w_out")
        with pytest.raises(ops.FvbError, match="no backward"):
            model.forward(x, text, t)
        with pytest.raises(ops.FvbError, match="no backward"):
            model.forward_inference(x, text, t.view(1, 1), None, None)
    model.w_out.requires_grad_(False)
    with torch.no_grad(), pytest.raises(ops.FvbError, match="CUDA"):  # no grad: it runs (and finds CPU tensors)
        model.forward(lat, text, t)
