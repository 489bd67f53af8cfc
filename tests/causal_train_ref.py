"""CPU restatement of the causal Wan model's training forward (CausalWanTransformer3DModel._forward_train,
fastvideo/models/dits/causal_wanvideo.py:420-471): the whole sequence at once, self-attention under the block-causal mask
the reference builds for flex_attention (causal_wanvideo.py:10-15, 120-123), everything else as oracle.causal_ref's
rollout (per-frame modulation, float64 RoPE at absolute positions, the same embedder, text padding and head).

The reference tree is not available here, so this file is anchored to the golden-pinned rollout oracle instead
(tests/test_causal_train_cpu.py): with local_attn_size = -1, no sink and the absolute RoPE policy, frame block b of
causal_model_train equals a causal_ref.causal_model_inference rollout fed blocks 0..b with the same latents and timesteps.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.wan_ref import apply_rotary, rmsnorm, rotary_tables, sdpa, timestep_embedding


linear = F.linear  # module attribute, so a test can wrap every linear of the restatement


def _lin(x, w, b):
    # oracle.causal_ref._lin through `linear`
    return linear(x.to(w.dtype), w, b)


def block_causal_mask(frames: int, frame_seqlen: int, frames_per_block: int, local_attn_size: int = -1) -> torch.Tensor:
    """bool [S, S], S = frames * frame_seqlen: token i of frame block b = i // (n fs) attends key j iff j < end_b =
    min((b + 1) n fs, S) and, when local_attn_size != -1, j >= end_b - local_attn_size fs."""
    S, L = frames * frame_seqlen, frames_per_block * frame_seqlen
    i = torch.arange(S)
    end = torch.clamp((i // L + 1) * L, max=S)[:, None]
    j = i[None, :]
    keep = j < end
    if local_attn_size != -1:
        keep &= j >= end - local_attn_size * frame_seqlen
    return keep


def causal_block_train(x, ctx, temb, sd, prefix, num_heads, cos, sin, mask, eps=1e-6):
    """oracle.causal_ref.causal_block with the KV-cache attention replaced by SDPA over all S tokens under `mask`
    ([S, S] bool). x [B, S, D], temb [B, F, 6, D], cos / sin for the S tokens."""
    g = lambda n: sd[prefix + n]
    B, S, D = x.shape
    H = num_heads
    d = D // H
    nf = temb.shape[1]
    tpf = S // nf
    orig = x.dtype
    e = g("scale_shift_table") + temb
    shift_msa, scale_msa, gate_msa, c_shift, c_scale, c_gate = e.chunk(6, dim=2)
    n1 = (F.layer_norm(x, (D,), None, None, eps).unflatten(1, (nf, tpf)) * (1 + scale_msa) + shift_msa).flatten(1, 2)
    q = rmsnorm(_lin(n1, g("to_q.weight"), g("to_q.bias")), g("norm_q.weight"), eps).unflatten(2, (H, d))
    k = rmsnorm(_lin(n1, g("to_k.weight"), g("to_k.bias")), g("norm_k.weight"), eps).unflatten(2, (H, d))
    v = _lin(n1, g("to_v.weight"), g("to_v.bias")).unflatten(2, (H, d))
    rq = apply_rotary(q, cos, sin).type_as(v)
    rk = apply_rotary(k, cos, sin).type_as(v)
    a = _lin(sdpa(rq, rk, v, mask=mask.to(x.device)).flatten(2), g("to_out.weight"), g("to_out.bias"))
    r = x + (a.unflatten(1, (nf, tpf)) * gate_msa).flatten(1, 2)
    n2 = F.layer_norm(r, (D,), g("self_attn_residual_norm.norm.weight"), g("self_attn_residual_norm.norm.bias"), eps)
    n2, x = n2.to(orig), r.to(orig)
    q2 = rmsnorm(_lin(n2, g("attn2.to_q.weight"), g("attn2.to_q.bias")), g("attn2.norm_q.weight"), eps).view(B, -1, H, d)
    k2 = rmsnorm(_lin(ctx, g("attn2.to_k.weight"), g("attn2.to_k.bias")), g("attn2.norm_k.weight"), eps).view(B, -1, H, d)
    v2 = _lin(ctx, g("attn2.to_v.weight"), g("attn2.to_v.bias")).view(B, -1, H, d)
    a2 = _lin(sdpa(q2, k2, v2).flatten(2), g("attn2.to_out.weight"), g("attn2.to_out.bias"))
    r = x + a2
    n3 = (F.layer_norm(r, (D,), None, None, eps).unflatten(1, (nf, tpf)) * (1.0 + c_scale) + c_shift).flatten(1, 2)
    f = _lin(F.gelu(_lin(n3, g("ffn.fc_in.weight"), g("ffn.fc_in.bias")), approximate="tanh"),
             g("ffn.fc_out.weight"), g("ffn.fc_out.bias"))
    return r + (f.unflatten(1, (nf, tpf)) * c_gate).flatten(1, 2)


def causal_model_train(latents, text, timestep, sd, num_heads, num_frames_per_block, start_frame=0, local_attn_size=-1,
                       text_len=512, patch_size=(1, 2, 2), freq_dim=256, eps=1e-6):
    """latents [B, C, F, H, W], text [B, L, text_dim], timestep [B, F] -> flow prediction [B, C, F, H, W]; the embedder,
    padding and per-frame head of oracle.causal_ref.causal_model_inference."""
    B, C, T, Hh, Ww = latents.shape
    pt, ph, pw = patch_size
    seq = (T // pt, Hh // ph, Ww // pw)
    fs = seq[1] * seq[2]
    D = sd["patch_embedding.proj.weight"].shape[0]
    d = D // num_heads
    cos, sin = rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)], start_frame=start_frame, keep_f64=True)
    cos, sin = cos.to(latents.device), sin.to(latents.device)
    mask = block_causal_mask(seq[0], fs, num_frames_per_block, local_attn_size)
    x = F.conv3d(latents, sd["patch_embedding.proj.weight"], sd["patch_embedding.proj.bias"], stride=patch_size)
    x = x.flatten(2).transpose(1, 2)
    text = torch.cat([text, text.new_zeros(B, text_len - text.size(1), text.size(2))], dim=1)
    ce = "condition_embedder."
    wdt = sd[ce + "time_embedder.mlp.fc_in.weight"].dtype
    t_freq = timestep_embedding(timestep.flatten(), freq_dim).to(wdt)
    temb = F.linear(F.silu(F.linear(t_freq, sd[ce + "time_embedder.mlp.fc_in.weight"], sd[ce + "time_embedder.mlp.fc_in.bias"])),
                    sd[ce + "time_embedder.mlp.fc_out.weight"], sd[ce + "time_embedder.mlp.fc_out.bias"])
    tproj = F.linear(F.silu(temb), sd[ce + "time_modulation.linear.weight"], sd[ce + "time_modulation.linear.bias"])
    tproj = tproj.unflatten(1, (6, D)).unflatten(0, timestep.shape)  # [B, F, 6, D]
    ctx = F.linear(F.gelu(F.linear(text, sd[ce + "text_embedder.fc_in.weight"], sd[ce + "text_embedder.fc_in.bias"]),
                          approximate="tanh"), sd[ce + "text_embedder.fc_out.weight"], sd[ce + "text_embedder.fc_out.bias"])
    i = 0
    while f"blocks.{i}.to_q.weight" in sd:
        x = causal_block_train(x, ctx, tproj, sd, f"blocks.{i}.", num_heads, cos, sin, mask, eps)
        i += 1
    te = temb.unflatten(0, timestep.shape).unsqueeze(2)
    shift, scale = (sd["scale_shift_table"].unsqueeze(1) + te).chunk(2, dim=2)  # [B, F, 1, D]
    nf = te.shape[1]
    n = F.layer_norm(x, (D,), None, None, eps)
    n = (n.unflatten(1, (nf, -1)) * (1.0 + scale) + shift).flatten(1, 2)
    y = F.linear(n, sd["proj_out.weight"], sd["proj_out.bias"])
    y = y.reshape(B, seq[0], seq[1], seq[2], pt, ph, pw, -1).permute(0, 7, 1, 4, 2, 5, 3, 6)
    return y.flatten(6, 7).flatten(4, 5).flatten(2, 3)
