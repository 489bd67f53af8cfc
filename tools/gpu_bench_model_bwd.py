"""Times a training step of the whole Wan 1.3B model (random weights, 30 layers) at 480p x 81 frames (latents
[1, 16, 21, 60, 104], S = 32 760 tokens, 512 text tokens), dense and VSA (sparsity 0.9), and writes one JSON line per
measurement to stdout and to tool_out/model_bwd.jsonl. The card's name, power limit and max SM clock are part of every line.

  engine     WanDiT.forward with checkpoint=True: per phase (forward without grad, forward with grad, MSE flow-matching loss
             against a random target, backward including the recompute, the whole step = the last three), CUDA events,
             medians of --iters; max_memory_allocated of the step; model TFLOP/s from shapes (see model_flops)
  recompute  8 layers (where keeping every activation still fits): steps with and without checkpoint, alternated
  routed     the way to train through the plug-in without the engine: oracle.wan_ref.wan_model in bf16 with its linears on
             plugin.linear_forward, RMSNorms on plugin.rms_norm_forward_cuda, dense attention on B200AttentionImpl and VSA
             on vsa.video_sparse_attn, torch.utils.checkpoint around each block; same shapes

    python tools/gpu_bench_model_bwd.py [--iters 3] [--skip-routed | --routed-only] [--attention dense|vsa|both]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LATENTS = (1, 16, 21, 60, 104)
TEXT = 512


def emit(rec):
    line = json.dumps(rec)
    print(line, flush=True)
    with open(os.path.join("tool_out", "model_bwd.jsonl"), "a") as f:
        f.write(line + "\n")


def model_flops(cfg, S, L, layers, topk_tiles=None):
    """Forward FLOPs of the model counted from shapes: every linear (2 M N K: patch embedding, per block qkv(+gate),
    to_out, q2, text K/V, to_out2, fc_in, fc_out, and proj_out; the embedders on one row or the text rows), self-attention
    (dense 4 S^2 D; VSA the selected tiles, 4 S (64 topk) D, plus the compression branch, 4 n^2 D over n tiles) and
    cross-attention 4 S L D. A training step counts 3x the forward (the backward is two GEMMs per forward GEMM); the
    checkpoint recompute is not counted."""
    D, F = cfg.hidden_size, cfg.ffn_dim
    blk = 2 * S * D * D * (4 if cfg.vsa else 3) + 2 * S * D * D * 3 + 2 * L * D * 2 * D + 2 * S * D * F * 2 + 4 * S * L * D
    if topk_tiles is None:
        blk += 4 * S * S * D
    else:
        n = math.ceil(S / 64)
        blk += 4 * S * 64 * topk_tiles * D + 4 * n * n * D
    head = 2 * S * 64 * D * 2 + 2 * L * (cfg.text_dim + D) * D
    return layers * blk + head


def make_inputs(cfg, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lat = torch.randn(LATENTS, device="cuda", generator=g).bfloat16()
    text = torch.randn(1, TEXT, cfg.text_dim, device="cuda", generator=g).bfloat16()
    target = torch.randn(LATENTS, device="cuda", generator=g).bfloat16()
    return lat, text, torch.tensor([700.0], device="cuda"), target


def step_times(model, lat, text, t, target, sparsity, checkpoint, with_nograd=True):
    """One step: (ms per phase, max_memory_allocated of the step in bytes)."""
    ev = lambda: torch.cuda.Event(enable_timing=True)
    e = [ev() for _ in range(5)]
    e[0].record()
    if with_nograd:
        with torch.no_grad():
            model.forward(lat, text, t, vsa_sparsity=sparsity)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e[1].record()
    y = model.forward(lat, text, t, vsa_sparsity=sparsity, checkpoint=checkpoint)
    e[2].record()
    loss = torch.nn.functional.mse_loss(y.float(), target.float())
    e[3].record()
    loss.backward()
    e[4].record()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    for p in model.tensors().values():
        p.grad = None
    del y, loss
    ms = dict(fwd_nograd=e[0].elapsed_time(e[1]) if with_nograd else None, fwd_grad=e[1].elapsed_time(e[2]),
              loss=e[2].elapsed_time(e[3]), bwd=e[3].elapsed_time(e[4]), step=e[1].elapsed_time(e[4]))
    return ms, peak


def med(v):
    return sorted(v)[len(v) // 2]


def make_model(vsa, layers):
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_1_3B, "num_layers": layers, "vsa": vsa})
    model = wan_dit.WanDiT.random(cfg, "cuda", 11)
    for p in model.tensors().values():
        p.requires_grad_(True)
    return cfg, model


def time_engine(card, vsa, iters):
    cfg, model = make_model(vsa, 30)
    lat, text, t, target = make_inputs(cfg)
    sparsity = 0.9 if vsa else None
    step_times(model, lat, text, t, target, sparsity, True)  # warm-up
    runs = [step_times(model, lat, text, t, target, sparsity, True) for _ in range(iters)]
    phases = {k: med([r[0][k] for r in runs]) for k in runs[0][0]}
    S = math.prod(LATENTS[2:]) // 4
    lay = model.layout((LATENTS[2], LATENTS[3] // 2, LATENTS[4] // 2), lat.device, sparsity)
    fl = 3 * model_flops(cfg, S, TEXT, 30, lay.topk if vsa else None)
    emit(dict(card=card, kind="engine", model="wan1.3b-vsa0.9" if vsa else "wan1.3b-dense", layers=30, tokens=S, text=TEXT,
              phases_ms=phases, max_memory_allocated_gib=max(r[1] for r in runs) / 2 ** 30,
              model_tflop_per_s=fl / phases["step"] / 1e9, flops_counted="3 x forward (model_flops), recompute not counted"))
    del model
    torch.cuda.empty_cache()


def time_recompute(card, vsa, iters):
    cfg, model = make_model(vsa, 8)
    lat, text, t, target = make_inputs(cfg)
    sparsity = 0.9 if vsa else None
    for cp in (True, False):
        step_times(model, lat, text, t, target, sparsity, cp, with_nograd=False)
    res = {True: [], False: []}
    peak = {True: 0, False: 0}
    for _ in range(iters):
        for cp in (True, False):
            ms, p = step_times(model, lat, text, t, target, sparsity, cp, with_nograd=False)
            res[cp].append(ms["step"])
            peak[cp] = max(peak[cp], p)
    emit(dict(card=card, kind="recompute", model="wan1.3b-vsa0.9" if vsa else "wan1.3b-dense", layers=8,
              step_ms_checkpoint=med(res[True]), step_ms_no_checkpoint=med(res[False]),
              overhead=med(res[True]) / med(res[False]) - 1, max_memory_allocated_gib_checkpoint=peak[True] / 2 ** 30,
              max_memory_allocated_gib_no_checkpoint=peak[False] / 2 ** 30))
    del model
    torch.cuda.empty_cache()


def _rms_self(weight, eps):
    return types.SimpleNamespace(weight=weight, variance_epsilon=eps, hidden_size=weight.numel(), has_weight=True,
                                 variance_size_override=None)


def time_routed(card, vsa, iters):
    from torch.utils.checkpoint import checkpoint
    from fastvideo_b200 import plugin, vsa as fvb_vsa, wan_dit
    from fastvideo_b200.attention import B200AttentionImpl
    from oracle import vsa_index, wan_ref
    cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_1_3B, "vsa": vsa})
    H, d = cfg.num_attention_heads, cfg.head_dim
    sd = {k: v.requires_grad_(True) for k, v in wan_dit.random_state_dict(cfg, "cuda", 11).items()}
    lat, text, t, target = make_inputs(cfg)
    seq = (LATENTS[2], LATENTS[3] // 2, LATENTS[4] // 2)
    rope = tuple(x.cuda() for x in wan_ref.rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)]))
    meta = None
    if vsa:
        tile = (4, 4, 4)
        vbs = torch.from_numpy(vsa_index.variable_block_sizes(seq, tile))
        meta = dict(tile_partition=torch.from_numpy(vsa_index.tile_partition_indices(seq, tile)).cuda(),
                    untile_combined=torch.from_numpy(vsa_index.untile_combined_index(seq, tile)).cuda(),
                    non_pad=torch.from_numpy(vsa_index.non_pad_index(vbs.numpy(), 64)).cuda(), vbs=vbs.cuda(),
                    s_pad=vbs.numel() * 64, topk=vsa_index.compute_topk(0.9, vbs.numel()))
    saved = wan_ref.linear, wan_ref.rmsnorm, wan_ref.video_sparse_attn, wan_ref.wan_block
    block = wan_ref.wan_block
    wan_ref.linear = plugin.linear_forward
    wan_ref.rmsnorm = lambda x, w, eps=1e-6: plugin.rms_norm_forward_cuda(_rms_self(w, eps), x)
    wan_ref.video_sparse_attn = lambda q, k, v, vbs, topk, gate=None: fvb_vsa.video_sparse_attn(q, k, v, vbs, vbs, topk, 64,
                                                                                              gate)
    wan_ref.wan_block = lambda *a, **kw: checkpoint(block, *a, use_reentrant=False, **kw)
    attn = B200AttentionImpl(H, d).forward
    ev = lambda: torch.cuda.Event(enable_timing=True)
    steps, peak = [], 0
    try:
        for it in range(iters + 1):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = ev(), ev()
            e0.record()
            with torch.device("cuda"):
                y = wan_ref.wan_model(lat, text, t, sd, H, attn_fn=attn, vsa_meta=meta, rope=rope)
            torch.nn.functional.mse_loss(y.float(), target.float()).backward()
            e1.record()
            torch.cuda.synchronize()
            peak = max(peak, torch.cuda.max_memory_allocated())
            for p in sd.values():
                p.grad = None
            del y
            if it:
                steps.append(e0.elapsed_time(e1))
    except torch.cuda.OutOfMemoryError:
        emit(dict(card=card, kind="routed", model="wan1.3b-vsa0.9" if vsa else "wan1.3b-dense", oom=True))
        return
    finally:
        wan_ref.linear, wan_ref.rmsnorm, wan_ref.video_sparse_attn, wan_ref.wan_block = saved
        del sd
        torch.cuda.empty_cache()
    emit(dict(card=card, kind="routed", model="wan1.3b-vsa0.9" if vsa else "wan1.3b-dense", layers=30,
              step_ms=med(steps), max_memory_allocated_gib=peak / 2 ** 30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--skip-routed", action="store_true")
    ap.add_argument("--attention", choices=["dense", "vsa", "both"], default="both")
    ap.add_argument("--routed-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    os.makedirs("tool_out", exist_ok=True)
    for vsa in {"dense": (False,), "vsa": (True,), "both": (False, True)}[args.attention]:
        if not args.routed_only:
            time_engine(card, vsa, args.iters)
            time_recompute(card, vsa, args.iters)
        if not args.skip_routed:
            time_routed(card, vsa, args.iters)


if __name__ == "__main__":
    main()
