"""Times one Wan 14B block for training at 720p x 81 frames (S = 75 600 tokens, 512 text tokens), dense and VSA
(sparsity 0.9), and writes one JSON line per measurement to stdout and to tool_out/block_bwd.jsonl. The card's name and
power limit are part of every line.

  engine   wan_dit.block_forward: forward without grad, forward with grad, backward (CUDA events, median of --iters),
           peak memory of forward + backward
  stages   one engine forward + backward under torch.profiler (a run of its own): CUDA time per kernel family; the block's
           linears counted from shapes (forward 2 M N K each, backward twice that) over the GEMM kernels' time, against the
           data sheet's 989 TFLOP/s; the new row kernels' bytes (from shapes) over their time, against 3.35 TB/s
  routed   the current way to train this block: oracle.wan_ref.wan_block in bf16 with its linears on plugin.linear_forward,
           its RMSNorms on plugin.rms_norm_forward_cuda, dense attention on attention.B200AttentionImpl and VSA on the
           plug-in's differentiable vsa.video_sparse_attn (padded layout), torch for the rest; forward + backward with CUDA
           events. When it runs out of memory the token count is halved until it fits, and the line says so.

    python tools/gpu_bench_block_bwd.py [--iters 3] [--skip-routed]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35


def linear_flops(S, L, D, F, vsa):
    """Forward FLOPs of the block's linears: qkv(+gate), to_out, q2, to_out2 on S tokens, text K/V on L, fc_in, fc_out."""
    return 2 * S * D * D * (4 if vsa else 3) + 2 * S * D * D * 3 + 2 * L * D * 2 * D + 2 * S * D * F * 2


def row_bytes(S, D):
    """Bytes each new row kernel moves per launch (reads + writes of its [S, D] operands), by demangled-name substring."""
    e = S * D
    return {"resid_gate_bwd_kernel<true>": 10 * e,     # fp32 dout, bf16 y, bf16 dy (to_out, fp32 residual stream)
            "resid_gate_bwd_kernel<false>": 6 * e,     # bf16 dout (fc_out)
            "layernorm_modulate_bwd_kernel<false, true>": 10 * e,   # norm1: bf16 x, dn, fp32 gin, bf16 dx
            "layernorm_modulate_bwd_kernel<true, false>": 12 * e,   # norm2: fp32 y, bf16 dn, bf16 gin, fp32 dy
            "layernorm_modulate_bwd_kernel<false, false>": 8 * e,   # norm3: bf16 x, dn, gin, dx
            "rmsnorm_rope_bwd_kernel": 12 * e}         # q and k: bf16 x, dy, dx each


def emit(rec):
    line = json.dumps(rec)
    print(line, flush=True)
    with open(os.path.join("tool_out", "block_bwd.jsonl"), "a") as f:
        f.write(line + "\n")


def make_engine(vsa, seq, text):
    from fastvideo_b200 import wan_dit
    cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_14B, "num_layers": 1, "vsa": vsa})
    sd = wan_dit.random_state_dict(cfg, "cuda", 7, layers=1)
    blk = wan_dit.WanBlock(sd, "blocks.0.", cfg)
    for n, t in blk.tensors().items():
        setattr(blk, n, t.detach().requires_grad_(True))
    lay = wan_dit.make_layout(seq, cfg, "cuda", 0.9 if vsa else None)
    S, D = lay.cos.shape[0], cfg.hidden_size
    x = (torch.randn(S, D, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    ctx = torch.randn(text, D, device="cuda").bfloat16()
    temb6 = (torch.randn(1, 6, D, device="cuda") * 0.1).bfloat16()
    return cfg, blk, lay, x, ctx, temb6, sd


def time_engine(card, vsa, seq, text, iters):
    from fastvideo_b200 import wan_dit
    cfg, blk, lay, x, ctx, temb6, sd = make_engine(vsa, seq, text)
    del sd
    S, D = x.shape
    dy = torch.randn(S, D, device="cuda").bfloat16()
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t_nograd, t_fwd, t_bwd, peak = [], [], [], 0
    for it in range(iters + 1):
        for t in [x, *blk.tensors().values()]:
            t.grad = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        e0, e1, e2, e3 = ev(), ev(), ev(), ev()
        e0.record()
        with torch.no_grad():
            wan_dit.block_forward(x, blk, ctx, temb6, lay, cfg)
        e1.record()
        y = wan_dit.block_forward(x, blk, ctx, temb6, lay, cfg)
        e2.record()
        y.backward(dy)
        e3.record()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        del y
        if it:
            t_nograd.append(e0.elapsed_time(e1))
            t_fwd.append(e1.elapsed_time(e2))
            t_bwd.append(e2.elapsed_time(e3))
    med = lambda v: sorted(v)[len(v) // 2]
    name = "wan14b-vsa0.9" if vsa else "wan14b-dense"
    emit(dict(card=card, kind="engine", block=name, tokens=S, text=text, fwd_nograd_ms=med(t_nograd), fwd_grad_ms=med(t_fwd),
              bwd_ms=med(t_bwd), fwd_plus_bwd_ms=med(t_fwd) + med(t_bwd), peak_fwd_bwd_gib=peak / 2 ** 30))

    # per-stage: one forward + backward under the profiler
    from torch.profiler import ProfilerActivity, profile
    for t in [x, *blk.tensors().values()]:
        t.grad = None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        y = wan_dit.block_forward(x, blk, ctx, temb6, lay, cfg)
        y.backward(dy)
        torch.cuda.synchronize()
    del y
    kernels = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            us = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if us > 0:
                kernels[e.key] = kernels.get(e.key, 0.0) + us / 1e3
    gemm_ms = sum(v for k, v in kernels.items() if "gemm_kernel" in k or "gemm_aux_kernel" in k)
    fl = linear_flops(S, text, D, cfg.ffn_dim, vsa) * 3  # forward + dgrad + wgrad
    rows = {}
    for sub, nbytes in row_bytes(S, D).items():
        ms = sum(v for k, v in kernels.items() if sub in k)
        if ms > 0:
            rows[sub] = dict(ms=ms, tb_per_s=nbytes / ms / 1e9, share_of_3_35=nbytes / ms / 1e9 / PEAK_TBS)
    top = sorted(kernels.items(), key=lambda kv: -kv[1])[:14]
    emit(dict(card=card, kind="stages", block=name, tokens=S, gemm_kernels_ms=gemm_ms,
              linear_tflop_per_s=fl / gemm_ms / 1e9, linear_share_of_989=fl / gemm_ms / 1e9 / PEAK_TFLOPS,
              row_kernels=rows, top_kernels_ms={k[:90]: round(v, 3) for k, v in top},
              all_kernels_ms=round(sum(kernels.values()), 3)))
    del blk, x
    torch.cuda.empty_cache()


def _rms_self(weight, eps):
    return types.SimpleNamespace(weight=weight, variance_epsilon=eps, hidden_size=weight.numel(), has_weight=True,
                                 variance_size_override=None)


def time_routed(card, vsa, seq, text, iters):
    """The oracle block routed through the plug-in; returns False when it ran out of memory."""
    import numpy as np
    from fastvideo_b200 import plugin, vsa as fvb_vsa, wan_dit
    from fastvideo_b200.attention import B200AttentionImpl
    from oracle import vsa_index, wan_ref
    cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_14B, "num_layers": 1, "vsa": vsa})
    D, H, d = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim
    S = int(np.prod(seq))
    sd = {k[len("blocks.0."):]: v.requires_grad_(True)
          for k, v in wan_dit.random_state_dict(cfg, "cuda", 7, layers=1).items() if k.startswith("blocks.0.")}
    x = (torch.randn(1, S, D, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    ctx = torch.randn(1, text, D, device="cuda").bfloat16()
    temb6 = (torch.randn(1, 6, D, device="cuda") * 0.1).bfloat16()
    dy = torch.randn(1, S, D, device="cuda").bfloat16()
    cos, sin = (t.cuda() for t in wan_ref.rotary_tables(seq, [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)]))
    meta = None
    if vsa:
        tile = (4, 4, 4)
        vbs = torch.from_numpy(vsa_index.variable_block_sizes(seq, tile))
        meta = dict(tile_partition=torch.from_numpy(vsa_index.tile_partition_indices(seq, tile)).cuda(),
                    untile_combined=torch.from_numpy(vsa_index.untile_combined_index(seq, tile)).cuda(),
                    non_pad=torch.from_numpy(vsa_index.non_pad_index(vbs.numpy(), 64)).cuda(), vbs=vbs.cuda(),
                    s_pad=vbs.numel() * 64, topk=vsa_index.compute_topk(0.9, vbs.numel()))
    saved = wan_ref.linear, wan_ref.rmsnorm, wan_ref.video_sparse_attn
    wan_ref.linear = plugin.linear_forward
    wan_ref.rmsnorm = lambda t, w, eps=1e-6: plugin.rms_norm_forward_cuda(_rms_self(w, eps), t)
    wan_ref.video_sparse_attn = lambda q, k, v, vbs, topk, gate=None: fvb_vsa.video_sparse_attn(
        q, k, v, vbs, vbs, topk, 64, gate)
    attn = B200AttentionImpl(H, d).forward
    ev = lambda: torch.cuda.Event(enable_timing=True)
    t_fwd, t_bwd = [], []
    try:
        for it in range(iters + 1):
            for t in [x, *sd.values()]:
                t.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            e0, e1, e2 = ev(), ev(), ev()
            e0.record()
            with torch.device("cuda"):
                y = wan_ref.wan_block(x, ctx, temb6, sd, "", H, cos, sin, attn_fn=attn, vsa_meta=meta)
            e1.record()
            y.backward(dy)
            e2.record()
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            del y
            if it:
                t_fwd.append(e0.elapsed_time(e1))
                t_bwd.append(e1.elapsed_time(e2))
    except torch.cuda.OutOfMemoryError:
        return False
    finally:
        wan_ref.linear, wan_ref.rmsnorm, wan_ref.video_sparse_attn = saved
        del sd, x
        torch.cuda.empty_cache()
    med = lambda v: sorted(v)[len(v) // 2]
    emit(dict(card=card, kind="routed", block="wan14b-vsa0.9" if vsa else "wan14b-dense", tokens=S, text=text,
              fwd_ms=med(t_fwd), bwd_ms=med(t_bwd), fwd_plus_bwd_ms=med(t_fwd) + med(t_bwd), peak_fwd_bwd_gib=peak / 2 ** 30))
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--text", type=int, default=512)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--skip-routed", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    os.makedirs("tool_out", exist_ok=True)
    seq = (21, 60, 60)  # 720p x 81 frames after the VAE and (1, 2, 2) patches: 75 600 tokens
    for vsa in (False, True):
        time_engine(card, vsa, seq, args.text, args.iters)
        if args.skip_routed:
            continue
        frames = seq[0]
        while frames >= 1:
            s = (frames, seq[1], seq[2])
            if time_routed(card, vsa, s, args.text, args.iters):
                if frames != seq[0]:  # the engine at the same shape, for the comparison
                    emit(dict(card=card, kind="note", block="vsa" if vsa else "dense",
                              note=f"routed path out of memory at 75600 tokens; largest that fits: {s}"))
                    time_engine(card, vsa, s, args.text, args.iters)
                break
            emit(dict(card=card, kind="oom", block="vsa" if vsa else "dense", tokens=frames * seq[1] * seq[2]))
            frames //= 2


if __name__ == "__main__":
    main()
