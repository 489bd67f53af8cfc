"""Times a training step of the causal Wan 1.3B model (random weights, 30 layers) at 480p x 81 frames (latents
[1, 16, 21, 60, 104], S = 32 760 tokens, 3-frame blocks, per-frame random timesteps, 512 text tokens) and writes one JSON
line per measurement to stdout and to tool_out/causal_train.jsonl. The card's name, power limit and max SM clock are part of
every line.

  engine     CausalWanDiT.forward_train with checkpoint=True, in the layout of tools/gpu_bench_model_bwd.py: forward without
             grad, forward with grad, backward (recompute included), the whole step (MSE loss against a random target),
             CUDA events, medians of --iters; max_memory_allocated of the step; model TFLOP/s on a block-causal FLOP model
  vs_dense   the same shapes through WanDiT.forward (dense self-attention, checkpoint=True), steps alternated with the causal one
  attention  block-causal attention forward / backward (the tile lists of forward_train) against dense ops.attention /
             ops.attention_bwd at S = 32 760, H = 12, each time ratio beside the mask's FLOP ratio (28/49)
  rowops     fvb_layernorm_modulate_grouped_bwd and fvb_resid_gate_grouped_bwd at the block's shapes: bytes from shapes over
             kernel time, against 3.35 TB/s

    python tools/gpu_bench_causal_train.py [--iters 3] [--layers 30]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_bench_model_bwd import LATENTS, TEXT, model_flops  # noqa: E402

N_PER_BLOCK = 3
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


CARD = {}


def emit(rec):
    line = json.dumps({**rec, **CARD})
    print(line, flush=True)
    with open(os.path.join("tool_out", "causal_train.jsonl"), "a") as f:
        f.write(line + "\n")


def timed(fn, iters, warmup=1):
    """Median milliseconds of fn() over iters, CUDA events."""
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def causal_pairs(F_, fs, n, local=-1):
    """(q, k) token pairs the block-causal mask keeps: sum over tokens of end_b (or the window)."""
    S, L = F_ * fs, n * fs
    total = 0
    for b0 in range(0, S, L):
        end = min(b0 + L, S)
        keys = end if local == -1 else min(end, local * fs)
        total += (end - b0) * keys
    return total


def causal_flops(cfg, S, L, layers, F_, fs):
    """model_flops with dense self-attention (4 S^2 D per block) replaced by the block-causal pairs (4 pairs D)."""
    return model_flops(cfg, S, L, layers) - layers * 4 * S * S * cfg.hidden_size + layers * 4 * causal_pairs(F_, fs, N_PER_BLOCK) * cfg.hidden_size


def bench_models(args):
    from fastvideo_b200 import causal_wan, wan_dit
    cfg = wan_dit.WanDiTConfig(**{**wan_dit.WAN_1_3B, "num_layers": args.layers})
    g = torch.Generator(device="cuda").manual_seed(0)
    lat = torch.randn(LATENTS, device="cuda", generator=g).bfloat16()
    text = torch.randn(1, TEXT, cfg.text_dim, device="cuda", generator=g).bfloat16()
    target = torch.randn(LATENTS, device="cuda", generator=g).bfloat16()
    F_ = LATENTS[2]
    fs = (LATENTS[3] // 2) * (LATENTS[4] // 2)
    S = F_ * fs
    t_frames = torch.randint(0, 1000, (1, F_), device="cuda", generator=g)
    causal = causal_wan.CausalWanDiT.random(cfg, causal_wan.CausalConfig(num_frames_per_block=N_PER_BLOCK), "cuda", 5)
    for p in causal.tensors().values():
        p.requires_grad_(True)

    def zero(m):
        for p in m.tensors().values():
            p.grad = None

    def fwd_nograd():
        with torch.no_grad():
            causal.forward_train(lat, text, t_frames)

    def fwd_grad():
        return causal.forward_train(lat, text, t_frames, checkpoint=True)

    def step_causal():
        zero(causal)
        y = causal.forward_train(lat, text, t_frames, checkpoint=True)
        torch.nn.functional.mse_loss(y.float(), target.float()).backward()

    step_causal()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t_nograd = timed(fwd_nograd, args.iters)
    t_fwd = timed(lambda: fwd_grad(), args.iters)
    bwd = []
    for _ in range(args.iters):
        zero(causal)
        y = fwd_grad()
        loss = torch.nn.functional.mse_loss(y.float(), target.float())
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss.backward()
        b.record()
        torch.cuda.synchronize()
        bwd.append(a.elapsed_time(b))
    t_bwd = sorted(bwd)[len(bwd) // 2]
    torch.cuda.reset_peak_memory_stats()
    t_step = timed(step_causal, args.iters, warmup=0)
    peak = torch.cuda.max_memory_allocated()
    flops = 3 * causal_flops(cfg, S, TEXT, args.layers, F_, fs)
    emit(dict(kind="engine", model="causal", layers=args.layers, S=S, fwd_nograd_ms=t_nograd, fwd_grad_ms=t_fwd,
              bwd_ms=t_bwd, step_ms=t_step, max_memory_allocated_gb=peak / 1e9, step_flops=flops,
              model_tflops=flops / t_step / 1e9))
    # dense training on the same shapes and weights (WanDiT.forward, one timestep), steps alternated with the causal one
    t_one = t_frames[:, 0].float()

    def step_dense():
        zero(causal)
        y = wan_dit.WanDiT.forward(causal, lat, text, t_one, checkpoint=True)
        torch.nn.functional.mse_loss(y.float(), target.float()).backward()

    step_dense()
    ts = {"causal": [], "dense": []}
    for _ in range(args.iters):
        for name, fn in (("causal", step_causal), ("dense", step_dense)):
            ts[name].append(timed(fn, 1, warmup=0))
    med = {k: sorted(v)[len(v) // 2] for k, v in ts.items()}
    emit(dict(kind="vs_dense", layers=args.layers, S=S, causal_step_ms=med["causal"], dense_step_ms=med["dense"],
              time_ratio=med["causal"] / med["dense"],
              flop_ratio=causal_flops(cfg, S, TEXT, args.layers, F_, fs) / model_flops(cfg, S, TEXT, args.layers)))
    return fs, F_


def bench_attention(args, fs, F_):
    from fastvideo_b200 import ops, wan_dit
    S, H, d = F_ * fs, 12, 128
    g = torch.Generator(device="cuda").manual_seed(1)
    q, k, v, do = (torch.randn(1, S, H, d, device="cuda", generator=g).bfloat16() for _ in range(4))
    c = wan_dit.block_causal_tiles(F_, fs, N_PER_BLOCK, -1, "cuda")
    fwd_c = lambda: ops.attention_blocklist(q, k, v, c.q2k_idx, c.q2k_num, return_lse=True, q_off=c.q_off, kv_off=c.kv_off,
                                            nkb=c.nkb)
    fwd_d = lambda: ops.attention(q, k, v, return_lse=True)
    oc, lc = fwd_c()
    od, ld = fwd_d()
    bwd_c = lambda: ops.attention_sparse_bwd(q, k, v, oc, lc, do, c.q2k_idx, c.q2k_num, c.k2q_idx, c.k2q_num, q_off=c.q_off,
                                             kv_off=c.kv_off)
    bwd_d = lambda: ops.attention_bwd(q, k, v, od, ld, do)
    ratio = causal_pairs(F_, fs, N_PER_BLOCK) / S ** 2
    res = {}
    for name, fn in (("fwd_causal", fwd_c), ("fwd_dense", fwd_d), ("bwd_causal", bwd_c), ("bwd_dense", bwd_d)):
        res[name] = timed(fn, max(5, args.iters), warmup=2)
    dense_fwd_flops = 4 * S * S * H * d
    emit(dict(kind="attention", S=S, H=H, nqb=c.q_off.numel() - 1, nkb=c.nkb, **{k + "_ms": v for k, v in res.items()},
              fwd_time_ratio=res["fwd_causal"] / res["fwd_dense"], bwd_time_ratio=res["bwd_causal"] / res["bwd_dense"],
              flop_ratio=ratio, fwd_dense_tflops=dense_fwd_flops / res["fwd_dense"] / 1e9,
              fwd_causal_tflops=ratio * dense_fwd_flops / res["fwd_causal"] / 1e9,
              bwd_dense_tflops=2.5 * dense_fwd_flops / res["bwd_dense"] / 1e9,
              bwd_causal_tflops=2.5 * ratio * dense_fwd_flops / res["bwd_causal"] / 1e9))


def bench_rowops(args, fs, F_):
    from fastvideo_b200 import ops
    M, D = F_ * fs, 1536
    g = torch.Generator(device="cuda").manual_seed(2)
    x, dn, y = (torch.randn(M, D, device="cuda", generator=g).bfloat16() for _ in range(3))
    gin = torch.randn(M, D, device="cuda", generator=g).bfloat16()
    e = torch.randn(F_, 6, D, device="cuda", generator=g).bfloat16().float()
    it = max(20, args.iters)
    t_ln = timed(lambda: ops.layernorm_modulate_grouped_bwd(x, dn, e[:, 1], fs, gin=gin), it, warmup=3)
    t_rg = timed(lambda: ops.resid_gate_grouped_bwd(dn, y, e[:, 2], fs), it, warmup=3)
    ln_bytes = 2 * M * D * 4 + 2 * F_ * D * 4 * 2  # x, dn, gin read, dx written (bf16); d_scale / d_shift
    rg_bytes = 2 * M * D * 3 + F_ * D * 4 + 2 * D
    for name, t, nbytes in (("layernorm_modulate_grouped_bwd", t_ln, ln_bytes), ("resid_gate_grouped_bwd", t_rg, rg_bytes)):
        emit(dict(kind="rowops", op=name, M=M, D=D, groups=F_, ms=t, bytes=nbytes, tb_per_s=nbytes / t / 1e9,
                  share_of_hbm=nbytes / t / 1e9 / (HBM_BYTES_PER_S / 1e12)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--layers", type=int, default=30)
    ap.add_argument("--skip-models", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bench_causal_train.py measures on the GPU: no CUDA device")
    os.makedirs("tool_out", exist_ok=True)
    CARD.update(card())
    fs, F_ = (LATENTS[3] // 2) * (LATENTS[4] // 2), LATENTS[2]
    bench_rowops(args, fs, F_)
    bench_attention(args, fs, F_)
    if not args.skip_models:
        bench_models(args)


if __name__ == "__main__":
    main()
