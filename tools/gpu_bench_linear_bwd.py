"""Backward of the bf16 linear on one H100, in one run: for each shape, the forward fvb_linear_bf16 (ops.linear), the dgrad
(fvb_linear_dgrad_bf16), the wgrad (fvb_linear_wgrad_bf16) and the bias grad (fvb_bias_grad_bf16), each alone, and torch's
bf16 autograd backward of F.linear (dx, dw and db on the same tensors) as the comparison point. Every shape is warmed up
first; the variants are alternated within each round and the median over the rounds is reported.
GEMM rates count 2 M N K FLOPs against the H100 SXM data sheet's 989 TFLOP/s dense BF16; the bias grad counts the bytes it
must move (dy read once, db written) against 3.35 TB/s. Both figures are for a 700 W card: the card's name, power limit and
max SM clock are read in the same run and printed with the numbers.
Usage: python tools/gpu_bench_linear_bwd.py [--rounds R] [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_TFLOPS = 989.0
HBM_TBS = 3.35
# (name, M, N, K): x [M, K], w [N, K], dy [M, N]
SHAPES = [("14B self-attn proj", 75600, 5120, 5120), ("14B ffn.fc_in", 75600, 13824, 5120),
          ("14B ffn.fc_out", 75600, 5120, 13824), ("14B text K/V", 512, 5120, 5120),
          ("1.3B self-attn proj", 32760, 1536, 1536), ("1.3B ffn.fc_in", 32760, 8960, 1536),
          ("1.3B ffn.fc_out", 32760, 1536, 8960), ("14B proj_out", 75600, 64, 5120)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 -- reported, the timing itself does not need it
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_ms(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def median(v):
    return sorted(v)[len(v) // 2]


def bench_shape(name, M, N, K, rounds):
    from fastvideo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(N + K)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g).bfloat16()
    dy = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    xl, wl, bl = (t.clone().requires_grad_(True) for t in (x, w, b))
    y = F.linear(xl, wl, bl)
    variants = {
        "forward": lambda: ops.linear(x, w),
        "dgrad": lambda: ops.linear_bwd(x, w, dy, True, False, False),
        "wgrad": lambda: ops.linear_bwd(x, w, dy, False, True, False),
        "bias_grad": lambda: ops.linear_bwd(x, w, dy, False, False, True),
        "torch_backward": lambda: torch.autograd.grad(y, (xl, wl, bl), dy, retain_graph=True),
    }
    flop = 2.0 * M * N * K
    iters = max(3, min(50, int(2e13 / flop)))
    for fn in variants.values():  # warm-up: module loads, tensor-map setup, torch's algorithm choice
        time_ms(fn, 2)
    times = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            times[k].append(time_ms(fn, iters))
    row = dict(name=name, M=M, N=N, K=K, iters=iters, **{f"{k}_ms": median(v) for k, v in times.items()},
               all_ms={k: sorted(v) for k, v in times.items()})
    for k in ("forward", "dgrad", "wgrad"):
        row[f"{k}_tflops"] = flop / row[f"{k}_ms"] / 1e9
        row[f"{k}_share_of_989"] = row[f"{k}_tflops"] / BF16_TFLOPS
    row["bias_grad_tbs"] = (M * N * 2 + N * 2) / row["bias_grad_ms"] / 1e9
    row["bias_grad_share_of_3.35"] = row["bias_grad_tbs"] / HBM_TBS
    row["ours_backward_ms"] = row["dgrad_ms"] + row["wgrad_ms"] + row["bias_grad_ms"]
    row["ours_over_torch_backward"] = row["ours_backward_ms"] / row["torch_backward_ms"]
    row["dgrad_rate_over_forward"] = row["dgrad_tflops"] / row["forward_tflops"]
    row["wgrad_rate_over_forward"] = row["wgrad_tflops"] / row["forward_tflops"]
    print(f"[{name}] M={M} N={N} K={K}: fwd {row['forward_ms']:.3f} ms ({row['forward_tflops']:.0f} TF/s)  dgrad "
          f"{row['dgrad_ms']:.3f} ms ({row['dgrad_tflops']:.0f})  wgrad {row['wgrad_ms']:.3f} ms ({row['wgrad_tflops']:.0f})  "
          f"db {row['bias_grad_ms']:.3f} ms ({row['bias_grad_tbs']:.2f} TB/s)  ours dx+dw+db {row['ours_backward_ms']:.3f} ms  "
          f"torch backward {row['torch_backward_ms']:.3f} ms", flush=True)
    del x, w, b, dy, xl, wl, bl, y
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=os.path.join("tool_out", "bench_linear_bwd.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bench_linear_bwd measures on a GPU; none is visible")
    res = dict(card=card(), torch=torch.__version__,
               peaks=dict(bf16_tflops=BF16_TFLOPS, hbm_tbs=HBM_TBS, source="H100 SXM data sheet, dense, 700 W"))
    print(f"[card] {res['card']}  (name, power limit, max SM clock)", flush=True)
    res["shapes"] = [bench_shape(*s, rounds=args.rounds) for s in SHAPES]
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
