"""Dense attention backward (fvb_attention_bwd) and RMSNorm backward (fvb_rmsnorm_bwd) timings.
  * forward without grad (ops.attention), forward with grad (the autograd Function, which also writes the LSE) and the
    backward alone (ops.attention_bwd on the saved tensors) at three Wan shapes; the backward's rate on the algorithm's
    5 matmuls, 10 * B * H * Sq * Skv * 128 FLOPs (the kernels run 7: the dQ kernel recomputes S and dP), against the H100 SXM
    data-sheet 989 TFLOP/s (bf16 dense, 700 W);
  * an in-run A/B against the mma.sync block-list backward (fvb_attention_blocklist_bwd) on full lists at
    (1, 12, 32 768, 32 768): the two alternate, median of the rounds;
  * the RMSNorm backward at M = 75 600, D = 5120 with a bf16 weight: bytes moved (x, dy read, dx written, once each) per
    second against 3.35 TB/s.
The card's name, power limit and max SM clock are read in the same run. Writes <out>/bench_attn_bwd.json.
Usage: python tools/gpu_bench_attn_bwd.py [--iters N] [--rounds R] [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_TFLOPS, HBM_TBS = 989.0, 3.35
SHAPES = {  # (B, H, Sq, Skv)
    "fastwan_1.3b_480p_self": (1, 12, 32760, 32760),
    "wan_14b_720p_cross": (1, 40, 75600, 512),
    "wan_14b_480p_self": (1, 40, 32760, 32760),
}
AB_SHAPE = (1, 12, 32768, 32768)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 -- reported, the timing itself does not need it
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_ms(fn, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bwd_flops(B, H, Sq, Skv):
    return 10.0 * B * H * Sq * Skv * 128


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="tool_out", help="directory for bench_attn_bwd.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastvideo_b200 import attention, ops

    res = {"card": card(), "shapes": {}}
    g = torch.Generator(device="cuda").manual_seed(0)

    def inputs(B, H, Sq, Skv):
        q, dO = (torch.randn(B, Sq, H, 128, device="cuda", generator=g, dtype=torch.bfloat16) for _ in range(2))
        k, v = (torch.randn(B, Skv, H, 128, device="cuda", generator=g, dtype=torch.bfloat16) for _ in range(2))
        return q, k, v, dO

    for name, (B, H, Sq, Skv) in SHAPES.items():
        q, k, v, dO = inputs(B, H, Sq, Skv)
        scale = 128 ** -0.5
        out, lse = ops.attention(q, k, v, return_lse=True)
        leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
        t_fwd = time_ms(lambda: ops.attention(q, k, v, softmax_scale=scale), args.iters)
        t_fwd_grad = time_ms(lambda: attention._DenseAttnFn.apply(*leaves, scale), args.iters)
        t_bwd = time_ms(lambda: ops.attention_bwd(q, k, v, out, lse, dO), args.iters)
        res["shapes"][name] = {"B_H_Sq_Skv": [B, H, Sq, Skv], "fwd_ms": t_fwd, "fwd_grad_ms": t_fwd_grad, "bwd_ms": t_bwd,
                               "bwd_tflops": bwd_flops(B, H, Sq, Skv) / t_bwd / 1e9,
                               "bwd_frac_989": bwd_flops(B, H, Sq, Skv) / t_bwd / 1e9 / BF16_TFLOPS}
        print(name, res["shapes"][name], flush=True)
        del q, k, v, dO, out, lse, leaves
        torch.cuda.empty_cache()

    # A/B against the mma.sync block-list backward on full lists
    B, H, Sq, Skv = AB_SHAPE
    q, k, v, dO = inputs(B, H, Sq, Skv)
    out, lse = ops.attention(q, k, v, return_lse=True)
    n = Sq // 64
    idx = torch.arange(n, dtype=torch.int32, device="cuda").expand(1, 1, n, n).contiguous()
    num = torch.full((1, 1, n), n, dtype=torch.int32, device="cuda")
    new_ms, old_ms = [], []
    for _ in range(args.rounds):
        new_ms.append(time_ms(lambda: ops.attention_bwd(q, k, v, out, lse, dO), 1, warmup=1))
        old_ms.append(time_ms(lambda: ops.attention_blocklist_bwd(q, k, v, out, lse, dO, idx, num, idx, num), 1, warmup=1))
    tn, to = statistics.median(new_ms), statistics.median(old_ms)
    res["ab"] = {"B_H_Sq_Skv": list(AB_SHAPE), "wgmma_ms": new_ms, "mma_sync_ms": old_ms, "wgmma_median_ms": tn,
                 "mma_sync_median_ms": to, "speedup": to / tn, "wgmma_tflops": bwd_flops(*AB_SHAPE) / tn / 1e9,
                 "mma_sync_tflops": bwd_flops(*AB_SHAPE) / to / 1e9}
    print("ab", res["ab"], flush=True)
    del q, k, v, dO, out, lse
    torch.cuda.empty_cache()

    # RMSNorm backward
    M, D = 75600, 5120
    x = torch.randn(M, D, device="cuda", generator=g, dtype=torch.bfloat16)
    dy = torch.randn(M, D, device="cuda", generator=g, dtype=torch.bfloat16)
    w = (1 + 0.1 * torch.randn(D, device="cuda", generator=g)).bfloat16()
    t = time_ms(lambda: ops.rmsnorm_bwd(x, w, dy, 1e-6), 20)
    nbytes = 3 * M * D * 2
    res["rmsnorm_bwd"] = {"M": M, "D": D, "ms": t, "tb_s": nbytes / t / 1e9, "frac_3.35": nbytes / t / 1e9 / HBM_TBS}
    print("rmsnorm_bwd", res["rmsnorm_bwd"], flush=True)

    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_attn_bwd.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
