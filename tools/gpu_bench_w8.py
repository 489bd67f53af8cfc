"""bf16 weights against INT8 weight-only linears (WanDiTConfig.int8_weights) on one H100, in one run:
  * the six block GEMM shapes of Wan 14B at S = 75 600 tokens (720p x 81 frames) plus the text-side attn2 K/V projection
    at M = 512, fvb_linear_bf16 against fvb_linear_w8_sp (same bf16 activations), alternated, median of the rounds;
  * the full Wan2.2-T2V-14B 720p x 81f VSA 0.9 transformer step (bench.py's workload), bf16 and int8_weights models with
    the same seeded weights, alternated: ms per step, max_memory_allocated of each model's forward, the model's weight
    bytes, and the rel-L2 of the INT8 step output against the bf16 one;
  * one causal rollout call (14B widths, 1560 tokens per frame, 3-frame block, 21-frame window), bf16 then INT8 (the two
    models and their KV caches do not fit on one card together, so these are not alternated): ms per call and peak memory.
TFLOP/s are stated against the H100 SXM data sheet's 989 TFLOP/s dense BF16 (700 W). Writes tool_out/bench_w8.json.
Usage: python tools/gpu_bench_w8.py [--no-step] [--no-causal] [--layers N] [--rounds R]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_TFLOPS = 989.0
S = 75600
# (name, M, N, K, epilogue) of WanBlock's linears (wan_dit.block_forward / cross_attention)
SHAPES = [("qkv+gate", S, 20480, 5120, 0), ("to_out", S, 5120, 5120, 2), ("attn2.to_q", S, 5120, 5120, 0),
          ("attn2.to_out", S, 5120, 5120, 4), ("ffn.fc_in", S, 13824, 5120, 1), ("ffn.fc_out", S, 5120, 13824, 3),
          ("attn2.to_kv", 512, 10240, 5120, 0)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 -- reported, the timing itself does not need it
        q = f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"
    return q


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


def median(v):
    return sorted(v)[len(v) // 2]


def bench_gemms(res, rounds):
    from fastvideo_b200 import ops
    res["gemm"] = []
    for name, M, N, K, epi in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(N + K)
        x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
        b = torch.zeros(N, device="cuda").bfloat16()
        resid = torch.randn(M, N, device="cuda", generator=g).bfloat16() if epi >= 2 else None
        gate = torch.randn(N, device="cuda", generator=g) if epi in (2, 3) else None
        w8 = ops.Int8Weight.quantize(w)
        out = torch.empty((M, N), dtype=torch.float32 if epi == 2 else torch.bfloat16, device="cuda")
        iters = 5 if M == S else 50
        t_bf, t_w8 = [], []
        for _ in range(rounds):
            t_bf.append(time_ms(lambda: ops.linear(x, w, b, epi, resid, gate, out=out), iters))
            t_w8.append(time_ms(lambda: ops.linear_any(x, w8, b, epi, resid, gate, out=out), iters))
        flop = 2.0 * M * N * K
        row = dict(name=name, M=M, N=N, K=K, epilogue=epi, bf16_ms=median(t_bf), w8_ms=median(t_w8), bf16_all_ms=t_bf,
                   w8_all_ms=t_w8)
        row.update(bf16_tflops=flop / row["bf16_ms"] / 1e9, w8_tflops=flop / row["w8_ms"] / 1e9)
        row.update(bf16_share_of_989=row["bf16_tflops"] / BF16_TFLOPS, w8_share_of_989=row["w8_tflops"] / BF16_TFLOPS,
                   w8_over_bf16_time=row["w8_ms"] / row["bf16_ms"])
        res["gemm"].append(row)
        print(f"[gemm] {name:12s} M={M:5d} N={N:5d} K={K:5d}  bf16 {row['bf16_ms']:8.3f} ms ({row['bf16_tflops']:5.0f} TF/s, "
              f"{row['bf16_share_of_989']:.2f} of 989)  w8a16 {row['w8_ms']:8.3f} ms ({row['w8_tflops']:5.0f} TF/s, "
              f"{row['w8_share_of_989']:.2f} of 989)  time ratio {row['w8_over_bf16_time']:.3f}", flush=True)
        del x, w, resid, w8, out
        torch.cuda.empty_cache()


def weight_bytes(model):
    from fastvideo_b200 import ops
    total = 0
    for obj in [model] + list(model.blocks):
        for v in vars(obj).values():
            if isinstance(v, ops.Int8Weight):
                total += v.nbytes
            elif torch.is_tensor(v):
                total += v.numel() * v.element_size()
    return total


def bench_step(res, layers, rounds):
    from fastvideo_b200.wan_dit import WanDiT, WanDiTConfig
    sys.argv = sys.argv[:1]
    from bench import WORKLOADS, DEFAULT_WORKLOAD
    arch, latent, text_len, sparsity = WORKLOADS[DEFAULT_WORKLOAD]
    arch = dict(arch)
    if layers:
        arch["num_layers"] = layers
    g = torch.Generator().manual_seed(1024)
    C, T, Hh, Ww = latent
    lat = torch.randn(1, C, T, Hh, Ww, generator=g).bfloat16().cuda()
    txt = torch.randn(1, text_len, 4096, generator=g).bfloat16().cuda()
    t = torch.full((1,), 500.0, device="cuda")
    models, peak, wbytes = {}, {}, {}
    # each model's forward peak is measured with only its own weights resident (int8 first, then the bf16 model on top
    # of it, whose peak is taken above what was allocated before it was built)
    for k in ("int8", "bf16"):
        base = torch.cuda.memory_allocated()
        t0 = time.time()
        models[k] = WanDiT.random(WanDiTConfig(vsa=True, int8_weights=(k == "int8"), **arch), "cuda")  # same seed, same weights
        wbytes[k] = weight_bytes(models[k])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            models[k].forward(lat, txt, t, vsa_sparsity=sparsity)
        torch.cuda.synchronize()
        peak[k] = torch.cuda.max_memory_allocated() - base
        print(f"[step] {k} model built in {time.time() - t0:.0f} s: weights {wbytes[k] / 2**30:.2f} GiB, forward peak "
              f"{peak[k] / 2**30:.2f} GiB", flush=True)
    with torch.no_grad():
        fwd = {k: (lambda m=m: m.forward(lat, txt, t, vsa_sparsity=sparsity)) for k, m in models.items()}
        times = {"bf16": [], "int8": []}
        for _ in range(rounds):
            for k in ("bf16", "int8"):
                times[k].append(time_ms(fwd[k], 1, warmup=0))
        outs = {k: f() for k, f in fwd.items()}
        torch.cuda.synchronize()
    a, b = outs["int8"].float(), outs["bf16"].float()
    rel = float((a - b).norm() / b.norm())
    st = dict(workload=DEFAULT_WORKLOAD + (f" (layers={layers})" if layers else ""), rounds=rounds,
              bf16_ms=sorted(times["bf16"]), int8_ms=sorted(times["int8"]), bf16_median_ms=median(times["bf16"]),
              int8_median_ms=median(times["int8"]), bf16_weight_bytes=wbytes["bf16"], int8_weight_bytes=wbytes["int8"],
              bf16_forward_peak_bytes=peak["bf16"], int8_forward_peak_bytes=peak["int8"], rel_l2_int8_vs_bf16=rel,
              finite=bool(torch.isfinite(a).all()))
    st["int8_over_bf16_time"] = st["int8_median_ms"] / st["bf16_median_ms"]
    res["step"] = st
    print(f"[step] bf16 {st['bf16_median_ms']:.0f} ms  int8 weights {st['int8_median_ms']:.0f} ms (median of {rounds}, "
          f"alternated; ratio {st['int8_over_bf16_time']:.3f})  weights {wbytes['bf16'] / 2**30:.2f} -> "
          f"{wbytes['int8'] / 2**30:.2f} GiB  forward peak {peak['bf16'] / 2**30:.2f} -> {peak['int8'] / 2**30:.2f} GiB  "
          f"rel-L2(int8 out, bf16 out) {rel:.3e}", flush=True)
    del models, fwd, outs, a, b
    gc.collect()
    torch.cuda.empty_cache()


def bench_causal(res, layers, iters):
    from fastvideo_b200 import causal_wan
    from fastvideo_b200.wan_dit import WanDiTConfig, WAN_14B
    F_, Hl, Wl = 3, 60, 104
    fs = (Hl // 2) * (Wl // 2)
    g = torch.Generator(device="cuda").manual_seed(1024)
    text = torch.randn(1, 512, 4096, device="cuda", generator=g).bfloat16()
    lat = torch.randn(1, 16, F_, Hl, Wl, device="cuda", generator=g).bfloat16()
    t = torch.tensor([[500, 500, 500]], device="cuda")
    out = {}
    for k in ("bf16", "int8"):
        cfg = WanDiTConfig(**{**WAN_14B, "num_layers": layers or 40}, int8_weights=(k == "int8"))
        ccfg = causal_wan.CausalConfig(local_attn_size=21, sink_size=0, num_frames_per_block=3)
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        model = causal_wan.CausalWanDiT.random(cfg, ccfg)
        kv, xc = model.new_caches(fs, "cuda")
        with torch.no_grad():
            for b in range(7):  # fill the 21-frame window; timed calls re-run the last block (full window)
                y = model.forward_inference(lat, text, t, kv, xc, current_start=b * F_ * fs, start_frame=b * F_)
            ms = [time_ms(lambda: model.forward_inference(lat, text, t, kv, xc, current_start=6 * F_ * fs, start_frame=6 * F_),
                          1, warmup=0) for _ in range(iters)]
        torch.cuda.synchronize()
        out[k] = dict(ms=sorted(ms), median_ms=median(ms), peak_bytes=torch.cuda.max_memory_allocated() - base,
                      weight_bytes=weight_bytes(model), finite=bool(torch.isfinite(y).all()))
        print(f"[causal] {k}: {out[k]['median_ms']:.0f} ms per call (median of {iters})  peak {out[k]['peak_bytes'] / 2**30:.2f} GiB"
              f"  weights {out[k]['weight_bytes'] / 2**30:.2f} GiB", flush=True)
        del model, kv, xc, y
        gc.collect()
        torch.cuda.empty_cache()
    out["int8_over_bf16_time"] = out["int8"]["median_ms"] / out["bf16"]["median_ms"]
    out["workload"] = "causal-wan-14b_480x832_block3_kv21" + (f" (layers={layers})" if layers else "")
    res["causal"] = out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-step", action="store_true", help="skip the full-step comparison")
    ap.add_argument("--no-causal", action="store_true", help="skip the causal rollout call")
    ap.add_argument("--layers", type=int, default=0, help="truncate the step / causal models (flagged in the output)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bench_w8 measures on a GPU; none is visible")
    res = dict(card=card(), torch=torch.__version__,
               peaks=dict(bf16_tflops=BF16_TFLOPS, source="H100 SXM data sheet, dense, 700 W"))
    print(f"[card] {res['card']}  (name, power limit, max SM clock)", flush=True)
    bench_gemms(res, max(args.rounds, 3))
    if not args.no_step:
        bench_step(res, args.layers, max(args.rounds, 3))
    if not args.no_causal:
        bench_causal(res, args.layers, max(args.rounds, 3))
    os.makedirs("tool_out", exist_ok=True)
    with open(os.path.join("tool_out", "bench_w8.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
