"""bf16 against INT8 weight-only (W8A16, WanDiTConfig.int8_weights) and W8A8 (int8_weights + int8_activations) linears on one
H100, in one run:
  * the six block GEMM shapes of Wan 14B at S = 75 600 tokens (720p x 81 frames) plus the text-side attn2 K/V projection at
    M = 512: fvb_linear_bf16, fvb_linear_w8_sp, fvb_linear_w8a8_sp on pre-quantised activations ("w8a8 GEMM") and
    fvb_quantize_int8_rows + fvb_linear_w8a8_sp ("w8a8 incl. quant"), alternated, median of the rounds;
  * fvb_quantize_int8_rows alone at those activation shapes, as bytes moved (bf16 in, int8 + scales out) per second;
  * the Wan2.2-T2V-14B 720p x 81f VSA 0.9 transformer step (bench.py's workload) for bf16, int8_weights and W8A8, alternated:
    ms per step, max_memory_allocated of one forward (weights included), and the rel-L2 of each output from the bf16 one.
    The W8A8 model is the int8_weights model with its Int8Weight objects marked for int8 activations: the same weights;
  * one causal rollout call (14B widths, 1560 tokens per frame, 3-frame block, 21-frame window) for the same three
    configurations (the bf16 and int8 models do not fit together with their caches, so the calls are not alternated).
The card's name, power limit and max SM clock are read in the same run. TFLOP/s are stated against the H100 SXM data sheet
(dense, 700 W): 989 bf16, 1979 int8. Writes <out>/bench_w8a8.json.
Usage: python tools/gpu_bench_w8a8.py [--no-step] [--no-causal] [--layers N] [--rounds R] [--out DIR]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time
from ctypes import c_int, c_int64

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_TFLOPS, INT8_TOPS = 989.0, 1979.0
HBM_TBS = 3.35
S = 75600
# (name, M, N, K, epilogue) of WanBlock's linears (wan_dit.block_forward / cross_attention)
SHAPES = [("qkv+gate", S, 20480, 5120, 0), ("to_out", S, 5120, 5120, 2), ("attn2.to_q", S, 5120, 5120, 0),
          ("attn2.to_out", S, 5120, 5120, 4), ("ffn.fc_in", S, 13824, 5120, 1), ("ffn.fc_out", S, 5120, 13824, 3),
          ("attn2.to_kv", 512, 10240, 5120, 0)]
CONFIGS = ("bf16", "int8", "w8a8")


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
    from fastvideo_b200._lib import check, lib, ptr, stream_ptr
    res["gemm"], res["quantize"] = [], []
    for name, M, N, K, epi in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(N + K)
        x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
        b = torch.zeros(N, device="cuda").bfloat16()
        resid = torch.randn(M, N, device="cuda", generator=g).bfloat16() if epi >= 2 else None
        gate = torch.randn(N, device="cuda", generator=g) if epi in (2, 3) else None
        w8 = ops.Int8Weight.quantize(w)
        a8 = ops.Int8Weight(w8.q, w8.scale, int8_activations=True)
        xq, xs = ops.quantize_int8_rows(x)
        out = torch.empty((M, N), dtype=torch.float32 if epi == 2 else torch.bfloat16, device="cuda")

        def gemm_only():  # fvb_linear_w8a8_sp on activations quantised once, outside the timed loop
            check(lib().fvb_linear_w8a8_sp(ptr(xq), c_int64(xq.stride(0)), ops._f32p(xs), ptr(a8.q), c_int64(a8.q.stride(0)),
                                           ops._f32p(a8.scale), ptr(b), ptr(out), c_int64(N), ptr(None), ptr(resid),
                                           c_int64(N if resid is not None else 0), ops._f32p(gate), c_int(0), c_int64(0),
                                           c_int(M), c_int(N), c_int(K), c_int(epi), stream_ptr()))
        fns = {"bf16": lambda: ops.linear(x, w, b, epi, resid, gate, out=out),
               "w8a16": lambda: ops.linear_any(x, w8, b, epi, resid, gate, out=out),
               "w8a8_gemm": gemm_only,
               "w8a8": lambda: ops.linear_any(x, a8, b, epi, resid, gate, out=out)}
        iters = 5 if M == S else 50
        t = {k: [] for k in fns}
        for _ in range(rounds):
            for k, f in fns.items():
                t[k].append(time_ms(f, iters))
        flop = 2.0 * M * N * K
        row = dict(name=name, M=M, N=N, K=K, epilogue=epi, all_ms=t)
        for k in fns:
            row[k + "_ms"] = median(t[k])
            row[k + "_over_bf16_time"] = row[k + "_ms"] / median(t["bf16"])
        row.update(bf16_share_of_989=flop / row["bf16_ms"] / 1e9 / BF16_TFLOPS,
                   w8a8_gemm_share_of_1979=flop / row["w8a8_gemm_ms"] / 1e9 / INT8_TOPS)
        res["gemm"].append(row)
        print(f"[gemm] {name:12s} M={M:5d} N={N:5d} K={K:5d}  bf16 {row['bf16_ms']:7.3f} ms ({row['bf16_share_of_989']:.2f} of 989)"
              f"  w8a16 {row['w8a16_ms']:7.3f}  w8a8 GEMM {row['w8a8_gemm_ms']:7.3f} ({row['w8a8_gemm_share_of_1979']:.2f} of 1979)"
              f"  w8a8 incl. quant {row['w8a8_ms']:7.3f}  ratios {row['w8a16_over_bf16_time']:.3f} / "
              f"{row['w8a8_gemm_over_bf16_time']:.3f} / {row['w8a8_over_bf16_time']:.3f}", flush=True)
        if M == S and K not in [q["K"] for q in res["quantize"]]:
            tq = median([time_ms(lambda: ops.quantize_int8_rows(x), iters) for _ in range(rounds)])
            nbytes = M * K * 2 + M * K + M * 4
            res["quantize"].append(dict(M=M, K=K, ms=tq, bytes=nbytes, tb_per_s=nbytes / tq / 1e9,
                                        share_of_3_35=nbytes / tq / 1e9 / HBM_TBS))
            print(f"[quant] {M} x {K}: {tq:.3f} ms, {nbytes / tq / 1e9:.2f} TB/s ({nbytes / tq / 1e9 / HBM_TBS:.2f} of 3.35)",
                  flush=True)
        del x, w, resid, w8, a8, xq, xs, out
        torch.cuda.empty_cache()


def set_int8_activations(model, on):
    """Mark (or unmark) every Int8Weight of the model's blocks for int8 activations: W8A8 on the int8_weights model's weights."""
    from fastvideo_b200 import ops
    for blk in model.blocks:
        for v in vars(blk).values():
            if isinstance(v, ops.Int8Weight):
                v.int8_activations = on


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
    models, peak = {}, {}
    fwd = lambda k: models["bf16" if k == "bf16" else "int8"].forward(lat, txt, t, vsa_sparsity=sparsity)

    def run(k):
        if k != "bf16":
            set_int8_activations(models["int8"], k == "w8a8")
        return fwd(k)
    # each forward peak is measured with only its own weights resident: the int8 configurations first, then the bf16 model
    # on top of them, whose peak is taken above what was allocated before it was built
    base = torch.cuda.memory_allocated()
    models["int8"] = WanDiT.random(WanDiTConfig(vsa=True, int8_weights=True, **arch), "cuda")  # same seed, same weights
    with torch.no_grad():
        for k in ("int8", "w8a8"):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            run(k)
            torch.cuda.synchronize()
            peak[k] = torch.cuda.max_memory_allocated() - base
    base = torch.cuda.memory_allocated()
    models["bf16"] = WanDiT.random(WanDiTConfig(vsa=True, **arch), "cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        run("bf16")
    torch.cuda.synchronize()
    peak["bf16"] = torch.cuda.max_memory_allocated() - base
    with torch.no_grad():
        times = {k: [] for k in CONFIGS}
        for _ in range(rounds):
            for k in CONFIGS:
                times[k].append(time_ms(lambda: run(k), 1, warmup=0))
        outs = {k: run(k).float() for k in CONFIGS}
        torch.cuda.synchronize()
    ref = outs["bf16"]
    st = dict(workload=DEFAULT_WORKLOAD + (f" (layers={layers})" if layers else ""), rounds=rounds)
    for k in CONFIGS:
        st[k] = dict(ms=sorted(times[k]), median_ms=median(times[k]), forward_peak_bytes=peak[k],
                     weight_bytes=weight_bytes(models["bf16" if k == "bf16" else "int8"]),
                     rel_l2_vs_bf16=float((outs[k] - ref).norm() / ref.norm()), finite=bool(torch.isfinite(outs[k]).all()),
                     over_bf16_time=median(times[k]) / median(times["bf16"]))
        print(f"[step] {k:5s} {st[k]['median_ms']:.0f} ms (x{st[k]['over_bf16_time']:.3f})  peak "
              f"{peak[k] / 2**30:.2f} GiB  weights {st[k]['weight_bytes'] / 2**30:.2f} GiB  rel-L2 vs bf16 "
              f"{st[k]['rel_l2_vs_bf16']:.3e}", flush=True)
    res["step"] = st
    set_int8_activations(models["int8"], False)
    del models, outs, ref
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
    for k in CONFIGS:
        cfg = WanDiTConfig(**{**WAN_14B, "num_layers": layers or 40}, int8_weights=(k != "bf16"),
                           int8_activations=(k == "w8a8"))
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
    for k in ("int8", "w8a8"):
        out[k]["over_bf16_time"] = out[k]["median_ms"] / out["bf16"]["median_ms"]
    out["workload"] = "causal-wan-14b_480x832_block3_kv21" + (f" (layers={layers})" if layers else "")
    res["causal"] = out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-step", action="store_true", help="skip the full-step comparison")
    ap.add_argument("--no-causal", action="store_true", help="skip the causal rollout call")
    ap.add_argument("--layers", type=int, default=0, help="truncate the step / causal models (flagged in the output)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="tool_out", help="directory for bench_w8a8.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bench_w8a8 measures on a GPU; none is visible")
    res = dict(card=card(), torch=torch.__version__,
               peaks=dict(bf16_tflops=BF16_TFLOPS, int8_tops=INT8_TOPS, hbm_tb_per_s=HBM_TBS,
                          source="H100 SXM data sheet, dense, 700 W"))
    print(f"[card] {res['card']}  (name, power limit, max SM clock)", flush=True)
    bench_gemms(res, max(args.rounds, 3))
    if not args.no_step:
        bench_step(res, args.layers, max(args.rounds, 3))
    if not args.no_causal:
        bench_causal(res, args.layers, max(args.rounds, 3))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_w8a8.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
