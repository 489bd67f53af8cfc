"""bf16 against FP8 linears on one H100, in one run:
  * the six token-stream GEMM shapes of a Wan 14B block at S = 75 600 tokens (720p x 81 frames), bf16 fvb_linear_bf16
    against fvb_linear_fp8 on pre-quantised activations, and the FP8 call including its activation quantisation;
  * the row quantiser (fvb_quantize_fp8_rows) in GB/s;
  * the full Wan2.2-T2V-14B 720p VSA 0.9 transformer step (40 layers, bench.py's workload), bf16 and FP8 models with the
    same seeded weights, timed alternately, and the rel-L2 of the FP8 step output against the bf16 one.
Rates are stated against the H100 SXM data sheet (dense: 989 TFLOP/s BF16, 1979 TFLOP/s FP8; 3.35 TB/s HBM3).
Writes tool_out/bench_fp8.json. Usage: python tools/gpu_bench_fp8.py [--no-step] [--layers N]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_TFLOPS, FP8_TFLOPS, HBM_TBS = 989.0, 1979.0, 3.35
S = 75600
# (name, N, K, epilogue) of WanBlock's token-stream linears (wan_dit.block_forward)
SHAPES = [("qkv+gate", 20480, 5120, 0), ("to_out", 5120, 5120, 2), ("attn2.to_q", 5120, 5120, 0),
          ("attn2.to_out", 5120, 5120, 4), ("ffn.fc_in", 13824, 5120, 1), ("ffn.fc_out", 5120, 13824, 3)]


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


def bench_gemms(res):
    from fastvideo_b200 import ops
    from ctypes import c_float, c_int, c_int64, POINTER, cast
    from fastvideo_b200._lib import check, lib, ptr, stream_ptr
    f32p = lambda t: cast(ptr(t), POINTER(c_float))
    res["gemm"] = []
    for name, N, K, epi in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(N + K)
        x = torch.randn(S, K, device="cuda", generator=g).bfloat16()
        w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
        b = torch.zeros(N, device="cuda").bfloat16()
        resid = torch.randn(S, N, device="cuda", generator=g).bfloat16() if epi >= 2 else None
        gate = torch.randn(N, device="cuda", generator=g) if epi in (2, 3) else None
        wf = ops.Fp8Weight.quantize(w)
        xq, xs = ops.quantize_fp8_rows(x)
        out = torch.empty((S, N), dtype=torch.float32 if epi == 2 else torch.bfloat16, device="cuda")

        def fp8_gemm_only():
            check(lib().fvb_linear_fp8(ptr(xq), c_int64(xq.stride(0)), f32p(xs), ptr(wf.q), c_int64(wf.q.stride(0)),
                                       f32p(wf.scale), ptr(b), ptr(out), c_int64(N), ptr(resid), c_int64(N), f32p(gate), c_int(0),
                                       c_int64(0), c_int(S), c_int(N), c_int(K), c_int(epi), stream_ptr()))

        flop = 2.0 * S * N * K
        row = dict(name=name, M=S, N=N, K=K, epilogue=epi)
        # alternate the three variants over several rounds; keep each one's best round
        t_bf, t_f8, t_f8q = [], [], []
        for _ in range(3):
            t_bf.append(time_ms(lambda: ops.linear(x, w, b, epi, resid, gate, out=out), 5))
            t_f8.append(time_ms(fp8_gemm_only, 5))
            t_f8q.append(time_ms(lambda: ops.linear_fp8(x, wf, b, epi, resid, gate, out=out), 5))
        row.update(bf16_ms=min(t_bf), fp8_gemm_ms=min(t_f8), fp8_with_quant_ms=min(t_f8q))
        row.update(bf16_tflops=flop / row["bf16_ms"] / 1e9, fp8_tflops=flop / row["fp8_gemm_ms"] / 1e9)
        row.update(bf16_share_of_989=row["bf16_tflops"] / BF16_TFLOPS, fp8_share_of_1979=row["fp8_tflops"] / FP8_TFLOPS,
                   fp8_speedup_gemm=row["bf16_ms"] / row["fp8_gemm_ms"], fp8_speedup_with_quant=row["bf16_ms"] / row["fp8_with_quant_ms"])
        res["gemm"].append(row)
        print(f"[gemm] {name:12s} N={N:5d} K={K:5d}  bf16 {row['bf16_ms']:7.3f} ms ({row['bf16_tflops']:5.0f} TF/s, "
              f"{row['bf16_share_of_989']:.2f} of 989)  fp8 {row['fp8_gemm_ms']:7.3f} ms ({row['fp8_tflops']:5.0f} TF/s, "
              f"{row['fp8_share_of_1979']:.2f} of 1979)  fp8+quant {row['fp8_with_quant_ms']:7.3f} ms  "
              f"speed-up {row['fp8_speedup_gemm']:.2f}x / {row['fp8_speedup_with_quant']:.2f}x", flush=True)
        del x, w, resid, wf, xq, out
        torch.cuda.empty_cache()
    # the row quantiser alone: HBM-bound (read 2 B, write 1 B per element, 4 B per row)
    res["quantize"] = []
    for K in (5120, 13824):
        x = torch.randn(S, K, device="cuda").bfloat16()
        ms = time_ms(lambda: ops.quantize_fp8_rows(x), 20)
        nbytes = S * K * 3 + S * 4
        gbs = nbytes / ms / 1e6
        res["quantize"].append(dict(M=S, K=K, ms=ms, GBps=gbs, share_of_3350=gbs / (HBM_TBS * 1e3)))
        print(f"[quant] M={S} K={K:5d}  {ms:.3f} ms  {gbs:6.0f} GB/s ({gbs / (HBM_TBS * 1e3):.2f} of 3.35 TB/s)", flush=True)
        del x


def bench_step(res, layers, rounds):
    from fastvideo_b200.wan_dit import WanDiT, WanDiTConfig
    sys.argv = sys.argv[:1]
    from bench import WORKLOADS, DEFAULT_WORKLOAD
    arch, latent, text_len, sparsity = WORKLOADS[DEFAULT_WORKLOAD]
    arch = dict(arch)
    if layers:
        arch["num_layers"] = layers
    t0 = time.time()
    m_bf = WanDiT.random(WanDiTConfig(vsa=True, **arch), "cuda")
    m_f8 = WanDiT.random(WanDiTConfig(vsa=True, fp8_linears=True, **arch), "cuda")  # same seed: same weights, quantised
    torch.cuda.synchronize()
    print(f"[step] models built in {time.time() - t0:.0f} s, {torch.cuda.memory_allocated() / 2**30:.1f} GiB allocated", flush=True)
    g = torch.Generator().manual_seed(1024)
    C, T, Hh, Ww = latent
    lat = torch.randn(1, C, T, Hh, Ww, generator=g).bfloat16().cuda()
    txt = torch.randn(1, text_len, 4096, generator=g).bfloat16().cuda()
    t = torch.full((1,), 500.0, device="cuda")
    S_tok = T * (Hh // 2) * (Ww // 2)
    with torch.no_grad():
        fwd = {"bf16": lambda: m_bf.forward(lat, txt, t, vsa_sparsity=sparsity),
               "fp8": lambda: m_f8.forward(lat, txt, t, vsa_sparsity=sparsity)}
        outs = {k: f() for k, f in fwd.items()}  # warm-up (layouts, first launches)
        times = {"bf16": [], "fp8": []}
        for _ in range(rounds):
            for k in ("bf16", "fp8"):
                times[k].append(time_ms(fwd[k], 1, warmup=0))
        outs = {k: f() for k, f in fwd.items()}
        torch.cuda.synchronize()
    a, b = outs["fp8"].float(), outs["bf16"].float()
    rel = float((a - b).norm() / b.norm())
    st = dict(workload=DEFAULT_WORKLOAD + (f" (layers={layers})" if layers else ""), tokens=S_tok, rounds=rounds,
              bf16_ms=sorted(times["bf16"]), fp8_ms=sorted(times["fp8"]),
              bf16_median_ms=sorted(times["bf16"])[rounds // 2], fp8_median_ms=sorted(times["fp8"])[rounds // 2],
              rel_l2_fp8_vs_bf16=rel, finite=bool(torch.isfinite(a).all()))
    st["speedup"] = st["bf16_median_ms"] / st["fp8_median_ms"]
    st["bf16_tokens_per_s"] = S_tok / st["bf16_median_ms"] * 1e3
    st["fp8_tokens_per_s"] = S_tok / st["fp8_median_ms"] * 1e3
    res["step"] = st
    print(f"[step] bf16 {st['bf16_median_ms']:.0f} ms  fp8 {st['fp8_median_ms']:.0f} ms  (median of {rounds}, alternated)  "
          f"speed-up {st['speedup']:.3f}x  latent tokens/s {st['bf16_tokens_per_s']:.0f} -> {st['fp8_tokens_per_s']:.0f}  "
          f"rel-L2(fp8 out, bf16 out) {rel:.3e}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-step", action="store_true", help="GEMM shapes and the quantiser only")
    ap.add_argument("--layers", type=int, default=0, help="truncate the model of the step comparison (flagged)")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bench_fp8 measures on a GPU; none is visible")
    res = dict(card=card(), torch=torch.__version__,
               peaks=dict(bf16_tflops=BF16_TFLOPS, fp8_tflops=FP8_TFLOPS, hbm_tbs=HBM_TBS,
                          source="H100 SXM data sheet, dense, 700 W"))
    print(f"[card] {res['card']}  (name, power limit, max SM clock)", flush=True)
    bench_gemms(res)
    if not args.no_step:
        bench_step(res, args.layers, args.rounds)
    os.makedirs("tool_out", exist_ok=True)
    with open(os.path.join("tool_out", "bench_fp8.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
