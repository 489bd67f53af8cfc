"""bf16 against 8-bit attention (INT8 Q K^T, FP8 P V) on one H100, in one run:
  * the quantiser (fvb_attention_8bit_quantize) in GB/s of the bytes it must move (read q, k, v once; write q8, k8, vt8 and
    the scales) against the 3.35 TB/s HBM3 data-sheet rate;
  * the attention kernel, bf16 against 8-bit, alternated over rounds, best round kept, without and with the quantiser, at
    - the Wan2.2-14B 720p x 81-frame VSA 0.9 sparse branch: S = 75 600, H = 40, per-q-block lists from the engine's top-k
      of the block-mean scores (fvb_attention_blocklist_fwd against fvb_attention_8bit_fwd with lists);
    - a dense FastWan-1.3B 480p x 81-frame self-attention: S = 32 760, H = 12 (fvb_attention_fwd against the dense 8-bit);
  * the full Wan2.2-T2V-14B 720p VSA 0.9 transformer step (bench.py's workload) for bf16, attention_8bit and
    attention_8bit + fp8_linears (same seeded weights), median of alternated runs, and the rel-L2 of each step output
    against the bf16 one.
Writes tool_out/bench_attn_8bit.json. Usage: python tools/gpu_bench_attn_8bit.py [--no-step] [--layers N] [--rounds R]"""
import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gpu_bench_fp8 import card, time_ms  # noqa: E402

HBM_TBS = 3.35


def _qkv(S, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    buf = torch.randn(1, S, 3, H, 128, device="cuda", generator=g)
    buf[:, :, 1] += torch.randn(H, 128, device="cuda", generator=g)  # a channel bias on K, as RMSNorm'd keys have
    qkv = buf.bfloat16()
    del buf
    return qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]


def _alternate(fns, rounds, iters):
    best = {k: float("inf") for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            best[k] = min(best[k], time_ms(f, iters))
    return best


def bench_quantiser(res, rounds):
    from fastvideo_b200 import ops
    res["quantize"] = []
    for name, S, H in (("14B 720p", 75600, 40), ("1.3B 480p", 32760, 12)):
        q, k, v = _qkv(S, H, S + H)
        ms = _alternate({"q": lambda: ops.quantize_attention_8bit(q, k, v)}, rounds, 10)["q"]
        nbytes = S * H * 128 * (3 * 2 + 3) + S * H * 4 * 2 + H * 128 * 4 * 2
        gbs = nbytes / ms / 1e6
        res["quantize"].append(dict(shape=name, S=S, H=H, ms=ms, GBps=gbs, share_of_3350=gbs / (HBM_TBS * 1e3)))
        print(f"[quant] {name} S={S} H={H}  {ms:.3f} ms  {gbs:6.0f} GB/s ({gbs / (HBM_TBS * 1e3):.2f} of 3.35 TB/s)", flush=True)
        del q, k, v
        torch.cuda.empty_cache()


def bench_vsa_attention(res, rounds):
    from fastvideo_b200 import ops
    seq = (21, 45, 80)
    S, H = math.prod(seq), 40
    t = ops.vsa_tile_index(seq, (4, 4, 4))
    vbs, off = t["variable_block_sizes"], t["block_offsets"]
    nblk = vbs.numel()
    topk = max(1, min(math.ceil(0.1 * nblk), nblk))
    q, k, v = _qkv(S, H, 7)
    q_c, k_c = ops.block_mean(q, nblk, off, vbs), ops.block_mean(k, nblk, off, vbs)
    scores = ops.gemm_batched(q_c.view(H, nblk, 128), k_c.view(H, nblk, 128), div=math.sqrt(128))
    idx, num, _ = ops.topk_index(scores, topk)
    idx, num = idx.view(1, H, nblk, nblk), num.view(1, H, nblk)
    qin = ops.quantize_attention_8bit(q, k, v, kv_off=off, kv_len=vbs, nkb=nblk)
    fns = {
        "bf16": lambda: ops.attention_blocklist(q, k, v, idx, num, softmax_scale=128 ** -0.5, q_off=off, kv_off=off, q_len=vbs,
                                                kv_len=vbs, nkb=nblk),
        "int8_fp8": lambda: ops.attention_8bit(qin, 128 ** -0.5, idx, num, q_off=off, q_len=vbs),
        "int8_fp8_with_quant": lambda: ops.attention_8bit(ops.quantize_attention_8bit(q, k, v, kv_off=off, kv_len=vbs, nkb=nblk),
                                                          128 ** -0.5, idx, num, q_off=off, q_len=vbs),
    }
    best = _alternate(fns, rounds, 5)
    o16, o8 = fns["bf16"](), fns["int8_fp8"]()
    pairs = int(num.sum()) * 64 * 64  # upper bound of (q, k) pairs: every selected block full
    flop = 4.0 * pairs * 128
    row = dict(shape="14B 720p x 81f VSA 0.9 sparse branch", S=S, H=H, nblk=nblk, topk=topk, **{f"{k}_ms": v for k, v in best.items()},
               bf16_tflops=flop / best["bf16"] / 1e9, int8_fp8_tflops=flop / best["int8_fp8"] / 1e9,
               speedup_kernel=best["bf16"] / best["int8_fp8"], speedup_with_quant=best["bf16"] / best["int8_fp8_with_quant"],
               rel_l2_vs_bf16=float((o8.float() - o16.float()).norm() / o16.float().norm()))
    res["attention"].append(row)
    _print_row(row)
    del q, k, v, qin
    torch.cuda.empty_cache()


def bench_dense_attention(res, rounds):
    from fastvideo_b200 import ops
    S, H = 21 * 30 * 52, 12
    q, k, v = _qkv(S, H, 9)
    qin = ops.quantize_attention_8bit(q, k, v)
    fns = {"bf16": lambda: ops.attention(q, k, v, softmax_scale=128 ** -0.5),
           "int8_fp8": lambda: ops.attention_8bit(qin, 128 ** -0.5),
           "int8_fp8_with_quant": lambda: ops.attention_8bit(ops.quantize_attention_8bit(q, k, v), 128 ** -0.5)}
    best = _alternate(fns, rounds, 3)
    o16, o8 = fns["bf16"](), fns["int8_fp8"]()
    flop = 4.0 * S * S * H * 128
    row = dict(shape="1.3B 480p x 81f dense self-attention", S=S, H=H, **{f"{k}_ms": v for k, v in best.items()},
               bf16_tflops=flop / best["bf16"] / 1e9, int8_fp8_tflops=flop / best["int8_fp8"] / 1e9,
               speedup_kernel=best["bf16"] / best["int8_fp8"], speedup_with_quant=best["bf16"] / best["int8_fp8_with_quant"],
               rel_l2_vs_bf16=float((o8.float() - o16.float()).norm() / o16.float().norm()))
    res["attention"].append(row)
    _print_row(row)


def _print_row(r):
    print(f"[attn] {r['shape']}: bf16 {r['bf16_ms']:.3f} ms ({r['bf16_tflops']:.0f} TF/s)  8-bit {r['int8_fp8_ms']:.3f} ms "
          f"({r['int8_fp8_tflops']:.0f} TF/s)  8-bit+quant {r['int8_fp8_with_quant_ms']:.3f} ms  speed-up "
          f"{r['speedup_kernel']:.2f}x / {r['speedup_with_quant']:.2f}x  rel-L2 vs bf16 {r['rel_l2_vs_bf16']:.3e}", flush=True)


def bench_step(res, layers, rounds):
    from fastvideo_b200.wan_dit import WanDiT, WanDiTConfig
    sys.argv = sys.argv[:1]
    from bench import WORKLOADS, DEFAULT_WORKLOAD
    arch, latent, text_len, sparsity = WORKLOADS[DEFAULT_WORKLOAD]
    arch = dict(arch)
    if layers:
        arch["num_layers"] = layers
    t0 = time.time()
    # attention_8bit is read at every forward, so one model per weight format serves both attention settings
    m_bf = WanDiT.random(WanDiTConfig(vsa=True, **arch), "cuda")
    m_f8 = WanDiT.random(WanDiTConfig(vsa=True, fp8_linears=True, attention_8bit=True, **arch), "cuda")
    torch.cuda.synchronize()
    print(f"[step] models built in {time.time() - t0:.0f} s, {torch.cuda.memory_allocated() / 2**30:.1f} GiB allocated", flush=True)
    g = torch.Generator().manual_seed(1024)
    C, T, Hh, Ww = latent
    lat = torch.randn(1, C, T, Hh, Ww, generator=g).bfloat16().cuda()
    txt = torch.randn(1, text_len, 4096, generator=g).bfloat16().cuda()
    tt = torch.full((1,), 500.0, device="cuda")

    def run(model, attn8):
        def f():
            model.cfg.attention_8bit = attn8
            return model.forward(lat, txt, tt, vsa_sparsity=sparsity)
        return f

    fwd = {"bf16": run(m_bf, False), "attn8": run(m_bf, True), "attn8_fp8": run(m_f8, True)}
    with torch.no_grad():
        for f in fwd.values():
            f()  # warm-up (layouts, first launches)
        times = {k: [] for k in fwd}
        for _ in range(rounds):
            for k, f in fwd.items():
                times[k].append(time_ms(f, 1, warmup=0))
        outs = {k: f().float() for k, f in fwd.items()}
        torch.cuda.synchronize()
    ref = outs["bf16"]
    st = dict(workload=DEFAULT_WORKLOAD + (f" (layers={layers})" if layers else ""), rounds=rounds)
    for k in fwd:
        st[f"{k}_ms"] = sorted(times[k])
        st[f"{k}_median_ms"] = sorted(times[k])[rounds // 2]
        if k != "bf16":
            st[f"{k}_speedup"] = st["bf16_median_ms"] / st[f"{k}_median_ms"]
            st[f"{k}_rel_l2_vs_bf16"] = float((outs[k] - ref).norm() / ref.norm())
            st[f"{k}_finite"] = bool(torch.isfinite(outs[k]).all())
    res["step"] = st
    print(f"[step] bf16 {st['bf16_median_ms']:.0f} ms  attention_8bit {st['attn8_median_ms']:.0f} ms "
          f"({st['attn8_speedup']:.3f}x, rel-L2 {st['attn8_rel_l2_vs_bf16']:.3e})  attention_8bit + fp8_linears "
          f"{st['attn8_fp8_median_ms']:.0f} ms ({st['attn8_fp8_speedup']:.3f}x, rel-L2 {st['attn8_fp8_rel_l2_vs_bf16']:.3e})  "
          f"(median of {rounds}, alternated)", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-step", action="store_true", help="quantiser and attention kernels only")
    ap.add_argument("--layers", type=int, default=0, help="truncate the model of the step comparison (flagged)")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bench_attn_8bit measures on a GPU; none is visible")
    res = dict(card=card(), torch=torch.__version__, attention=[],
               peaks=dict(hbm_tbs=HBM_TBS, source="H100 SXM data sheet, 700 W"))
    print(f"[card] {res['card']}  (name, power limit, max SM clock)", flush=True)
    with torch.no_grad():
        bench_quantiser(res, args.rounds)
        bench_vsa_attention(res, args.rounds)
        bench_dense_attention(res, args.rounds)
    if not args.no_step:
        bench_step(res, args.layers, max(3, args.rounds // 2 * 2 + 1))
    os.makedirs("tool_out", exist_ok=True)
    with open(os.path.join("tool_out", "bench_attn_8bit.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
