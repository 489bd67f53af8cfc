"""Causal (self-forcing) Wan rollout step on H100 -- BASELINE.json config #4 geometry: Wan 14B widths, 480x832 latents
(60x104 -> 30x52 = 1560 tokens per latent frame), 3-frame blocks (4680 query tokens) against a 21-frame KV window
(32 760 keys), random-init weights, synthetic latents. One "step" = one CausalWanDiT.forward_inference call (all 40
layers) for one frame block at one denoising timestep. Reports ms/step at (a) the full window with in-place overwrite
(second and later denoising passes over the same block) and (b) advancing blocks with eviction (ring cache: no copies),
tokens/s, and TFLOP/s against the 2.42e14 FLOP/(block x step) model of SURVEY.md section 8d."""
import json, sys
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import causal_wan, ops
from fastvideo_b200.wan_dit import WanDiTConfig, WAN_14B


def timed(fn, warm, iters):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    evs = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in evs)


def main():
    layers = int(sys.argv[1]) if len(sys.argv) > 1 else 40
    cfg = WanDiTConfig(**{**WAN_14B, "num_layers": layers})
    ccfg = causal_wan.CausalConfig(local_attn_size=21, sink_size=0, num_frames_per_block=3)
    model = causal_wan.CausalWanDiT.random(cfg, ccfg)
    F_, Hl, Wl = 3, 60, 104
    fs = (Hl // 2) * (Wl // 2)
    kv, xc = model.new_caches(fs, "cuda")
    g = torch.Generator(device="cuda").manual_seed(1024)
    text = torch.randn(1, 512, 4096, device="cuda", generator=g).bfloat16()
    lat = torch.randn(1, 16, F_, Hl, Wl, device="cuda", generator=g).bfloat16()
    t = torch.tensor([[500, 500, 500]], device="cuda")
    state = {"block": 0}

    def step_same():
        b = state["block"]
        return model.forward_inference(lat, text, t, kv, xc, current_start=b * F_ * fs, start_frame=b * F_)

    def step_advance():
        state["block"] += 1
        return step_same()

    for b in range(7):  # fill the 21-frame window
        state["block"] = b
        y = step_same()
    torch.cuda.synchronize()
    assert kv[0].local_end_index == 21 * fs and bool(torch.isfinite(y).all())
    n0 = ops.launch_count() if hasattr(ops, "launch_count") else None
    ms_same = timed(step_same, 3, 5)
    ms_adv = timed(step_advance, 3, 5)
    assert kv[0].head != 0
    flop = 2.42e14 * layers / 40
    med = lambda v: v[len(v) // 2]
    res = dict(workload="causal-wan-14b_480x832_block3_kv21", layers=layers, q_tokens=F_ * fs, kv_tokens=21 * fs,
               ms_per_step_full_window=med(ms_same), ms_per_step_advancing_with_eviction=med(ms_adv),
               all_ms_full_window=ms_same, all_ms_advancing=ms_adv,
               tokens_per_s=F_ * fs / med(ms_same) * 1e3, tflops_model=flop / med(ms_same) / 1e9,
               frac_of_sustained_bf16_peak=flop / med(ms_same) / 1e9 / 1447.0,
               peak_mem_gib=torch.cuda.max_memory_allocated() / 2 ** 30, finite=True)
    print(json.dumps(res))
    json.dump(res, open("tool_out/causal_bench.json", "w"), indent=1)


if __name__ == "__main__":
    main()
