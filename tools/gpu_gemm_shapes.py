"""Time the GEMM shapes of one Wan 14B layer at 75 600 tokens (run once per FVB_GEMM_STRIPE_N setting)."""
import json, os, sys
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import ops
S = int(os.environ.get("FVB_S", "75600"))
IT = 5 if S > 20000 else 40
shapes = [("qkvg", 20480, 5120, 0), ("out", 5120, 5120, 2), ("cross_q", 5120, 5120, 0), ("fc_in", 13824, 5120, 1), ("fc_out", 5120, 13824, 3)]
res = dict(S=S, stripe=os.environ.get("FVB_GEMM_STRIPE_N", "default"), cases=[])
for name, N, K, epi in shapes:
    x = torch.randn(S, K, device="cuda").bfloat16(); w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    b = torch.zeros(N, device="cuda").bfloat16()
    resid = torch.randn(S, N, device="cuda").bfloat16() if epi >= 2 else None
    gate = torch.randn(N, device="cuda") if epi in (2, 3) else None
    for _ in range(2): ops.linear(x, w, b, epi, resid, gate)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(IT): ops.linear(x, w, b, epi, resid, gate)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / IT
    res["cases"].append(dict(name=name, N=N, K=K, ms=ms, tflops=2.0 * S * N * K / ms / 1e9))
    del x, w, resid
print(json.dumps(res))
os.makedirs("tool_out", exist_ok=True)
json.dump(res, open(f"tool_out/gemm_shapes_S{S}_stripe{res['stripe']}.json", "w"), indent=1)
