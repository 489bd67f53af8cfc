"""Row-kernel timing at the Wan 14B 720p shapes (75 600 x 5120)."""
import json, os, sys
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import ops
from fastvideo_b200.rope import get_rotary_pos_embed
S, D = 75600, 5120
def timed(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
x = torch.randn(S, D, device="cuda").bfloat16(); x32 = torch.randn(S, D, device="cuda")
sc = torch.randn(D, device="cuda"); sh = torch.randn(D, device="cuda"); w = torch.ones(D, device="cuda"); b = torch.zeros(D, device="cuda")
qkv = torch.randn(S, 4 * D, device="cuda").bfloat16(); nw = torch.ones(D, device="cuda").bfloat16()
cos, sin = get_rotary_pos_embed((21, 45, 80), [44, 42, 42]); cos, sin = cos.cuda(), sin.cuda()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
res = {}
res["ln_bf16_mod"] = timed(lambda: ops.layernorm_modulate(x, sc, sh))
res["ln_bf16_round_mod"] = timed(lambda: ops.layernorm_modulate(x, sc, sh, round_ln=True))
res["ln_f32_affine_hidden"] = timed(lambda: ops.layernorm_modulate(x32, None, None, w, b, want_hidden=True))
res["rmsnorm_rope_qk"] = timed(lambda: ops.rmsnorm_rope_(qkv[:, :D], nw, qkv[:, D:2 * D], nw, cos, sin, head_dim=128))
res["rmsnorm_q_only"] = timed(lambda: ops.rmsnorm_rope_(x, nw, head_dim=128))
gb = {"ln_bf16_mod": 2 * S * D * 2, "ln_bf16_round_mod": 2 * S * D * 2, "ln_f32_affine_hidden": S * D * (4 + 2 + 2), "rmsnorm_rope_qk": 4 * S * D * 2, "rmsnorm_q_only": 2 * S * D * 2}
out = {k: dict(ms=v, tb_s=gb[k] / v / 1e9) for k, v in res.items()}
print(json.dumps(out))
os.makedirs("tool_out", exist_ok=True); json.dump(out, open("tool_out/rowops_time.json", "w"), indent=1)
