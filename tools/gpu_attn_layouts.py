"""Sparse attention time vs memory layout: contiguous BHSD (reference kernels' layout) vs strided slices of the fused
[S, 4*D] QKV buffer (what the engine feeds), 720P geometry, 40 heads, top-k 144, random lists."""
import sys, json
import numpy as np, torch
sys.path.insert(0, ".")
from fastvideo_b200 import ops
from oracle import vsa_index

def timed(fn, iters=5, warm=2):
    for _ in range(warm): fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(iters): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters

latent = (21, 45, 80); H = 40
vbs_np = vsa_index.variable_block_sizes(latent, (4, 4, 4)); nb = vbs_np.size; topk = 144
vbs = torch.from_numpy(vbs_np).cuda()
off = torch.cat([torch.zeros(1, dtype=torch.int32), torch.from_numpy(vbs_np).cumsum(0).to(torch.int32)]).cuda()
S = int(vbs_np.sum()); S_pad = nb * 64
torch.manual_seed(0)
scores = torch.randn(1, H, nb, nb, device="cuda")
keep = torch.zeros_like(scores, dtype=torch.bool); keep.scatter_(-1, scores.topk(topk, dim=-1).indices, True)
idx, num = ops.map_to_index(keep); sched, cnt = ops.pair_schedule(keep)
res = {}
# (a) contiguous BHSD padded
q, k, v = (torch.randn(1, H, S_pad, 128, device="cuda", dtype=torch.bfloat16) for _ in range(3))
o = torch.empty_like(q)
res["bhsd_padded_ws"] = timed(lambda: ops.attention_blocklist(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), idx, num, out=o.transpose(1, 2), kv_len=vbs))
res["bhsd_padded_union"] = timed(lambda: ops.attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), out=o.transpose(1, 2), sched=sched, sched_cnt=cnt, kv_len=vbs, nqb=nb, nkb=nb))
del q, k, v, o
# (b) fused token-major buffer [S, 4D], compact tile-major rows
D = H * 128
qkvg = torch.randn(S, 4 * D, device="cuda", dtype=torch.bfloat16)
qv, kv_, vv = (qkvg[:, i * D:(i + 1) * D].unflatten(1, (H, 128)).unsqueeze(0) for i in range(3))
o2 = torch.empty(1, S, H, 128, device="cuda", dtype=torch.bfloat16)
res["fused_compact_ws"] = timed(lambda: ops.attention_blocklist(qv, kv_, vv, idx, num, out=o2, q_off=off, kv_off=off, q_len=vbs, kv_len=vbs, nkb=nb))
res["fused_compact_union"] = timed(lambda: ops.attention(qv, kv_, vv, out=o2, sched=sched, sched_cnt=cnt, q_off=off, kv_off=off, q_len=vbs, kv_len=vbs, nqb=nb, nkb=nb))
# (c) separate token-major [S, D] tensors (BSHD contiguous per tensor)
q3, k3, v3 = (torch.randn(1, S, H, 128, device="cuda", dtype=torch.bfloat16) for _ in range(3))
res["bshd_compact_ws"] = timed(lambda: ops.attention_blocklist(q3, k3, v3, idx, num, out=o2, q_off=off, kv_off=off, q_len=vbs, kv_len=vbs, nkb=nb))
print(json.dumps(res))
json.dump(res, open("tool_out/attn_layouts.json", "w"), indent=1)
