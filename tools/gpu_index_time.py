"""Time the VSA block-map stage at the 720p geometry (40 heads x 1440 q tiles x 1440 kv tiles, top-k 144):
topk_mask + map_to_index (two passes) vs topk_index (one pass). FVB_TOPK_WARP=0 forces the block-per-row top-k kernel."""
import json, os, sys
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import ops
torch.manual_seed(0)
s = (torch.randn(1, 40, 1440, 1440, device="cuda") * 0.5).bfloat16()
def timed(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
res = {"topk_warp": os.environ.get("FVB_TOPK_WARP", "1")}
res["topk_mask_ms"] = timed(lambda: ops.topk_mask(s, 144))
m = ops.topk_mask(s, 144)
res["map_to_index_ms"] = timed(lambda: ops.map_to_index(m))
res["topk_index_ms"] = timed(lambda: ops.topk_index(s, 144))
res["bytes_scores_plus_lists"] = s.numel() * 2 + s.numel() * 4
res["topk_index_tb_s"] = res["bytes_scores_plus_lists"] / res["topk_index_ms"] / 1e9
print(json.dumps(res))
os.makedirs("tool_out", exist_ok=True)
json.dump(res, open(f"tool_out/index_time_warp{res['topk_warp']}.json", "w"), indent=1)
