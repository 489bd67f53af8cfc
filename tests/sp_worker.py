"""Worker of tests/test_gpu_sp_multi.py (bf16), tests/test_gpu_w8.py (int8) and tests/test_gpu_w8a8.py (w8a8), launched with
torchrun (one rank per GPU) as `sp_worker.py [bf16|int8|w8a8]`, the linear-weight format of the models it builds.

The sequence-parallel forward on N GPUs must equal the single-rank forward BIT FOR BIT, for dense and Video-Sparse attention,
for a token count that does not divide by N (zero-padded shard), and for both exchange implementations (symmetric-memory
push, NCCL all-to-all). The head-sharded causal rollout reduces in another order than one rank, so it is held within bf16
rounding of the single-rank engine; in bf16 also to the parity rule against the reference's golden rollouts, under both
RoPE cache policies. The int8 formats run one (ragged) latent shape and the absolute policy only. Rank 0 writes the verdicts
to the JSON file named by SP_WORKER_OUT."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastvideo_b200 import causal_wan, wan_dit  # noqa: E402
from fastvideo_b200 import distributed as fd  # noqa: E402

FORMATS = {"bf16": {}, "int8": dict(int8_weights=True), "w8a8": dict(int8_weights=True, int8_activations=True)}


def _all_ranks(ok, dev):
    flag = torch.tensor([int(ok)], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item())


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def dense_section(rank, world, dev, fmt):
    g = torch.load(os.path.join(ROOT, "tests", "golden", "wan_model_dense.pt"))
    sd = {k: v.to(dev) for k, v in g["sd"].items()}
    # (T, H, W) latents -> tokens: 5x6x7 = 210 (divides by 2, ragged at 4), 3x5x7 = 105 (ragged at 2 and 4)
    shapes = ((5, 12, 14), (3, 10, 14)) if fmt == "bf16" else ((3, 10, 14),)
    out = []
    for vsa in (False, True):
        cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                                   ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                                   text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], vsa=vsa,
                                   **FORMATS[fmt])
        sd2 = dict(sd)
        if vsa:
            gen = torch.Generator(device=dev).manual_seed(0)
            for i in range(2):
                sd2[f"blocks.{i}.to_gate_compress.weight"] = (torch.randn(cfg.hidden_size, cfg.hidden_size, device=dev, generator=gen) / 16).bfloat16()
                sd2[f"blocks.{i}.to_gate_compress.bias"] = torch.zeros(cfg.hidden_size, device=dev).bfloat16()
        model = wan_dit.WanDiT(cfg, sd2)
        for lat_shape in shapes:
            lat = torch.randn(1, 16, *lat_shape, generator=torch.Generator().manual_seed(1)).bfloat16().to(dev)
            args = (lat, g["text"].to(dev), g["timestep"].to(dev))
            sp = 0.5 if vsa else None
            y1 = model.forward(*args, vsa_sparsity=sp)
            for comm in ("push", "nccl"):
                eng = fd.SPWanDiT(model, rank, world, comm=comm)
                y2 = eng.forward(*args, vsa_sparsity=sp)
                y3 = eng.forward(*args, vsa_sparsity=sp) if fmt == "bf16" else y2  # buffers are reused across forwards
                torch.cuda.synchronize()
                out.append(dict(vsa=vsa, tokens=lat_shape[0] * lat_shape[1] * lat_shape[2] // 4, requested=comm, used=eng.comm,
                                world=world, ok_all_ranks=_all_ranks(torch.equal(y1, y2) and torch.equal(y1, y3), dev),
                                max_abs=float((y1.float() - y2.float()).abs().max())))
                if rank == 0:
                    print(json.dumps(out[-1]), flush=True)
    return out


def causal_section(rank, world, dev, fmt, policy):
    """Head-sharded KV cache rollout (causal_wan.SPCausalWanDiT) vs the single-rank CausalWanDiT and, in bf16, the reference's
    golden rollout (tests/golden/wan_causal_model[_rel].pt): three 2-frame blocks x two denoising passes, window 4 frames,
    1 sink frame."""
    g = torch.load(os.path.join(ROOT, "tests", "golden", "wan_causal_model_rel.pt" if policy == "relativistic" else "wan_causal_model.pt"))
    if g["heads"] % world:
        return [dict(causal=True, skipped=f"{g['heads']} heads not divisible by {world}")]
    sd = {k: v.to(dev) for k, v in g["sd"].items()}
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], text_len=g["text_len"],
                               **FORMATS[fmt])
    ccfg = causal_wan.CausalConfig(local_attn_size=g["window_frames"], sink_size=g["sink_frames"],
                                   num_frames_per_block=g["frames_per_call"], rope_cache_policy=policy)
    model = causal_wan.CausalWanDiT(cfg, sd, ccfg)
    c0 = g["calls"][0]["latents"]
    fs = (c0.shape[3] // 2) * (c0.shape[4] // 2)
    if fs % world:
        return [dict(causal=True, skipped=f"{fs} tokens per frame not divisible by {world}")]
    kv1, xc1 = model.new_caches(fs, dev)
    eng = causal_wan.SPCausalWanDiT(model, rank, world)
    kv2, xc2 = eng.new_caches(fs, c0.shape[2] * fs, dev)
    text = g["text"].to(dev)
    out = []
    for i, c in enumerate(g["calls"]):
        args = (c["latents"].to(dev), text, c["timestep"].to(dev))
        kw = dict(current_start=c["start_frame"] * fs, start_frame=c["start_frame"])
        y1 = model.forward_inference(*args, kv1, xc1, **kw)
        y2 = eng.forward_inference(*args, kv2, xc2, **kw)
        torch.cuda.synchronize()
        r = dict(causal=True, policy=policy, call=i, world=world, rel_vs_single_rank=_rel(y2, y1))
        ok = r["rel_vs_single_rank"] < 6e-3 and bool(torch.isfinite(y2.float()).all())
        if fmt == "bf16":
            r.update(rel_vs_fp32=_rel(y2.cpu(), c["y_fp32"]), ref_bf16_floor=_rel(c["y_ref_bf16"], c["y_fp32"]))
            ok = ok and r["rel_vs_fp32"] <= r["ref_bf16_floor"] + 1e-3
        r["ok_all_ranks"] = _all_ranks(ok, dev)
        out.append(r)
        if rank == 0:
            print(json.dumps(r), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("fmt", nargs="?", default="bf16", choices=sorted(FORMATS))
    fmt = ap.parse_args().fmt
    rank, world, dev = fd.init_from_env()
    if not dist.is_initialized():  # init_from_env creates no group for one rank; the verdicts and SPCausalWanDiT need one
        dist.init_process_group(backend="nccl", rank=rank, world_size=world, device_id=dev)
    results = dense_section(rank, world, dev, fmt)
    for policy in ("absolute", "relativistic") if fmt == "bf16" else ("absolute",):
        results += causal_section(rank, world, dev, fmt, policy)
    if rank == 0 and os.environ.get("SP_WORKER_OUT"):
        json.dump(results, open(os.environ["SP_WORKER_OUT"], "w"), indent=1)
    dist.barrier()
    dist.destroy_process_group()
    if not all(r["ok_all_ranks"] for r in results if "skipped" not in r):
        sys.exit(3)


if __name__ == "__main__":
    main()
