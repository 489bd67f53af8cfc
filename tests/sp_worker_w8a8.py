"""Worker of tests/test_gpu_w8a8.py::test_sp_w8a8_equals_single_rank, launched with torchrun (one rank per GPU): with
WanDiTConfig(int8_weights=True, int8_activations=True), the sequence-parallel forward must equal the single-rank forward bit
for bit (dense and VSA, both exchange implementations), and the head-sharded causal rollout must stay within bf16 rounding
of the single-rank CausalWanDiT. The activations are quantised per token and every reduction is exact, so the
token-sharded forward sees the same rows as one rank. Rank 0 writes the verdicts to the JSON file named by SP_WORKER_OUT."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastvideo_b200 import causal_wan, wan_dit  # noqa: E402
from fastvideo_b200 import distributed as fd  # noqa: E402


def _all_ranks(ok, dev):
    flag = torch.tensor([int(ok)], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item())


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def dense_section(rank, world, dev):
    g = torch.load(os.path.join(ROOT, "tests", "golden", "wan_model_dense.pt"))
    sd = {k: v.to(dev) for k, v in g["sd"].items()}
    out = []
    for vsa in (False, True):
        cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                                   ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                                   text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], vsa=vsa,
                                   int8_weights=True, int8_activations=True)
        sd2 = dict(sd)
        if vsa:
            gen = torch.Generator(device=dev).manual_seed(0)
            for i in range(2):
                sd2[f"blocks.{i}.to_gate_compress.weight"] = (torch.randn(cfg.hidden_size, cfg.hidden_size, device=dev, generator=gen) / 16).bfloat16()
                sd2[f"blocks.{i}.to_gate_compress.bias"] = torch.zeros(cfg.hidden_size, device=dev).bfloat16()
        model = wan_dit.WanDiT(cfg, sd2)
        lat = torch.randn(1, 16, 3, 10, 14, generator=torch.Generator().manual_seed(1)).bfloat16().to(dev)  # 105 tokens: ragged
        args = (lat, g["text"].to(dev), g["timestep"].to(dev))
        sp = 0.5 if vsa else None
        y1 = model.forward(*args, vsa_sparsity=sp)
        for comm in ("push", "nccl"):
            eng = fd.SPWanDiT(model, rank, world, comm=comm)
            y2 = eng.forward(*args, vsa_sparsity=sp)
            torch.cuda.synchronize()
            out.append(dict(vsa=vsa, requested=comm, used=eng.comm, world=world, ok_all_ranks=_all_ranks(torch.equal(y1, y2), dev),
                            max_abs=float((y1.float() - y2.float()).abs().max())))
            if rank == 0:
                print(json.dumps(out[-1]), flush=True)
    return out


def causal_section(rank, world, dev):
    g = torch.load(os.path.join(ROOT, "tests", "golden", "wan_causal_model.pt"))
    if g["heads"] % world:
        return [dict(causal=True, skipped=f"{g['heads']} heads not divisible by {world}")]
    sd = {k: v.to(dev) for k, v in g["sd"].items()}
    cfg = wan_dit.WanDiTConfig(hidden_size=sd["proj_out.weight"].shape[1], num_attention_heads=g["heads"],
                               ffn_dim=sd["blocks.0.ffn.fc_in.weight"].shape[0], num_layers=2,
                               text_dim=sd["condition_embedder.text_embedder.fc_in.weight"].shape[1], text_len=g["text_len"],
                               int8_weights=True, int8_activations=True)
    ccfg = causal_wan.CausalConfig(local_attn_size=g["window_frames"], sink_size=g["sink_frames"],
                                   num_frames_per_block=g["frames_per_call"])
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
        # the head-sharded cache reduces in another order than one rank: bf16 rounding apart, as in tests/sp_worker.py
        ok = _rel(y2, y1) < 6e-3 and bool(torch.isfinite(y2.float()).all())
        out.append(dict(causal=True, call=i, world=world, rel_vs_single_rank=_rel(y2, y1), ok_all_ranks=_all_ranks(ok, dev)))
        if rank == 0:
            print(json.dumps(out[-1]), flush=True)
    return out


def main():
    rank, world, dev = fd.init_from_env()
    results = dense_section(rank, world, dev) + causal_section(rank, world, dev)
    if rank == 0 and os.environ.get("SP_WORKER_OUT"):
        json.dump(results, open(os.environ["SP_WORKER_OUT"], "w"), indent=1)
    dist.barrier()
    dist.destroy_process_group()
    if not all(r["ok_all_ranks"] for r in results if "skipped" not in r):
        sys.exit(3)


if __name__ == "__main__":
    main()
