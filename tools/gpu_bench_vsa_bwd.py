"""Forward and backward of video_sparse_attn (reference signature, padded layout) at the Wan 14B 720p x 81f attention shape:
the 21 x 45 x 80 latent grid in 4 x 4 x 4 tiles (1440 tiles, S_pad = 92 160), 40 heads of 128, top-k 144 (VSA sparsity 0.9).
  * forward without grad (video_sparse_attn_bshd), forward with grad (the autograd Function), forward + backward;
  * the backward's stages, each timed alone on the saved tensors of one forward, with the calls the backward makes:
    sparse (inverse lists + fvb_attention_blocklist_bwd), compression (four fvb_gemm_batched_bf16 + fvb_softmax_rows_bwd),
    combine (fvb_vsa_combine_bwd), block means (three fvb_block_mean_bwd);
  * the sparse backward's rate on the model 2.5 x forward FLOPs, forward = 4 * 64 * 64 * 128 per selected (q block, kv
    block) pair, against the H100 SXM data-sheet 989 TFLOP/s (bf16 dense, 700 W);
  * the row kernels' bytes moved (each tensor read or written once) per second, against 3.35 TB/s;
  * the compact layout (tile-major, no pad rows, S = 75 600) through VideoSparseAttentionImpl.forward: forward without
    grad, forward with grad, forward + backward, and its sparse stage alone (inverse lists + fvb_attention_sparse_bwd);
  * on the padded layout's lists, fvb_attention_sparse_bwd (wgmma) and fvb_attention_blocklist_bwd (mma.sync) alternating
    in one run, each with its rate on the same FLOP model.
The card's name, power limit and max SM clock are read in the same run. Writes <out>/bench_vsa_bwd.json.
Usage: python tools/gpu_bench_vsa_bwd.py [--iters N] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BF16_TFLOPS, HBM_TBS = 989.0, 3.35
GRID, TILE, HEADS, TOPK = (21, 45, 80), (4, 4, 4), 40, 144


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 -- reported, the timing itself does not need it
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default="tool_out", help="directory for bench_vsa_bwd.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from fastvideo_b200 import ops, vsa

    res = {"card": card(), "grid": GRID, "heads": HEADS, "topk": TOPK}
    vbs = ops.vsa_tile_index(GRID, TILE)["variable_block_sizes"]
    nblk = vbs.numel()
    S, d, B, H = 64 * nblk, 128, 1, HEADS
    res.update(nblk=nblk, S_pad=S)
    valid = (torch.arange(64, device="cuda")[None, :] < vbs[:, None]).reshape(-1)
    g = torch.Generator(device="cuda").manual_seed(0)
    m = valid[None, None, :, None]
    q, k, v, gate, dO = ((torch.randn(B, H, S, d, device="cuda", generator=g) * m).bfloat16() for _ in range(5))
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v, gate)]

    def fwd_nograd():
        with torch.no_grad():
            return vsa.video_sparse_attn(q, k, v, vbs, vbs, TOPK, compress_attn_weight=gate)

    def fwd_grad():
        return vsa.video_sparse_attn(*leaves[:3], vbs, vbs, TOPK, compress_attn_weight=leaves[3])

    def fwd_bwd():
        for t in leaves:
            t.grad = None
        fwd_grad().backward(dO)

    out_ng = fwd_nograd()
    out_g = fwd_grad()
    res["forward_bit_identical_with_grad"] = bool(torch.equal(out_ng, out_g.detach()))
    res["forward_ms"] = time_ms(fwd_nograd, args.iters)
    res["forward_with_grad_ms"] = time_ms(lambda: fwd_grad(), args.iters)
    res["forward_backward_ms"] = time_ms(fwd_bwd, args.iters)
    res["peak_memory_gib_forward_backward"] = torch.cuda.max_memory_allocated() / 2 ** 30

    # the backward's stages on one forward's saved tensors (the calls of _VideoSparseAttnFn.backward)
    (q_, k_, v_, gate_, vbs_, q_ct, k_ct, v_c, attn, out_c, out_s, lse, q2k_idx, q2k_num,
     block_map) = out_g.grad_fn.saved_tensors[:15]
    BH = B * H
    go = dO.contiguous().transpose(1, 2)
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    d_gate = torch.empty_like(gate)
    d_out_c, d_out_c_t = ops.vsa_combine_bwd(go, out_c, gate.transpose(1, 2), vbs, d_gate=d_gate.transpose(1, 2))
    d_attn = ops.gemm_batched(d_out_c.view(BH, nblk, d), v_c.view(BH, nblk, d))
    d_scores, d_scores_t, attn_t = ops.softmax_rows_bwd(attn, d_attn, scale=d ** -0.5, want_transposed=True)
    dq, dk, dv = ops.attention_blocklist_bwd(qt, kt, vt, out_s, lse, go, q2k_idx, q2k_num,
                                             *ops.map_to_index(block_map.transpose(-1, -2).contiguous()), kv_len=vbs)
    d_c = d_out_c.contiguous()

    def sparse():
        k2q_idx, k2q_num = ops.map_to_index(block_map.transpose(-1, -2).contiguous())
        ops.attention_blocklist_bwd(qt, kt, vt, out_s, lse, go, q2k_idx, q2k_num, k2q_idx, k2q_num, kv_len=vbs)

    def compression():
        da = ops.gemm_batched(d_out_c.view(BH, nblk, d), v_c.view(BH, nblk, d))
        ds, ds_t, a_t = ops.softmax_rows_bwd(attn, da, scale=d ** -0.5, want_transposed=True)
        ops.gemm_batched(a_t, d_out_c_t.reshape(BH, d, nblk))
        ops.gemm_batched(ds, k_ct.reshape(BH, d, nblk))
        ops.gemm_batched(ds_t, q_ct.reshape(BH, d, nblk))

    stages = {
        "sparse": sparse,
        "compression": compression,
        "softmax_rows_bwd_alone": lambda: ops.softmax_rows_bwd(attn, d_attn, scale=d ** -0.5, want_transposed=True),
        "combine": lambda: ops.vsa_combine_bwd(go, out_c, gate.transpose(1, 2), vbs, d_gate=d_gate.transpose(1, 2)),
        "block_means": lambda: [ops.block_mean_bwd(x, d_c.view(B, H, nblk, d), vbs, out=x) for x in (dq, dk, dv)],
    }
    res["backward_stage_ms"] = {n: time_ms(fn, args.iters) for n, fn in stages.items()}
    st = res["backward_stage_ms"]

    pairs = int(q2k_num.long().sum())
    fwd_flop = 4.0 * pairs * 64 * 64 * d
    res["sparse_pairs"] = pairs
    res["sparse_bwd_tflops_at_2.5x_fwd"] = 2.5 * fwd_flop / (st["sparse"] * 1e-3) / 1e12
    res["sparse_bwd_share_of_989_tflops"] = res["sparse_bwd_tflops_at_2.5x_fwd"] / BF16_TFLOPS

    tok = B * S * H * d * 2  # one [B, S, H, 128] bf16 tensor
    sq = BH * nblk * nblk * 2  # one [BH, nblk, nblk] bf16 block matrix
    small = BH * nblk * d * 2
    nbytes = {"combine": 3 * tok + 3 * small,  # dO, gate in; d_gate out; out_c in; d_out_c and its transpose out
              "block_means": 3 * (2 * tok + small),  # per tensor: dx_s in, dx out, d_mean in
              "softmax_rows_bwd_alone": 5 * sq}  # p, dp in; ds, ds^T, p^T out
    res["row_kernels"] = {n: {"bytes": b, "ms": st[n], "TB_s": b / (st[n] * 1e-3) / 1e12,
                              "share_of_3.35_TB_s": b / (st[n] * 1e-3) / 1e12 / HBM_TBS} for n, b in nbytes.items()}

    # ---- compact layout, the plug-in's VSA impl
    from types import SimpleNamespace
    from fastvideo_b200.attention import VideoSparseAttentionImpl
    off = torch.zeros(nblk + 1, dtype=torch.int32, device="cuda")
    off[1:] = torch.cumsum(vbs, 0)
    row_block = torch.repeat_interleave(torch.arange(nblk, device="cuda", dtype=torch.int32), vbs.long())
    md = SimpleNamespace(VSA_sparsity=1.0 - (TOPK - 0.5) / nblk, variable_block_sizes=vbs, block_offsets=off,
                         row_block=row_block)
    comp = [t[:, :, valid].transpose(1, 2).contiguous() for t in (q, k, v, gate, dO)]
    res["S_compact"] = comp[0].shape[1]
    cleaves = [t.clone().requires_grad_(True) for t in comp[:4]]
    impl = VideoSparseAttentionImpl(HEADS, d)

    def c_nograd():
        with torch.no_grad():
            return impl.forward(*comp[:4], md)

    def c_grad():
        return impl.forward(*cleaves, md)

    def c_fwd_bwd():
        for t in cleaves:
            t.grad = None
        c_grad().backward(comp[4])

    c_out = c_grad()
    res["compact_forward_bit_identical_with_grad"] = bool(torch.equal(c_nograd(), c_out.detach()))
    res["compact_forward_ms"] = time_ms(c_nograd, args.iters)
    res["compact_forward_with_grad_ms"] = time_ms(c_grad, args.iters)
    res["compact_forward_backward_ms"] = time_ms(c_fwd_bwd, args.iters)
    sv = c_out.grad_fn.saved_tensors
    c_q2k_idx, c_q2k_num, c_map = sv[12], sv[13], sv[14]
    c_go = comp[4]

    def c_sparse():
        k2q_idx, k2q_num = ops.map_to_index(c_map.transpose(-1, -2).contiguous())
        ops.attention_sparse_bwd(*comp[:3], sv[10], sv[11], c_go, c_q2k_idx, c_q2k_num, k2q_idx, k2q_num, q_off=off,
                                 q_len=vbs, kv_off=off, kv_len=vbs)

    res["compact_sparse_stage_ms"] = time_ms(c_sparse, args.iters)
    c_pairs = int(c_q2k_num.long().sum())
    res["compact_sparse_bwd_tflops_at_2.5x_fwd"] = 2.5 * 4.0 * c_pairs * 64 * 64 * d / (res["compact_sparse_stage_ms"] * 1e-3) / 1e12

    # ---- the two sparse backward kernels on the padded layout's lists, alternating
    k2q = ops.map_to_index(block_map.transpose(-1, -2).contiguous())
    kern = {"fvb_attention_sparse_bwd": lambda: ops.attention_sparse_bwd(qt, kt, vt, out_s, lse, go, q2k_idx, q2k_num, *k2q,
                                                                         q_len=vbs, kv_len=vbs),
            "fvb_attention_blocklist_bwd": lambda: ops.attention_blocklist_bwd(qt, kt, vt, out_s, lse, go, q2k_idx, q2k_num,
                                                                               *k2q, kv_len=vbs)}
    ms = {n: [] for n in kern}
    for _ in range(3):
        for n, fn in kern.items():
            ms[n].append(time_ms(fn, args.iters))
    res["padded_lists_kernel_ms"] = {n: min(v) for n, v in ms.items()}
    res["padded_lists_kernel_ms_all"] = ms
    res["padded_lists_kernel_tflops_at_2.5x_fwd"] = {n: 2.5 * fwd_flop / (t * 1e-3) / 1e12
                                                    for n, t in res["padded_lists_kernel_ms"].items()}
    res["sparse_bwd_speedup_over_mma_sync"] = (res["padded_lists_kernel_ms"]["fvb_attention_blocklist_bwd"]
                                               / res["padded_lists_kernel_ms"]["fvb_attention_sparse_bwd"])
    a, b = kern["fvb_attention_sparse_bwd"](), kern["fvb_attention_blocklist_bwd"]()
    m = valid.view(1, -1, 1, 1)
    res["padded_lists_rel_l2_new_vs_mma_sync"] = {n: float(((x.float() - y.float()) * m).norm() / ((y.float() * m).norm() + 1e-30))
                                                   for n, x, y in zip(("dq", "dk", "dv"), a, b)}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_vsa_bwd.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
