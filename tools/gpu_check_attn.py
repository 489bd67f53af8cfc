"""GPU check of the attention kernel and the row kernels against fp32 torch."""
import sys, math, json, time
import numpy as np
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import ops
from oracle import vsa_index

dev = "cuda"
LOG2E = 1.4426950408889634

def ref_attn(q, k, v, mask=None, scale=None):
    # q: [B,Sq,H,d]
    B, Sq, H, d = q.shape
    scale = scale or d ** -0.5
    qf, kf, vf = (t.float().transpose(1, 2) for t in (q, k, v))
    s = (qf @ kf.transpose(-1, -2)) * scale
    if mask is not None:
        s = s.masked_fill(~mask, float("-inf"))
    lse = torch.logsumexp(s, dim=-1) * LOG2E
    p = torch.softmax(s, dim=-1)
    p = torch.nan_to_num(p, nan=0.0)
    o = (p @ vf).transpose(1, 2)
    return o, lse

def report(name, got, ref, got_lse=None, ref_lse=None):
    g, r = got.float(), ref.float()
    rel = ((g - r).norm() / r.norm().clamp_min(1e-30)).item()
    mx = (g - r).abs().max().item()
    msg = f"{name}: rel={rel:.3e} maxabs={mx:.3e}"
    if got_lse is not None:
        fin = torch.isfinite(ref_lse)
        ld = (got_lse[fin] - ref_lse[fin]).abs().max().item() if fin.any() else 0.0
        same_inf = bool((torch.isinf(got_lse) == torch.isinf(ref_lse)).all())
        msg += f" lse_maxabs={ld:.3e} inf_match={same_inf}"
    print(msg, flush=True)
    return rel, mx

def dense_case(B, H, Sq, Skv, seed=0, layout="bshd"):
    torch.manual_seed(seed)
    if layout == "bshd":
        q = torch.randn(B, Sq, H, 128, device=dev).bfloat16()
        k = torch.randn(B, Skv, H, 128, device=dev).bfloat16()
        v = torch.randn(B, Skv, H, 128, device=dev).bfloat16()
    else:  # bhsd storage, viewed as bshd
        q = torch.randn(B, H, Sq, 128, device=dev).bfloat16().transpose(1, 2)
        k = torch.randn(B, H, Skv, 128, device=dev).bfloat16().transpose(1, 2)
        v = torch.randn(B, H, Skv, 128, device=dev).bfloat16().transpose(1, 2)
    o, lse = ops.attention(q, k, v, return_lse=True)
    torch.cuda.synchronize()
    ro, rl = ref_attn(q, k, v)
    return report(f"dense B{B} H{H} Sq{Sq} Skv{Skv} {layout}", o, ro, lse, rl)

def block_case(nblk, topk, H, ragged, seed=0, B=1, zero_rows=False):
    torch.manual_seed(seed); rng = np.random.default_rng(seed)
    S = nblk * 64
    q = torch.randn(B, H, S, 128, device=dev).bfloat16().transpose(1, 2)
    k = torch.randn(B, H, S, 128, device=dev).bfloat16().transpose(1, 2)
    v = torch.randn(B, H, S, 128, device=dev).bfloat16().transpose(1, 2)
    bmap = np.zeros((B, H, nblk, nblk), dtype=bool)
    for b in range(B):
        for h in range(H):
            for qb in range(nblk):
                kk = topk if not zero_rows or (qb % 3) else 0
                bmap[b, h, qb, rng.permutation(nblk)[:kk]] = True
    vbs = rng.integers(32, 65, size=nblk).astype(np.int32) if ragged else np.full(nblk, 64, np.int32)
    sched, cnt = vsa_index.pair_union_schedule(bmap)
    sched_t = torch.from_numpy(sched).to(dev); cnt_t = torch.from_numpy(cnt).to(dev)
    vbs_t = torch.from_numpy(vbs).to(dev)
    o, lse = ops.attention(q, k, v, return_lse=True, sched=sched_t, sched_cnt=cnt_t, kv_len=vbs_t, nqb=nblk, nkb=nblk)
    torch.cuda.synchronize()
    keep = torch.from_numpy(bmap).to(dev).repeat_interleave(64, 2).repeat_interleave(64, 3)
    colvalid = torch.from_numpy((np.arange(64)[None, :] < vbs[:, None]).reshape(-1)).to(dev)
    keep = keep & colvalid[None, None, None, :]
    ro, rl = ref_attn(q, k, v, mask=keep)
    r = report(f"block nblk{nblk} topk{topk} H{H} ragged={ragged} zero_rows={zero_rows}", o, ro, lse, rl)
    if zero_rows:
        empty = ~keep.any(-1)  # [B,H,S]
        z = o.transpose(1, 2)[empty]
        print(f"   empty rows exact zero: {bool((z == 0).all())}, lse -inf: {bool(torch.isinf(lse[empty]).all())}", flush=True)
    return r

def elementwise_cases():
    torch.manual_seed(1)
    for (M, D) in [(777, 1536), (1000, 5120)]:
        x = torch.randn(M, D, device=dev).bfloat16() * 2 + 0.3
        scale = torch.randn(D, device=dev) * 0.1; shift = torch.randn(D, device=dev) * 0.1
        w = torch.randn(D, device=dev) * 0.5 + 1; bb = torch.randn(D, device=dev) * 0.1
        F = torch.nn.functional
        # norm1: LN(x.float())*(1+scale)+shift -> bf16
        ref = (F.layer_norm(x.float(), (D,), None, None, 1e-6) * (1 + scale) + shift).bfloat16()
        got = ops.layernorm_modulate(x, scale, shift)
        mm = (got.float() != ref.float()).float().mean().item()
        report(f"ln_mod M{M} D{D} (mismatch {mm:.5f})", got, ref)
        # cross: bf16(LN(x)) * (1+scale) + shift
        ref = (F.layer_norm(x.float(), (D,), None, None, 1e-6).bfloat16() * (1 + scale) + shift).bfloat16()
        got = ops.layernorm_modulate(x, scale, shift, round_ln=True)
        mm = (got.float() != ref.float()).float().mean().item()
        report(f"ln_round_mod M{M} D{D} (mismatch {mm:.5f})", got, ref)
        # self-attn residual norm: fp32 in, affine, hidden out
        r32 = torch.randn(M, D, device=dev) * 3
        ref = F.layer_norm(r32, (D,), w, bb, 1e-6).bfloat16()
        got, hid = ops.layernorm_modulate(r32, None, None, w, bb, want_hidden=True)
        mm = (got.float() != ref.float()).float().mean().item()
        report(f"ln_affine_f32 M{M} D{D} (mismatch {mm:.5f})", got, ref)
        print("   hidden exact:", bool((hid == r32.bfloat16()).all()), flush=True)
        # rmsnorm + rope on q,k inside a fused qkv buffer
        H = D // 128
        qkv = torch.randn(M, 3 * D, device=dev).bfloat16()
        wq = (torch.randn(D, device=dev) * 0.2 + 1).bfloat16(); wk = (torch.randn(D, device=dev) * 0.2 + 1).bfloat16()
        ang = torch.rand(M, 64, device=dev, dtype=torch.float64) * 6.28
        cos = ang.cos().repeat_interleave(2, -1).float().contiguous(); sin = ang.sin().repeat_interleave(2, -1).float().contiguous()
        def ref_rms_rope(x, wgt):
            xf = x.float()
            n = (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)).bfloat16() * wgt
            n = n.view(M, H, 128)
            xr, xi = n.float().reshape(M, H, 64, 2).unbind(-1)
            rot = torch.stack([-xi, xr], -1).flatten(-2)
            return (n.float() * cos[:, None] + rot * sin[:, None]).bfloat16().view(M, D)
        rq = ref_rms_rope(qkv[:, :D], wq); rk = ref_rms_rope(qkv[:, D:2 * D], wk)
        buf = qkv.clone()
        ops.rmsnorm_rope_(buf[:, :D], wq, buf[:, D:2 * D], wk, cos, sin)
        mmq = (buf[:, :D].float() != rq.float()).float().mean().item()
        report(f"rms_rope q M{M} D{D} (mismatch {mmq:.5f})", buf[:, :D], rq)
        report(f"rms_rope k M{M} D{D}", buf[:, D:2 * D], rk)
        print("   v untouched:", bool((buf[:, 2 * D:] == qkv[:, 2 * D:]).all()), flush=True)

def timing():
    # Cfg2-like dense (1.3B 480p): 12 heads, S=32760; and cross-attn; and VSA 720p union schedule
    for (H, Sq, Skv) in [(12, 32760, 32760), (40, 75600, 512), (5, 75600, 75600)]:
        q = torch.randn(1, Sq, H, 128, device=dev).bfloat16(); k = torch.randn(1, Skv, H, 128, device=dev).bfloat16(); v = torch.randn(1, Skv, H, 128, device=dev).bfloat16()
        o = torch.empty_like(q)
        for _ in range(2): ops.attention(q, k, v, out=o)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        n = 3
        for _ in range(n): ops.attention(q, k, v, out=o)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        fl = 4 * H * Sq * Skv * 128
        print(f"time dense H{H} Sq{Sq} Skv{Skv}: {ms:.3f} ms = {fl/ms/1e9:.0f} TFLOP/s", flush=True)
    # VSA 720p: 1440 blocks, topk 144, random lists (K1 bench shape, fewer heads to bound time)
    rng = np.random.default_rng(0)
    nblk, topk, H = 1440, 144, 8
    S = nblk * 64
    bmap = np.zeros((1, H, nblk, nblk), dtype=bool)
    for h in range(H):
        for qb in range(nblk):
            bmap[0, h, qb, rng.choice(nblk, topk, replace=False)] = True
    sched, cnt = vsa_index.pair_union_schedule(bmap)
    print("   mean union entries per pair:", cnt.mean(), flush=True)
    sched_t = torch.from_numpy(sched).to(dev); cnt_t = torch.from_numpy(cnt).to(dev)
    q = torch.randn(1, H, S, 128, device=dev).bfloat16().transpose(1, 2); k = torch.randn(1, H, S, 128, device=dev).bfloat16().transpose(1, 2); v = torch.randn(1, H, S, 128, device=dev).bfloat16().transpose(1, 2)
    o = torch.empty(1, H, S, 128, device=dev, dtype=torch.bfloat16).transpose(1, 2)
    for _ in range(2): ops.attention(q, k, v, out=o, sched=sched_t, sched_cnt=cnt_t, nqb=nblk, nkb=nblk)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(3): ops.attention(q, k, v, out=o, sched=sched_t, sched_cnt=cnt_t, nqb=nblk, nkb=nblk)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 3
    fl = 4 * H * S * topk * 64 * 128
    print(f"time VSA 720p H{H} topk{topk} random lists: {ms:.3f} ms = {fl/ms/1e9:.0f} useful TFLOP/s (x40/8 heads -> {ms*5:.2f} ms)", flush=True)

if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "ew"): elementwise_cases()
    if which in ("all", "attn"):
        dense_case(1, 1, 128, 128)
        dense_case(1, 2, 256, 256)
        dense_case(1, 2, 128, 512)
        dense_case(2, 3, 1000, 777)
        dense_case(1, 4, 1024, 1024, layout="bhsd")
        dense_case(1, 2, 333, 64)
        block_case(8, 4, 4, False)
        block_case(8, 4, 4, True)
        for tk in (1, 2, 3, 5, 7): block_case(8, tk, 2, True, seed=tk)
        block_case(16, 3, 2, True)
        block_case(9, 3, 2, True)     # odd block count
        block_case(8, 3, 2, True, zero_rows=True)
    if which in ("all", "time"): timing()
