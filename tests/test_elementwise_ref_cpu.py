"""CPU: the element-by-element references of tests/elementwise_ref.py hold what they claim, and every checker rejects the
defects it exists to catch."""
import math

import numpy as np
import pytest
import torch

import elementwise_ref as R

CPU = "cpu"
K_MAX = 13824  # the largest reduction the GPU tests use on grid inputs (Wan's MLP width)


def _gen(seed):
    return torch.Generator(device=CPU).manual_seed(seed)


def test_grid_sums_are_exact_in_fp32_in_any_order():
    """Products of grid operands summed in fp32 sequentially, in shuffled orders, in 16-wide chains and pairwise: all equal
    the exact sum."""
    g = _gen(0)
    rows = 8
    x = R.grid_bf16((rows, K_MAX), g, CPU).float().numpy()
    w = R.grid_bf16((rows, K_MAX), g, CPU).float().numpy()
    # worst case too: every product at the largest magnitude with one sign
    x[0], w[0] = 15 / 16, 15 / 16
    prod = (x * w).astype(np.float32)
    assert np.array_equal(prod.astype(np.float64), x.astype(np.float64) * w.astype(np.float64))
    exact = prod.astype(np.float64).sum(1)
    rng = np.random.default_rng(1)
    for order in range(6):
        p = prod[:, rng.permutation(K_MAX)] if order else prod
        seq = np.cumsum(p, axis=1, dtype=np.float32)[:, -1]
        chains = p.reshape(rows, -1, 16).sum(2, dtype=np.float32)
        chained = np.cumsum(chains, axis=1, dtype=np.float32)[:, -1]
        pairwise = p.sum(1, dtype=np.float32)
        for s in (seq, chained, pairwise):
            assert np.array_equal(s.astype(np.float64), exact)


@pytest.mark.parametrize("K", [64, 1000, 5120, K_MAX])
def test_fp64_bound_accepts_fp32_sums_in_several_orders(K):
    g = _gen(K)
    x, w = R.rand_bf16((16, K), g, CPU), R.rand_bf16((16, K), g, CPU, K ** -0.5)
    b = R.rand_bf16((16,), g, CPU)
    e, A = R.exact_gemm(x, w)
    e, A = e.diagonal(), A.diagonal()
    p = (x.float() * w.float()).numpy()
    rng = np.random.default_rng(K)
    for order in range(4):
        q = p[:, rng.permutation(K)] if order else p
        acc = torch.from_numpy(np.cumsum(q, axis=1, dtype=np.float32)[:, -1].copy())
        assert bool(((acc.double() - e).abs() <= R.acc_coeff(K) * A).all())
        y = (acc + b.float()).bfloat16()
        ref, bound = R.epilogue_bound(e, A, K, R.EPI_BIAS, bias=b)
        R.assert_within(y, ref, bound, "bias epilogue")
        for epi in (R.EPI_GATE_F32, R.EPI_GATE_BF16, R.EPI_GATE_BF16R, R.EPI_RESID_BF16, R.EPI_GELU):
            r, gate = R.rand_bf16((16,), g, CPU), torch.randn(16, generator=g)
            if epi == R.EPI_GELU:
                out = R.gelu64(y.double()).float().bfloat16()
            else:
                out = R.epilogue_ref(acc, epi, bias=b, resid=r, gate=gate)
            ref, bound = R.epilogue_bound(e, A, K, epi, bias=b, resid=r, gate=gate)
            R.assert_within(out, ref, bound, f"epilogue {epi}")


def test_gelu_grid_bound_covers_the_kernel_formula():
    """The kernel's GELU(tanh) (t = 1 - 2 / (exp(2u) + 1), fp32), evaluated here in fp32 with a perturbed exp, stays within
    gelu_grid_bound, including y far below -4 where 1 + t cancels."""
    y = (torch.arange(-15 * 16, 15 * 16 + 1) / 16.0).bfloat16().float()
    k0, k1 = 0.7978845608028654, 0.044715
    u = torch.tensor(k0, dtype=torch.float32) * (y + torch.tensor(k1, dtype=torch.float32) * y * y * y)
    for rel in (1 + 2.0 ** -22, 1 - 2.0 ** -22):
        e = torch.exp(u * 2) * rel
        t = 1.0 - (2.0 / (e + 1.0)) * (1 + 2.0 ** -23)
        out = (0.5 * y * (1.0 + t)).bfloat16()
        ref, bound = R.gelu_grid_bound(y.double())
        R.assert_within(out, ref, bound, "gelu")
        assert bool((bound[y < -4] > R.ulp_bf16(ref[y < -4])).all())  # the absolute term carries the tail


# ------------------------------------------------------------------------------------------------ GEMM defects
def _gemm_case(grid, M=256, N=256, K=448, seed=3):
    g = _gen(seed)
    mk = (lambda s: R.grid_bf16(s, g, CPU)) if grid else (lambda s: R.rand_bf16(s, g, CPU))
    x, w, b = mk((M, K)), mk((N, K)), mk((N,))
    e, A = R.exact_gemm(x, w)
    out = R.epilogue_ref(e.float(), R.EPI_BIAS, bias=b)  # a correct kernel's output on grid inputs
    if not grid:
        out = (x.float() @ w.float().t() + b.float()).bfloat16()
    return x, w, b, e, A, out


def _defects(x, w, b, e, out):
    drop = x[128:256, 64:128].double() @ w[128:256, 64:128].double().t()
    kblock = out.clone()
    kblock[128:256, 128:256] = (e[128:256, 128:256] - drop + b[128:256].double()).float().bfloat16()
    swap = out.clone()
    swap[0:64, 8:16], swap[0:64, 16:24] = out[0:64, 16:24], out[0:64, 8:16]
    shift = out.clone()
    shift[129] = out[130]
    return {"k-block missing": kblock, "8-column groups swapped": swap, "row shifted": shift}


@pytest.mark.parametrize("grid", [True, False])
def test_gemm_checkers_reject_defects(grid):
    x, w, b, e, A, out = _gemm_case(grid)
    ref, bound = R.epilogue_bound(e, A, x.shape[1], R.EPI_BIAS, bias=b)
    check = (lambda o: R.assert_exact(o, R.epilogue_ref(e.float(), R.EPI_BIAS, bias=b), "gemm")) if grid else \
        (lambda o: R.assert_within(o, ref, bound, "gemm"))
    check(out)
    for name, mutant in _defects(x, w, b, e, out).items():
        with pytest.raises(AssertionError):
            check(mutant)


def test_sentinel_buffer_rejects_a_write_past_n():
    M, N, ldo = 5, 13, 24
    gd = R.Guarded(((M + 2) * ldo,), torch.bfloat16, CPU, seed=1)
    out = gd.region(gd.buf.as_strided((M, 16), (ldo, 1), ldo))
    out.fill_(1.0)
    gd.assert_untouched("inside only")
    gd.buf.view(torch.int16)[ldo + 16] ^= 1  # row 0, first column past N rounded to 8
    with pytest.raises(AssertionError):
        gd.assert_untouched("past N")
    f = R.Guarded((3, 8), torch.float32, CPU, seed=2)
    assert bool(torch.isfinite(f.buf).all())


# ------------------------------------------------------------------------------------------------ attention constructions
def simulate_kernel(q, k, v, visible, scale, tile=64):
    """The bf16 kernel's online softmax in fp32 (64-key tiles, running max, p = exp2(x - m), bf16 P, rescaled O and l)."""
    B, Sq, H, D = q.shape
    Skv = k.shape[1]
    sl = torch.tensor(R.scale_log2_f32(scale), dtype=torch.float32)
    o = torch.zeros(B, H, Sq, D)
    m = torch.full((B, H, Sq), float("-inf"))
    l = torch.zeros(B, H, Sq)
    qh, kh, vh = (t.permute(0, 2, 1, 3).float() for t in (q, k, v))
    for t0 in range(0, Skv, tile):
        s = (qh.double() @ kh[:, :, t0:t0 + tile].double().transpose(-1, -2)).float()
        x = (s * sl).masked_fill(~visible[..., t0:t0 + tile], float("-inf"))
        m_new = torch.maximum(m, x.amax(-1))
        m_use = torch.where(torch.isinf(m_new), torch.zeros_like(m_new), m_new)
        alpha = torch.exp2(m - m_use)
        p = torch.exp2(x - m_use[..., None])
        l = l * alpha + p.sum(-1)
        o = o * alpha[..., None] + (p.bfloat16().double() @ vh[:, :, t0:t0 + tile].double()).float()
        m = m_new
    inv = torch.where(l > 0, torch.ones_like(l) / l.clamp_min(1e-30), torch.zeros_like(l))
    out = (o * inv[..., None]).bfloat16()
    lse = torch.where(l > 0, m + torch.log2(l), torch.full_like(l, float("-inf")))
    return out.permute(0, 2, 1, 3), lse


def _blocks_visible(B, H, Sq, Skv, g):
    kv_len = [64, 0, 37, 64, 1]
    q_len = [64, 30, 64, 1, 64]
    q_block = R.block_of_rows(Sq, [64 * i for i in range(5)], q_len, CPU)
    kv_block = R.block_of_rows(Skv, [64 * i for i in range(5)], kv_len, CPU)
    sel = torch.rand(B, H, 5, 5, generator=g) < 0.4
    sel[:, :, 0, 2] = True
    return R.visible_mask(B, H, Sq, Skv, CPU, q_block, kv_block, sel)


@pytest.mark.parametrize("kind", ["uniform", "onehot"])
@pytest.mark.parametrize("masks", ["dense", "blocks"])
def test_tie_constructions_match_the_online_softmax(kind, masks):
    B, H = 2, 3
    g = _gen(7)
    Sq, Skv = (65, 257) if masks == "dense" else (320, 320)  # rows see more than 128 keys
    visible = R.visible_mask(B, H, Sq, Skv, CPU) if masks == "dense" else _blocks_visible(B, H, Sq, Skv, g)
    if kind == "uniform":
        q = torch.zeros(B, Sq, H, 128, dtype=torch.bfloat16)
        k = R.rand_bf16((B, Skv, H, 128), g, CPU)
    else:
        q, k, target = R.onehot_qk(B, H, Sq, Skv, visible, g, CPU)
    v = R.grid_bf16((B, Skv, H, 128), g, CPU)
    scale = 0.0625
    o, lse, cnt = R.tie_attention_ref(q, k, v, visible, scale)
    so, slse = simulate_kernel(q, k, v, visible, scale)
    R.assert_exact(so, o, "simulated o")
    R.assert_lse_tie(slse, lse, cnt, "simulated lse")
    if kind == "onehot":  # exactly one winner per row that sees a key: the target's v row and logit
        seen = target >= 0
        assert bool(seen.any()) and torch.equal(cnt, seen.float())
        vt = v.permute(0, 2, 1, 3).gather(2, target.clamp_min(0)[..., None].expand(B, H, Sq, 128))
        assert torch.equal(o.permute(0, 2, 1, 3)[seen], vt[seen])
        logit = torch.tensor(8192.0) * torch.tensor(R.scale_log2_f32(scale), dtype=torch.float32)
        assert bool((lse[seen] == logit).all())
        if masks == "blocks":
            assert int(visible.sum(-1).max()) > 128
    if kind == "uniform":
        assert torch.equal(cnt, visible.sum(-1).float())


def test_attention_bound_accepts_the_online_softmax_on_random_inputs():
    B, H, Sq, Skv = 1, 2, 70, 200
    g = _gen(9)
    q, k, v = (R.rand_bf16((B, S, H, 128), g, CPU) for S in (Sq, Skv, Skv))
    for visible in (R.visible_mask(B, H, Sq, Skv, CPU), _blocks_visible(B, H, 320, 320, g)[:, :, :Sq, :Skv]):
        so, slse = simulate_kernel(q, k, v, visible, 128 ** -0.5)
        oref, ob, lref, lb = R.attention_bound(q, k, v, visible, 128 ** -0.5)
        R.assert_within(so, oref, ob, "o")
        R.assert_lse_within(slse, lref, lb, "lse")


def test_attention_checkers_reject_defects():
    B, H, Sq, Skv = 2, 3, 65, 128
    g = _gen(11)
    visible = R.visible_mask(B, H, Sq, Skv, CPU)
    # uniform: one masked key counted
    q = torch.zeros(B, Sq, H, 128, dtype=torch.bfloat16)
    k = R.rand_bf16((B, Skv, H, 128), g, CPU)
    v = R.grid_bf16((B, Skv, H, 128), g, CPU)
    vis = visible.clone()
    vis[:, :, :, 100:] = False  # keys 100.. masked (a kv_len of 100)
    o, lse, cnt = R.tie_attention_ref(q, k, v, vis, 0.0625)
    counted = vis.clone()
    counted[1, 2, 40, 100] = True
    mo, ml = simulate_kernel(q, k, v, counted, 0.0625)
    with pytest.raises(AssertionError):
        R.assert_exact(mo, o, "masked key counted")
    with pytest.raises(AssertionError):
        R.assert_lse_tie(ml, lse, cnt, "masked key counted")
    # one-hot: a neighbouring head's K read by one head
    q, k, _ = R.onehot_qk(B, H, Sq, Skv, visible, g, CPU)
    o, lse, cnt = R.tie_attention_ref(q, k, v, visible, 0.0625)
    k_wrong = k.clone()
    k_wrong[:, :, 1] = k[:, :, 2]
    mo, ml = simulate_kernel(q, k_wrong, v, visible, 0.0625)
    with pytest.raises(AssertionError):
        R.assert_exact(mo, o, "neighbouring head's K")
    # a row shifted by one, on both constructions' reference and on the random bound
    shifted = o.clone()
    shifted[0, 10] = o[0, 11]
    with pytest.raises(AssertionError):
        R.assert_exact(shifted, o, "row shifted")
    q, k, v = (R.rand_bf16((B, S, H, 128), g, CPU) for S in (Sq, Skv, Skv))
    so, _ = simulate_kernel(q, k, v, visible, 128 ** -0.5)
    oref, ob, _, _ = R.attention_bound(q, k, v, visible, 128 ** -0.5)
    R.assert_within(so, oref, ob, "random")
    bad = so.clone()
    bad[0, 10] = so[0, 11]
    with pytest.raises(AssertionError):
        R.assert_within(bad, oref, ob, "row shifted")
    bad = simulate_kernel(q, torch.roll(k, 1, 2), v, visible, 128 ** -0.5)[0]
    with pytest.raises(AssertionError):
        R.assert_within(bad, oref, ob, "neighbouring head's K")


# ------------------------------------------------------------------------------------------------ attention backward
def simulate_bwd(q, k, v, o, dO, lse, visible, scale, order=1, perturb=0, tile=64):
    """The attention backward in fp32 the way the kernels tile it: S and dP in fp32 from exact dots, P = exp2(fma(s,
    scale_log2, -lse)) with a relative perturbation of perturb * 2^-22 (ex2 is exact at 0), bf16 P and dS, and dV, dK, dQ
    accumulated in fp32 one 64-row tile at a time, in ascending (order 1) or descending (order -1) walk order. Returns dq,
    dk, dv (BSHD bf16) and delta (fp32 [B, H, Sq])."""
    qh, kh, vh, oh, gh = (t.permute(0, 2, 1, 3).double() for t in (q, k, v, o, dO))
    Sq, Skv = qh.shape[2], kh.shape[2]
    sl = R.scale_log2_f32(scale)
    delta = (gh * oh).sum(-1).float()
    s = (qh @ kh.transpose(-1, -2)).float()
    dp = (gh @ vh.transpose(-1, -2)).float()
    x = (s.double() * sl - lse.double()[..., None]).float()  # fma: the exact product, one rounding
    p = torch.exp2(x.double())
    p = torch.where(x == 0, p, p * (1 + perturb * 2.0 ** -22)).float().masked_fill(~visible, 0)
    ds = (p * (dp - delta[..., None])) * torch.full_like(p, R.f32(scale))
    pb, dsb = p.bfloat16().double(), ds.bfloat16().double()
    dq = torch.zeros(qh.shape, dtype=torch.float32)
    dk = torch.zeros(kh.shape, dtype=torch.float32)
    dv = torch.zeros(kh.shape, dtype=torch.float32)
    for t in list(range(0, Sq, tile))[::order]:
        r = slice(t, t + tile)
        dv += (pb[:, :, r].transpose(-1, -2) @ gh[:, :, r]).float()
        dk += (dsb[:, :, r].transpose(-1, -2) @ qh[:, :, r]).float()
    for t in list(range(0, Skv, tile))[::order]:
        c = slice(t, t + tile)
        dq += (dsb[:, :, :, c] @ kh[:, :, c]).float()
    out = lambda a: a.bfloat16().permute(0, 2, 1, 3)
    return out(dq), out(dk), out(dv), delta


BWD_EXACT = ["onehot", "uniform_q", "uniform_k"]


def _bwd_case(kind, masks, seed, scale=2.0 ** -4):
    B, H = 2, 3
    g = _gen(seed)
    Sq, Skv = (65, 257) if masks == "dense" else (320, 320)
    visible = R.visible_mask(B, H, Sq, Skv, CPU) if masks == "dense" else _blocks_visible(B, H, Sq, Skv, g)
    return R.bwd_inputs(kind, B, H, Sq, Skv, visible, g, CPU, scale), visible


@pytest.mark.parametrize("kind", BWD_EXACT)
@pytest.mark.parametrize("masks", ["dense", "blocks"])
def test_bwd_constructions_match_the_tiled_simulation(kind, masks):
    (q, k, v, o, dO, lse), visible = _bwd_case(kind, masks, 21)
    dq, dk, dv, delta, P = R.bwd_exact_ref(q, k, v, o, dO, lse, visible, 2.0 ** -4)
    if masks == "blocks":  # rows that see more than 128 keys, rows that see none
        assert int(visible.sum(-1).max()) > 128 and bool((~visible.any(-1)).any())
    for order in (1, -1):
        for perturb in (1, -1):
            sq, sk, sv, sd = simulate_bwd(q, k, v, o, dO, lse, visible, 2.0 ** -4, order, perturb)
            for got, ref, name in ((sq, dq, "dq"), (sk, dk, "dk"), (sv, dv, "dv")):
                R.assert_exact(got, ref, f"simulated {name}", where=R.bwd_coords)
            assert torch.equal(sd, delta)
    seen = visible.any(-1)
    if kind == "onehot":  # exactly one key per row that sees any: dV_j sums dO over the rows that target j
        assert torch.equal(P.sum(-1), seen.double())
    else:  # every visible pair
        assert torch.equal(P.bool(), visible)
    nz = lambda t: bool((t != 0).any())
    assert nz(dq) == (kind != "uniform_k") and nz(dk) == (kind != "uniform_q") and nz(dv)


@pytest.mark.parametrize("scale", [2.0 ** -4, 128 ** -0.5])
@pytest.mark.parametrize("masks", ["dense", "blocks"])
def test_attention_bwd_bound_accepts_the_simulation(scale, masks):
    (q, k, v, o, dO, lse), visible = _bwd_case("random", masks, 23, scale)
    bounds = R.attention_bwd_bound(q, k, v, o, dO, lse, visible, scale)
    for order in (1, -1):
        for perturb in (1, -1):
            sim = simulate_bwd(q, k, v, o, dO, lse, visible, scale, order, perturb)
            for got, (ref, b), name in zip(sim, bounds, ("dq", "dk", "dv", "delta")):
                R.assert_within(got, ref, b, f"simulated {name}", where=R.bwd_coords if name != "delta" else None)


def _bwd_checker(kind, q, k, v, o, dO, lse, visible, scale):
    """check(dq, dk, dv) against the exact reference (constructions) or the element bound (random)."""
    if kind == "random":
        refs = R.attention_bwd_bound(q, k, v, o, dO, lse, visible, scale)[:3]
        return lambda *outs: [R.assert_within(t, r, b, n) for t, (r, b), n in zip(outs, refs, "qkv")]
    refs = R.bwd_exact_ref(q, k, v, o, dO, lse, visible, scale)[:3]
    return lambda *outs: [R.assert_exact(t, r, n) for t, r, n in zip(outs, refs, "qkv")]


@pytest.mark.parametrize("kind", ["onehot", "uniform_q", "uniform_k", "random"])
def test_attention_bwd_checkers_reject_defects(kind):
    """Each defect, made by running the simulation on altered inputs or editing its output, fails the check of at least
    the gradient it touches."""
    B, H, Sq, Skv = 2, 3, 129, 192
    g = _gen(31)
    visible = R.visible_mask(B, H, Sq, Skv, CPU)
    visible[:, :, :, 150:] = False  # a kv_len of 150: masked keys to count
    scale = 2.0 ** -4
    q, k, v, o, dO, lse = R.bwd_inputs(kind, B, H, Sq, Skv, visible, g, CPU, scale)
    check = _bwd_checker(kind, q, k, v, o, dO, lse, visible, scale)
    dq, dk, dv, _ = simulate_bwd(q, k, v, o, dO, lse, visible, scale)
    check(dq, dk, dv)

    def rejects(*outs):
        with pytest.raises(AssertionError):
            check(*outs)

    def sim(vis=visible, l=lse):
        return simulate_bwd(q, k, v, o, dO, l, vis, scale)

    vis = visible.clone()
    vis[1, 2, 64:128, 64:128] = False  # one 64-key tile missing from one dQ tile, one q tile from one dK / dV tile
    mq, mk, mv, _ = sim(vis)
    m = dq.clone()
    m[1, 64:128, 2] = mq[1, 64:128, 2]
    if kind != "uniform_k":
        rejects(m, dk, dv)
    m = dv.clone()
    m[1, 64:128, 2] = mv[1, 64:128, 2]
    rejects(dq, dk, m)
    if kind != "uniform_q":
        m = dk.clone()
        m[1, 64:128, 2] = mk[1, 64:128, 2]
        rejects(dq, m, dv)
    # a row shifted by one, a head swapped, in the gradients the construction makes row- and head-dependent
    for i, t in enumerate((dq, dk, dv)):
        if not bool((t != 0).any()) or (kind.startswith("uniform") and i == 2):
            continue  # uniform: every dv row of a head sums the same rows
        outs = [dq, dk, dv]
        shifted = t.clone()
        shifted[1, 70] = t[1, 71]
        outs[i] = shifted
        rejects(*outs)
        head = t.clone()
        head[0, 64:128, 1] = t[0, 64:128, 2]
        outs[i] = head
        rejects(*outs)
    if kind.startswith("uniform"):  # one masked key counted in one row
        vis = visible.clone()
        vis[1, 2, 100, 150] = True
        mq, mk, mv, _ = sim(vis)
        rejects(dq, dk, mv)
        rejects(dq, mk, dv) if kind == "uniform_k" else rejects(mq, dk, dv)
    if kind in ("onehot", "random"):  # an lse off by 0.25 in one row
        l2 = lse.clone()
        l2[0, 1, 40] += 0.25
        mq, mk, mv, _ = sim(l=l2)
        rejects(mq, dk, dv)
        rejects(dq, dk, mv)


# ------------------------------------------------------------------------------------------------ row kernels
def _sim_rstd(x, D, eps, warp, centred, mean=None):
    """The kernels' statistics in torch fp32: block-per-row sums (256 per-thread partials, then a tree) with IEEE division,
    or warp-per-row pairwise sums over the 32 lanes with a multiply by fl(1 / D) fused into one fma; rsqrt rounded to
    fp32 and moved one ulp (within rsqrtf's 2 ulp)."""
    xf = x.float()
    M = xf.shape[0]
    lanes = 32 if warp else 256
    pad = (-D) % (8 * lanes)
    xp = torch.cat([xf, xf.new_zeros(M, pad)], 1).view(M, -1, lanes, 8)

    def tree(v):  # per-lane sums in chunk order, then a butterfly over the lanes
        acc = v[:, 0].sum(-1)
        for k in range(1, v.shape[1]):
            acc = acc + v[:, k].sum(-1)
        while acc.shape[1] > 1:
            acc = acc[:, 0::2] + acc[:, 1::2]
        return acc[:, 0]

    Dt = torch.full((M,), float(D))
    inv = torch.ones(M) / Dt
    if centred:
        s = tree(xp)
        mean = s * inv if warp else s / Dt
        d = xp - torch.where(torch.arange(xp.shape[1] * lanes * 8).view(1, -1, lanes, 8) < D, mean[:, None, None, None], xp)
        q = tree(d * d)
    else:
        mean = torch.zeros(M)
        q = tree(xp * xp)
    v = (q.double() * inv.double() + R.f32(eps)).float() if warp else q / Dt + torch.full((M,), R.f32(eps))
    r = torch.nextafter((1.0 / v.double().sqrt()).float(), torch.full((M,), math.inf))
    return mean, r


def _row_sim(M, D, seed, f32_rows=False):
    g = _gen(seed)
    x, c, qz, qx = R.exact_rows(M, D, g, CPU)
    return (x if f32_rows else x.bfloat16()), c, qz, qx, g


@pytest.mark.parametrize("warp", [False, True])
@pytest.mark.parametrize("D", [8, 264, 1536, 2056, 5120])
def test_layernorm_reference_accepts_the_kernel_arithmetic(D, warp):
    """Exact rows: the simulated kernel (either path's sum order, a perturbed rsqrt) equals ln_chain at one candidate rstd
    per row, for every modulation form; the fp64 bound accepts the simulation on random rows."""
    x, c, qz, _, g = _row_sim(40, D, D)
    mean, r = _sim_rstd(x, D, 1e-6, warp, True)
    assert torch.equal(mean, c)
    cands = R.rstd_candidates(R.var_forms(qz, D, 1e-6, warp))
    w, b, sc, sh = (torch.randn(D, generator=g) * 0.5 for _ in range(4))
    for kw in (dict(round_ln=1, scale=sc, shift=sh), dict(w=w, b=b), dict(round_ln=3, scale=sc.bfloat16().float(),
                                                                            shift=sh.bfloat16().float())):
        got = R.ln_chain(x, mean, r, **kw)
        R.assert_rows_match(got, lambda rr: R.ln_chain(x, c, rr, **kw), cands, "sim")
        xr = (torch.randn(40, D, generator=g) * 2 + 1).bfloat16()
        m2, r2 = _sim_rstd(xr, D, 1e-6, warp, True)
        ref, bound = R.ln_fwd_bound(xr.float(), 1e-6, **kw)
        R.assert_within(R.ln_chain(xr, m2, r2, **kw), ref, bound, "sim random")


def test_layernorm_checkers_reject_wrong_statistics_and_groups():
    """One row normalised with the previous row's statistics, and the last rows of a modulation group given the next
    group's vectors: both fail the exact check (and the statistics defect the bound)."""
    M, D, Rg = 24, 1536, 10
    x, c, qz, _, g = _row_sim(M, D, 1)
    cands = R.rstd_candidates(R.var_forms(qz, D, 1e-6, True))
    mean, r = _sim_rstd(x, D, 1e-6, True, True)
    sc, sh = torch.randn(3, D, generator=g), torch.randn(3, D, generator=g)
    grp = torch.arange(M) // Rg
    chain = lambda rr: R.ln_chain(x, c, rr, scale=sc[grp], shift=sh[grp], round_ln=1)
    m2, r2 = mean.clone(), r.clone()
    m2[7], r2[7] = mean[6], r[6]
    with pytest.raises(AssertionError, match="match no candidate"):
        R.assert_rows_match(R.ln_chain(x, m2, r2, scale=sc[grp], shift=sh[grp], round_ln=1), chain, cands, "stats")
    grp2 = grp.clone()
    grp2[8:10] = 1
    with pytest.raises(AssertionError, match="match no candidate"):
        R.assert_rows_match(R.ln_chain(x, mean, r, scale=sc[grp2], shift=sh[grp2], round_ln=1), chain, cands, "group")
    xr = (torch.randn(M, D, generator=g) * 2 + torch.randn(M, 1, generator=g)).bfloat16()
    m3, r3 = _sim_rstd(xr, D, 1e-6, True, True)
    ref, bound = R.ln_fwd_bound(xr.float(), 1e-6)
    m3[7], r3[7] = m3[6], r3[6]
    with pytest.raises(AssertionError, match="outside the element bound"):
        R.assert_within(R.ln_chain(xr, m3, r3), ref, bound, "stats random")


def _rope_case(M, D, hd, f64, g):
    x, c, qz, qx = R.exact_rows(M, D, g, CPU)
    x = x.bfloat16()
    S = M + 5
    prow = torch.randperm(S, generator=g)[:M]
    ang = torch.rand(S, hd // 2, generator=g, dtype=torch.float64) * 6.3
    cos, sin = (f(ang).repeat_interleave(2, 1) for f in (torch.cos, torch.sin))
    if not f64:
        cos, sin = cos.float(), sin.float()
    cols = torch.arange(D) % hd
    w = (torch.randn(D, generator=g) * 0.5 + 1).bfloat16()
    return x, qx, w, prow, cos, sin, cols


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("hd", [24, 128, 512])
def test_rmsnorm_rope_reference_accepts_and_rejects(hd, f64):
    """The simulated kernel matches rms_rope_chain at one candidate per row; a table slice 8 columns off inside a head,
    cos and sin swapped, and rope_row ignored all fail."""
    M, D = 16, 1536
    x, qx, w, prow, cos, sin, cols = _rope_case(M, D, hd, f64, _gen(hd))
    _, r = _sim_rstd(x, D, 1e-6, True, False)
    cands = R.rstd_candidates(R.var_forms(qx, D, 1e-6, True))
    ce, se = cos[prow][:, cols], sin[prow][:, cols]
    chain = lambda rr: R.rms_rope_chain(x, rr, w, False, ce, se, f64)
    R.assert_rows_match(R.rms_rope_chain(x, r, w, False, ce, se, f64), chain, cands, "sim")
    shifted = (cols // hd) * hd + (cols % hd + 8) % hd
    for name, (c2, s2) in {"shift 8": (cos[prow][:, shifted], sin[prow][:, shifted]), "swap": (se, ce),
                           "rope_row ignored": (cos[:M][:, cols], sin[:M][:, cols])}.items():
        with pytest.raises(AssertionError, match="match no candidate"):
            R.assert_rows_match(R.rms_rope_chain(x, r, w, False, c2, s2, f64), chain, cands, name)


def _sim_colsum(T, parts, order=None, drop=None, twice=None):
    """Kernel-style column sums with optional defects: partials added in another order, one dropped or added twice."""
    _, acc = R.colsum_replay(T, parts)
    idx = list(range(parts)) if order is None else order
    if drop is not None:
        idx.remove(drop)
    if twice is not None:
        idx.append(twice)
    return R.partial_sum(acc[idx])


@pytest.mark.parametrize("M,N", [(2048, 1032), (1793, 8), (529, 1536)])
def test_column_sum_replay_and_its_defects(M, N):
    """The replay equals a row-by-row fp32 simulation of the kernels (including the 8-row unrolled loop, which keeps
    the order); a dropped, doubled or reordered partial and a missing last 1024-column block all change the bits."""
    g = _gen(M + N)
    T = R.rand_bf16((M, N), g, CPU).float()
    parts = min(M, R.BG_PARTS if M != 529 else R.RB_CTAS)
    acc = torch.zeros(parts, N)
    for row in range(M):  # the kernel's loop, one row at a time
        acc[row % parts] = acc[row % parts] + T[row]
    ref = R.colsum_replay(T, parts)[0]
    assert torch.equal(R.partial_sum(acc), ref)
    defects = {"dropped": _sim_colsum(T, parts, drop=parts - 1), "twice": _sim_colsum(T, parts, twice=0),
               "reversed": _sim_colsum(T, parts, order=list(range(parts))[::-1])}
    if N > 1024:
        cut = ref.clone()
        cut[1024:] = 0  # the last 1024-column block never launched
        defects["last column block"] = cut
    for name, got in defects.items():
        with pytest.raises(AssertionError, match="not bit-exact"):
            R.assert_exact(got, ref, name)  # the fp32 sums (d_gate, d_offset, d_shift are stored unrounded)


@pytest.mark.parametrize("M,Rg,budget", [(45, 8, 528), (1003, 100, 256), (700, 1, 256), (1000, 1200, 528)])
def test_grouped_replay_and_an_unwritten_partial(M, Rg, budget):
    """The grouped replay equals a row-by-row simulation; a CTA with no rows that leaves its partial unwritten (NaN
    workspace) changes its group's sum."""
    g = _gen(M)
    T = R.rand_bf16((M, 16), g, CPU).float()
    G, P = -(-M // Rg), R.grouped_parts(M, Rg, budget)
    acc = torch.zeros(G, P, 16)
    for row in range(M):
        gi, r = divmod(row, Rg)
        acc[gi, r % P] = acc[gi, r % P] + T[row]
    tot, parts = R.grouped_colsum_replay(T, Rg, budget)
    assert torch.equal(parts, acc)
    assert torch.equal(tot, torch.stack([R.partial_sum(acc[i]) for i in range(G)]))
    last = M - (G - 1) * Rg
    if last < P:
        bad = acc.clone()
        bad[G - 1, P - 1] = float("nan")
        with pytest.raises(AssertionError):
            R.assert_exact(R.partial_sum(bad[G - 1]), tot[G - 1], "unwritten partial")


def test_row_case_lists_reach_every_path():
    """The GPU file's case lists reach every launch choice of each entry point."""
    T = pytest.importorskip("test_gpu_rowops_elementwise")
    ln = [T.ln_path(M, D, f32, aff, mod, Rg) for M, D, f32, aff, mod, Rg, rl, h in T.LN_CASES]
    assert {p["warp"] for p in ln} == {True, False}
    assert {p["nw"] for p in ln if p["warp"]} >= {16, 9, 12, 8}
    assert {p["stages"] for p in ln if p["warp"]} == {1, 2} and {p["tab_kind"] for p in ln if p["warp"]} == {0, 1, 2}
    assert any(p["wraps"] > 2 and p["ragged"] for p in ln if p["warp"])
    assert {p["chunks"] for p in ln if not p["warp"]} == {1, 2, 3, 4}
    assert any(not p["warp"] and c[2] and c[1] > 6144 for p, c in zip(ln, T.LN_CASES))
    assert {c[6] for c in T.LN_CASES} == {0, 1, 3} and {c[2] for c in T.LN_CASES} == {True, False}
    assert {c[5] for c in T.LN_CASES} >= {0, 1} and any(c[5] >= c[0] for c in T.LN_CASES)
    assert any(c[5] > 1 and c[0] % c[5] for c in T.LN_CASES)
    assert {c[1] for c in T.LN_CASES} >= {8, 256, 264, 1536, 2048, 2056, 5120, 6144, 8192}
    rms = [(T.rms_path(M, D, hd, f64), c) for c in T.RMS_CASES for M, D, hd, two, f64, wf, rr, sc in [c]]
    for warp in (True, False):
        assert {p["hoisted"] for p, c in rms if p["warp"] == warp} == {True, False}
        assert any(c[7] for p, c in rms if p["warp"] == warp)  # col_offsets
        assert any(c[4] for p, c in rms if p["warp"] == warp) and any(c[5] for p, c in rms if p["warp"] == warp)
    assert {p["stages"] for p, c in rms if p["warp"]} == {1, 2}
    assert {c[2] for c in T.RMS_CASES} >= {24, 64, 96, 128, 192, 512}
    assert {c[3] for c in T.SCATTER_CASES} == {"norm", "rope_only", "copy"} and any(c[0] == 1 for c in T.SCATTER_CASES)
    assert {c[0] for c in T.RMS_BWD_CASES} >= {1, 527, 528, 529, 1063} and {c[0] for c in T.LN_BWD_CASES} >= {1, 527, 528, 529, 1063}
    assert {T.bwd_path("ln", M, D)["chunks"] for M, D, *_ in T.LN_BWD_CASES} == {1, 2, 3, 4}
    assert {c[5] for c in T.LN_BWD_CASES} == {None, "bf16", "f32"} and {c[4] for c in T.LN_BWD_CASES} == {0, 1}
    assert {c[3] for c in T.LN_BWD_CASES} == {True, False} and {c[2] for c in T.LN_BWD_CASES} == {True, False}
    bias = [T.bwd_path("bias", M, N) for M in T.BIAS_M for N in T.BIAS_N]
    assert {p["col_blocks"] for p in bias} == {1, 2, 5} and {p["unrolled"] for p in bias} == {True, False}
    for kind, budget in (("ln_grouped", R.RB_CTAS), ("gate_grouped", R.BG_PARTS)):
        gp = [(T.bwd_path(kind, M, N, Rg), Rg) for M, Rg, N in T.GROUPED_CASES]
        assert any(p["G"] == 1 and p["P"] == min(budget, Rg) for p, Rg in gp)
        assert any(p["G"] > budget and p["P"] == 1 for p, Rg in gp)
        assert any(p["P"] == Rg and p["G"] > 1 for p, Rg in gp)
        assert any(p["last"] < Rg and p["empty_parts"] for p, Rg in gp)
        assert any(p["G"] == 21 and Rg == 1560 for p, Rg in gp)


# ------------------------------------------------------------------------------------------------ convolutions
def _conv_operands(g, T_in, H, W, Cin, Cout, k, pad=0):
    x = R.grid_bf16((T_in, H, W, Cin), g, CPU).float()
    w = R.grid_bf16((Cout, k[0] * k[1] * k[2], Cin + pad), g, CPU).float()
    return x, w


@pytest.mark.parametrize("k,t_off,T_out", [((3, 3, 3), 0, 3), ((3, 3, 3), 1, 2), ((3, 3, 3), 2, 1), ((1, 1, 1), 0, 2),
                                           ((1, 3, 3), 0, 2), ((3, 1, 1), 1, 2)])
def test_conv_reference_matches_torch_conv3d(k, t_off, T_out):
    """conv_exact against F.conv3d (fp32, grid operands: exact) on the causal, zero-padded input, channels past Cin
    ignored, frames past t_off + T_out unused."""
    import torch.nn.functional as F
    g = _gen(1)
    T_in, H, W, Cin, Cout = t_off + T_out + 1, 9, 17, 24, 40
    x, w = _conv_operands(g, T_in, H, W, Cin, Cout, k, pad=8)
    x[t_off + T_out:] = 1e30
    e, A = R.conv_exact(x, w, k, T_out, t_off)
    kt, kh, kw = k
    xc = x[:t_off + T_out].permute(3, 0, 1, 2)[None]
    xc = F.pad(xc, (kw // 2, kw // 2, kh // 2, kh // 2, kt - 1, 0))
    wc = w[:, :, :Cin].reshape(Cout, kt, kh, kw, Cin).permute(0, 4, 1, 2, 3)
    ref = F.conv3d(xc, wc)[0, :, -T_out:].permute(1, 2, 3, 0)
    assert torch.equal(e.float(), ref)
    assert bool((A >= e.abs()).all())
    R.assert_conv_exact_premise(A, 2.0 ** -8, "grid")


def test_conv_reference_matches_fp8_restatement():
    """conv_exact on e4m3 operands against vae_fp8_ref.fp8_conv3d_exact (channels-first, F.conv3d in fp64)."""
    import vae_fp8_ref
    g = _gen(2)
    x = torch.randn(4, 8, 16, 32, generator=g).clamp(-400, 400).to(torch.float8_e4m3fn)
    w = (torch.randn(48, 32, 3, 3, 3, generator=g) * 4).to(torch.float8_e4m3fn)
    ws = torch.rand(48, generator=g) + 0.5
    y = vae_fp8_ref.fp8_conv3d_exact(x.float().permute(3, 0, 1, 2)[None], 0.25, w.float(), ws)[0].permute(1, 2, 3, 0)
    e, _ = R.conv_exact(x.float(), w.float().permute(0, 2, 3, 4, 1).reshape(48, 27, 32), (3, 3, 3), 4, 0)
    assert torch.allclose(e * 0.25 * ws.double(), y, rtol=1e-12, atol=1e-9)


def test_conv_probe_weights_cover_every_tap_and_chunk():
    g = _gen(3)
    for Cout, ntaps, Cin in ((96, 27, 96), (192, 27, 384), (104, 9, 48), (128, 3, 128)):
        w = R.probe_weights(Cout, ntaps, Cin, Cin + 32, g, CPU)
        nz = (w != 0).sum((1, 2))
        assert bool((nz >= 1).all() and (nz <= 3).all()) and bool((w[:, :, Cin:] == 0).all())
        taps, chunks = R.probe_coverage(Cout, ntaps, Cin)
        assert taps == set(range(ntaps)) and chunks == set(range(-(-Cin // 32)))
        single = w[0::3]
        assert bool(((single != 0).sum((1, 2)) == 1).all())
        for j in range(single.shape[0]):
            tap, ch = (single[j] != 0).nonzero()[0].tolist()
            assert tap == j % ntaps and ch // 32 == j % -(-Cin // 32)


def test_conv_case_lists_reach_every_instantiation():
    """The GPU file's dispatch cases reach every (fp8, BN, BK, NORM, KSUB) the host can launch, with the channel counts
    whose TMA box runs past Cin, every Cout boundary, every spatial and time edge."""
    T = pytest.importorskip("test_gpu_conv_elementwise")
    cases = T.DISPATCH_CASES + T.EDGE_CASES + T.NORM_CASES + T.PERSISTENT_CASES
    reached = {T.conv_path(c["Cin"], c["Cout"], c["fp8"], c["norm"]) for c in cases}
    assert reached == T.conv_instantiations() and len(reached) == 77
    # the host's tile choice, restated: BN by Cout boundaries, BK by Cin_pad, KSUB where three k-blocks share a stage
    assert [T.conv_path(64, n, False, 0)[1] for n in (16, 17, 96, 97, 128, 129)] == [16, 96, 96, 128, 128, 192]
    assert {c["Cin"] for c in cases if not c["fp8"]} >= {16, 40, 72} and 48 in {c["Cin"] for c in cases if c["fp8"]}
    assert {c["W"] for c in cases} >= {1, 15, 16, 17, 33} and {c["H"] for c in cases} >= {1, 7, 8, 9}
    assert {(c["k"][0], c["t_off"]) for c in cases} >= {(3, 0), (3, 1), (3, 2), (1, 0)}
    assert max(c["T_out"] for c in cases if c["k"][0] == 3) == 4
    assert {c["interleave"] for c in cases} >= {32, 64, 384}
    assert {c["Cout"] for c in cases} >= {3, 200, 384, 576, 768}
    assert any(c["fp8"] and c["Cout"] > 512 for c in cases)
    assert any(c["out_gap"] % 2 for c in cases) and any(c["out_off"] % 2 for c in cases)
    assert any(c["resid"] and c["resid_gap"] for c in cases)
    norm = [c for c in cases if c["norm"]]
    assert {c["Cout"] for c in norm} >= {24, 96, 128, 136, 192}
    assert {(c["fp8"], c["norm"], c["raw"], c["silu"]) for c in norm} >= {(f, n, r, False) for f in (0, 1) for n in (1, 2)
                                                                         for r in (0, 1)}
    assert any(c["bound0"] for c in norm) and any(c["norm_gap"] for c in norm)


def _norm_row(g, P, C):
    return R.rand_bf16((P, C), g, CPU)


def test_conv_norm_replay_matches_the_formula():
    """The fused norm's replay and the row pass's replay against the fp64 formula (a few fp32 ulp apart), their sums of
    squares against an fp64 sum, and the e4m3 code against vae_fp8_ref.quantize_static where v is not -0."""
    import vae_fp8_ref
    g = _gen(4)
    for C in (24, 96, 136, 192, 8, 264, 384):
        y = _norm_row(g, 300, C)
        y[0] = 0  # the 1e-12 floor
        gamma = 1 + 0.2 * torch.randn(C, generator=g)
        y64 = y.double()
        ref = y64 / y64.norm(dim=1, keepdim=True).clamp_min(1e-12) * math.sqrt(C) * gamma.double()
        for v in ([R.conv_norm_replay(y, gamma, C)] if C <= 192 else []) + [R.rownorm_replay(y, gamma)]:
            assert torch.allclose(v.double(), ref, rtol=2 ** -20, atol=1e-30)
        ss = R.norm_sum_replay(y, C) if C <= 192 else None
        if ss is not None:
            assert torch.allclose(ss.double(), (y.double() ** 2).sum(1), rtol=C * 2 ** -24)
        bound = vae_fp8_ref.norm_bound(gamma)
        v = R.rownorm_replay(y, gamma)
        code = R.e4m3_code(v, R.e4m3_qscale(bound))
        pos = v != 0
        assert torch.equal(code.view(torch.uint8)[pos], vae_fp8_ref.quantize_static(v, bound).view(torch.uint8)[pos])
    assert R.e4m3_code(torch.tensor([-1.0, 1.0]), 0.0).view(torch.uint8).tolist() == [0x80, 0]


def test_conv_norm_checkers_reject_defects():
    """A norm with sqrt(BN) in place of sqrt(Cout), a sum that skips the last column group, and one e4m3 code a step off
    fail the exact check; SiLU outputs one bf16 ulp off the interval fail assert_rounds_from."""
    g = _gen(5)
    C = 104
    y = _norm_row(g, 500, C)
    gamma = 1 + 0.2 * torch.randn(C, generator=g)
    qs = R.e4m3_qscale(math.sqrt(C) * float(gamma.abs().max()))
    good = R.e4m3_code(R.conv_norm_replay(y, gamma, C), qs).view(torch.uint8)
    bad_bn = R.e4m3_code(R.conv_norm_replay(y, gamma, C, sqrt_of=128), qs).view(torch.uint8)
    with pytest.raises(AssertionError):
        R.assert_exact(bad_bn, good, "sqrt(BN)")
    short = R.e4m3_code(R.conv_norm_replay(y[:, :96].contiguous(), gamma[:96], 96, sqrt_of=C), qs).view(torch.uint8)
    with pytest.raises(AssertionError):
        R.assert_exact(short, good[:, :96], "a column group missing from the sum")
    step = good.clone()
    step[7, 11] += 1
    with pytest.raises(AssertionError):
        R.assert_exact(step, good, "one code one step off")
    v = R.conv_norm_replay(y, gamma, C)
    ref, b = R.silu_bound(v)
    got = (v.double() * torch.sigmoid(v.double())).float().bfloat16()
    assert R.assert_rounds_from(got.float(), ref, b, "silu") < 0.05
    off = got.float().clone()
    off[3, 4] = torch.nextafter(off[3, 4].bfloat16(), torch.tensor(1e30, dtype=torch.bfloat16)).float()
    off[3, 4] = off[3, 4] + R.ulp_bf16(off[3, 4:5]).float()[0]
    with pytest.raises(AssertionError):
        R.assert_rounds_from(off, ref, b, "one ulp off")


def test_conv_checkers_reject_data_movement_defects():
    """On a CPU-simulated grid output: one tap dropped in a border tile, one tile's halo shifted by a pixel, two 8-column
    groups swapped in the second N block, bias column n - 512 for n >= 512, interleave frames swapped."""
    g = _gen(6)
    k, T_out, t_off = (3, 3, 3), 2, 1
    x, w = _conv_operands(g, 4, 9, 33, 16, 600, k)
    bias = R.grid_bf16((600,), g, CPU)
    e, A = R.conv_exact(x, w, k, T_out, t_off)
    R.assert_conv_exact_premise(A, 2.0 ** -8, "sim")
    ref = R.conv_epilogue_ref(e.float(), bias)
    where = lambda i: R.conv_coords(i, 192)

    def rejected(m, name):
        with pytest.raises(AssertionError):
            R.assert_exact(m, ref, name, where)

    w2 = w.clone()
    w2[:, 18] = 0  # tap (dt 2, dh 0, dw 0): pixel (8, 32) reads (7, 31) through it
    m = ref.clone()
    m[:, 8:, 32:] = R.conv_epilogue_ref(R.conv_exact(x, w2, k, T_out, t_off, False)[0].float(), bias)[:, 8:, 32:]
    rejected(m, "tap dropped")
    m = ref.clone()
    m[:, :8, 16:32] = R.conv_epilogue_ref(R.conv_exact(torch.roll(x, 1, 2), w, k, T_out, t_off, False)[0].float(),
                                          bias)[:, :8, 16:32]
    rejected(m, "halo shifted")
    m = ref.clone()
    m[..., 192:200], m[..., 200:208] = ref[..., 200:208], ref[..., 192:200]
    rejected(m, "column groups swapped")
    rejected(R.conv_epilogue_ref(e.float(), torch.cat([bias[:512], bias[:88]])), "bias n - 512")
    il = torch.stack([ref[..., :300], ref[..., 300:]], 1).flatten(0, 1)  # frames 2t, 2t + 1
    swapped = torch.stack([ref[..., 300:], ref[..., :300]], 1).flatten(0, 1)
    assert not torch.equal(il, swapped)
    assert R.conv_coords((1, 8, 32, 200), 192) == dict(t=1, y=8, x=32, n=200, tile=(1, 2), row=0, warpgroup=0, warp=0,
                                                        n_blk=1, col_group=1)


def test_softmax_bound_holds_for_float32_softmax():
    g = _gen(7)
    x = torch.randn(6, 1350, generator=g) * 4
    x[2, ::7] = float("-inf")
    ref, b = R.softmax_bound(x)
    got = torch.softmax(x, -1).bfloat16()
    R.assert_within(got, ref, b, "torch fp32 softmax")
    assert bool(((b / ref.clamp_min(1e-300))[ref > 1e-30] < 2 ** -7).all())
