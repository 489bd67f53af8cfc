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
