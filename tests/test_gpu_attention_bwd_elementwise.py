"""GPU: the attention backward (fvb_attention_bwd, fvb_attention_sparse_bwd, fvb_attention_blocklist_bwd) element by
element: the one-hot, uniform-q and uniform-k constructions bit for bit, random inputs against fp64 element bounds
(tests/elementwise_ref.py, "Attention backward"); dq, dk, dv written into sentinel buffers with gaps between tokens and
heads, the delta workspace checked too, lse read from a buffer with gaps; two calls give the same bits."""
from ctypes import c_float, c_int, c_int64
import zlib

import pytest
import torch

import elementwise_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
KINDS = ["onehot", "uniform_q", "uniform_k", "random"]
EXACT_SCALE = 2.0 ** -4


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    R.print_summary(request.config)


def _abi():
    from fastvideo_b200 import _lib, ops
    return _lib.lib(), _lib.check, _lib.ptr, _lib.stream_ptr, ops._f32p, ops._i32p


def _strides(t):
    return (c_int64 * 3)(t.stride(0), t.stride(1), t.stride(2))


def _runs(rows):
    """bool [S] -> the (start, end) runs of True."""
    out, start = [], None
    for i, r in enumerate(rows.tolist() + [False]):
        if r and start is None:
            start = i
        elif not r and start is not None:
            out.append((start, i))
            start = None
    return out


class Grads:
    """dq in a [B, Sq + 2, H, 136] sentinel buffer, dk and dv in [B, Skv + 2, H, 136] ones (rows 1..S are the views), and
    the delta workspace with 32 spare elements after it."""

    def __init__(self, B, H, Sq, Skv, seed):
        self.g = [R.Guarded((B, S + 2, H, 136), torch.bfloat16, DEV, seed=seed + i) for i, S in enumerate((Sq, Skv, Skv))]
        self.dq, self.dk, self.dv = (g.buf[:, 1:S + 1, :, :128] for g, S in zip(self.g, (Sq, Skv, Skv)))
        self.dg = R.Guarded((B * H * Sq + 32,), torch.float32, DEV, seed=seed + 3)
        self.delta = self.dg.region(self.dg.buf[:B * H * Sq]).view(B, H, Sq)

    def mark(self, rows_q, rows_k):
        """rows_q / rows_k: bool [Sq] / [Skv], the rows the kernel writes."""
        for g, view, rows in zip(self.g, (self.dq, self.dk, self.dv), (rows_q, rows_k, rows_k)):
            for a, b in _runs(rows):
                g.region(view[:, a:b])

    def untouched(self, name):
        torch.cuda.synchronize()
        for g, n in zip(self.g + [self.dg], ("dq", "dk", "dv", "delta")):
            g.assert_untouched(f"{name} ({n})")


def gapped_lse(lse):
    """lse [B, H, Sq] copied into a buffer with lse_stride_h = Sq + 8, lse_stride_b = H (Sq + 8) + 16; the gaps hold 3.0."""
    B, H, Sq = lse.shape
    sh, sb = Sq + 8, H * (Sq + 8) + 16
    view = torch.full((B * sb,), 3.0, device=DEV).as_strided((B, H, Sq), (sb, sh, 1))
    view.copy_(lse)
    return view


def place(ins, layout, layout_od, gapped=True):
    """The case's q, k, v (layout) and o, dO (layout_od) copied into strided views, lse into a gapped buffer."""
    q, k, v, o, dO, lse = ins
    B, Sq, H, _ = q.shape
    Skv = k.shape[1]
    views = R.make_qkv(B, Sq, Skv, H, layout, DEV) + R.make_qkv(B, Sq, Sq, H, layout_od, DEV)[1:]
    for dst, src in zip(views, (q, k, v, o, dO)):
        dst.copy_(src)
    return (*views, gapped_lse(lse) if gapped else lse.contiguous())


def run(mode, ins, out, scale, lists=None, tiles=None):
    L, check, ptr, sp, f32p, i32p = _abi()
    q, k, v, o, dO, lse = ins
    B, Sq, H, _ = q.shape
    Skv = k.shape[1]
    heads = (ptr(q), ptr(k), ptr(v), ptr(o), ptr(dO), f32p(lse))
    grads = (ptr(out.dq), ptr(out.dk), ptr(out.dv), f32p(out.delta))
    strides = tuple(_strides(t) for t in (q, k, v, o, dO, out.dq, out.dk, out.dv))
    dims = (c_int(B), c_int(H), c_int(Sq), c_int(Skv), c_int(128), c_float(scale))
    lse_st = (c_int64(lse.stride(0)), c_int64(lse.stride(1)))
    if mode == "dense":
        check(L.fvb_attention_bwd(*heads, *lse_st, *grads, *strides, *dims, sp()))
        return
    qi, qn, ki, kn = lists["q2k"] + lists["k2q"]
    (isb, ish), (ksb, ksh) = lists["q2k_strides"], lists["k2q_strides"]
    lst = (i32p(qi), i32p(qn), c_int(qi.shape[-1]), i32p(ki), i32p(kn), c_int(ki.shape[-1]), c_int64(isb), c_int64(ish),
           c_int64(ksb), c_int64(ksh))
    t = tiles
    if mode == "blocklist":
        assert lse.is_contiguous() and t["q_off"] is None and t["kv_off"] is None
        check(L.fvb_attention_blocklist_bwd(*heads, *grads, *strides, *dims, *lst, i32p(t["kv_len"]), sp()))
        return
    check(L.fvb_attention_sparse_bwd(*heads, *lse_st, *grads, *strides, *dims, *lst, i32p(t["q_off"]), i32p(t["q_len"]),
                                     c_int(t["nqb"]), i32p(t["kv_off"]), i32p(t["kv_len"]), c_int(t["nkb"]), sp()))


def padded_lists(sel, cap, g):
    """Ascending lists of sel's rows, int32 [b, h, n, cap] with cap larger than every count, and the counts. The slots past
    a count hold a tile that row did not select: a kernel that reads past num walks a wrong tile (wrong bits), never an
    index out of range."""
    idx, num = R.block_lists(sel)
    n = sel.shape[-1]
    assert cap > n and bool((~sel).any(-1).all())
    full = torch.cat([idx, torch.full((*idx.shape[:-1], cap - n), -1, dtype=torch.int32, device=DEV)], -1)
    other = torch.rand(sel.shape, generator=g, device=DEV).masked_fill(sel, -1).argmax(-1, keepdim=True).to(torch.int32)
    pos = torch.arange(cap, device=DEV)
    return torch.where(pos < num[..., None], full, other).contiguous(), num


def make_lists(sel, g):
    """q2k lists of sel, k2q lists of its transpose (block_lists(sel^T)), each with its (batch, head) row strides."""
    b, h, nqb, nkb = sel.shape
    st = lambda n: (0 if b == 1 else h * n, 0 if h == 1 else n)
    return dict(q2k=padded_lists(sel, nkb + 3, g), k2q=padded_lists(sel.transpose(-1, -2).contiguous(), nqb + 2, g),
                q2k_strides=st(nqb), k2q_strides=st(nkb))


def bwd_select(nqb, nkb, bcast, g):
    """select_blocks (q tile 3 selects only the kv tiles 1 and 6, empty in the ragged layouts), edited so that the tile pairs
    a CTA owns have every relation of lists: q tiles 0, 1 identical, 2, 3 disjoint, 5 empty; kv tiles 0, 1 disjoint, 2, 3
    identical, 5 (50 keys in the ragged layouts) selected by no q tile."""
    sel = R.select_blocks(nqb, nkb, 3, bcast, g, DEV)
    sel[:, :, 1] = sel[:, :, 0]
    sel[:, :, 2] &= ~sel[:, :, 3]
    sel[:, :, 5] = False
    sel[:, :, :, 5] = False
    sel[:, :, :, 3] = sel[:, :, :, 2]
    sel[:, :, :, 1] = False
    sel[:, :, 3, 1] = True
    return sel


def garbage_rows(ins, q_rows, k_rows, g):
    """Rows outside every tile: randn * 1e3 in q, dO (q_rows False) and k, v (k_rows False). Large, but every dot product
    stays far from fp32 overflow."""
    q, k, v, o, dO, lse = (t.clone() for t in ins)
    for t, rows in ((q, q_rows), (dO, q_rows), (k, k_rows), (v, k_rows)):
        pad = ~rows
        t[:, pad] = R.rand_bf16(t[:, pad].shape, g, DEV, 1e3)
    return q, k, v, o, dO, lse


def _where(rows):
    idx = rows.nonzero().squeeze(1).tolist()
    return lambda i: R.bwd_coords([i[0], idx[i[1]], i[2], i[3]])


def check_case(mode, kind, ins, out, scale, visible, rows_q, rows_k, grid_q, name, walk=(None, None), **kw):
    """Run, check every written row of dq, dk, dv, delta on the rows with grid inputs (grid_q), and the sentinels; then run
    again and compare bits. Returns the written dq, dk, dv."""
    run(mode, ins, out, scale, **kw)
    out.untouched(name)
    q, k, v, o, dO, lse = ins
    got = (out.dq[:, rows_q], out.dk[:, rows_k], out.dv[:, rows_k])
    fam = f"attention bwd {mode}"
    names = ("dq", "dk", "dv")
    wh = (_where(rows_q), _where(rows_k), _where(rows_k))
    rsel = (rows_q, rows_k, rows_k)
    if kind == "random":
        bounds = R.attention_bwd_bound(q, k, v, o, dO, lse, visible, scale, *walk)
        for t, (r, b), n, w, rs in zip(got, bounds, names, wh, rsel):
            R.assert_within(t, r[:, rs], b[:, rs], f"{name} {n}", where=w, family=f"{fam} {n}")
        (dr, db) = bounds[3]
        R.assert_within(out.delta[:, :, grid_q], dr[:, :, grid_q], db[:, :, grid_q], f"{name} delta", family=f"{fam} delta")
    else:
        assert scale == EXACT_SCALE
        refs = R.bwd_exact_ref(q, k, v, o, dO, lse, visible, scale)
        for t, r, n, w, rs in zip(got, refs, names, wh, rsel):
            R.assert_exact(t, r[:, rs], f"{name} {n}", where=w, family=f"{fam} {n}")
        R.assert_exact(out.delta[:, :, grid_q], refs[3][:, :, grid_q], f"{name} delta", family=f"{fam} delta")
    first = [t.clone() for t in got] + [out.delta.clone()]
    run(mode, ins, out, scale, **kw)
    again = [out.dq[:, rows_q], out.dk[:, rows_k], out.dv[:, rows_k], out.delta]
    assert all(torch.equal(a.view(torch.int16 if a.dtype == torch.bfloat16 else torch.int32),
                           b.view(torch.int16 if b.dtype == torch.bfloat16 else torch.int32))
               for a, b in zip(first, again)), name + ": two calls differ"
    return got


# ------------------------------------------------------------------------------------------------ dense
SIZES = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257, 385, 449]
DENSE = sorted({(s, 193) for s in SIZES} | {(129, s) for s in SIZES} | {(449, 449), (65, 1)})
LAYOUTS = ["bshd", "bhsd", "fused"]


@pytest.mark.parametrize("Sq,Skv", DENSE)
def test_dense(Sq, Skv):
    """fvb_attention_bwd. Sq and Skv from 1 to 449: one to eight walked tiles against the 3-stage ring (partial ring, exact
    wrap, wrap plus partial), an odd number of owned tiles (the last CTA's second warpgroup owns nothing), tails of every
    size; B = 2, H = 3; layouts of q, k, v and of o, dO vary with the case; lse in a gapped buffer."""
    B, H = 2, 3
    i = DENSE.index((Sq, Skv))
    layout, layout_od = LAYOUTS[i % 3], LAYOUTS[(i // 3) % 3]
    visible = R.visible_mask(B, H, Sq, Skv, DEV)
    g = torch.Generator(device=DEV).manual_seed(Sq * 1000 + Skv)
    allq, allk = torch.ones(Sq, dtype=torch.bool, device=DEV), torch.ones(Skv, dtype=torch.bool, device=DEV)
    for kind in KINDS:
        scale = (128 ** -0.5 if i % 2 == 0 else EXACT_SCALE) if kind == "random" else EXACT_SCALE
        ins = place(R.bwd_inputs(kind, B, H, Sq, Skv, visible, g, DEV, scale), layout, layout_od)
        out = Grads(B, H, Sq, Skv, seed=i)
        out.mark(allq, allk)
        check_case("dense", kind, ins, out, scale, visible, allq, allk, allq, f"dense {Sq}x{Skv} {layout}/{layout_od} {kind}")


def test_dense_checkers_reject_defects_on_kernel_output():
    """The defects of the CPU self-test, edited into copies of a passing kernel output, fail the checks; so does one element
    written past the owned rows."""
    B, H, Sq, Skv = 2, 3, 129, 192
    visible = R.visible_mask(B, H, Sq, Skv, DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    allq, allk = torch.ones(Sq, dtype=torch.bool, device=DEV), torch.ones(Skv, dtype=torch.bool, device=DEV)
    for kind in KINDS:
        scale = EXACT_SCALE
        ins = place(R.bwd_inputs(kind, B, H, Sq, Skv, visible, g, DEV, scale), "bshd", "bshd")
        out = Grads(B, H, Sq, Skv, seed=9)
        out.mark(allq, allk)
        got = [t.clone() for t in check_case("dense", kind, ins, out, scale, visible, allq, allk, allq, f"mutation base {kind}")]

        def refs(vis=visible, lse=ins[5]):  # what a correct kernel would give on other lists or another lse
            a = ins[:5] + (lse,)
            if kind == "random" or lse is not ins[5]:
                return [r.bfloat16() for r, _ in R.attention_bwd_bound(*a, vis, scale)[:3]]
            return list(R.bwd_exact_ref(*a, vis, scale)[:3])

        if kind == "random":
            bounds = R.attention_bwd_bound(*ins, visible, scale)[:3]
            check = lambda outs: [R.assert_within(t, r, b, "mutant") for t, (r, b) in zip(outs, bounds)]
        else:
            exact = R.bwd_exact_ref(*ins, visible, scale)[:3]
            check = lambda outs: [R.assert_exact(t, r, "mutant") for t, r in zip(outs, exact)]

        def rejects(i, mutant):
            outs = list(got)
            outs[i] = mutant
            with pytest.raises(AssertionError):
                check(outs)

        live = [bool((t != 0).any()) for t in got]  # uniform-q: dk = 0; uniform-k: dq = 0
        vis = visible.clone()
        vis[1, 2, 64:128, 64:128] = False  # one key tile missing from one dQ tile, one q tile from one dK / dV tile
        for i, m in enumerate(refs(vis)):
            if live[i]:
                t = got[i].clone()
                t[1, 64:128, 2] = m[1, 64:128, 2]
                rejects(i, t)
        for i, t in enumerate(got):
            if not live[i] or (kind.startswith("uniform") and i == 2):
                continue  # uniform: every dv row of a head sums the same rows
            shifted = t.clone()
            shifted[1, 70] = t[1, 71]
            rejects(i, shifted)
            head = t.clone()
            head[0, 64:128, 1] = t[0, 64:128, 2]
            rejects(i, head)
        if kind.startswith("uniform"):  # one masked key counted: the kernel's output against a reference without it
            vis = visible.clone()
            vis[1, 2, 100, 5] = False
            m = refs(vis)
            for i in (0 if kind == "uniform_q" else 1, 2):
                with pytest.raises(AssertionError):
                    R.assert_exact(got[i], m[i], "mutant")
        else:  # an lse off by 0.25 in one row
            lse = ins[5].clone()
            lse[0, 1, 40] += 0.25
            m = refs(lse=lse)
            rejects(0, m[0])
            rejects(2, m[2])
        out.g[0].buf.view(torch.int16)[0, Sq + 1, 0, 0] ^= 1  # one dq element past the last owned row
        with pytest.raises(AssertionError):
            out.untouched("mutant")


# ------------------------------------------------------------------------------------------------ block modes
KV_LEN = [64, 0, 37, 64, 1, 50, 0]
Q_LEN = [64, 30, 64, 1, 64, 63, 17]
GAP = [3, 0, 5, 8, 0, 1, 2]  # "both": rows between tiles that belong to none


def tile_layout(addressing, nqb, nkb):
    """The tile tables of one addressing: "none" (64-row tiles, ragged last tile), "len" (padded: q_len / kv_len), "off"
    (compact: q_off / kv_off) or "both" (off and len, with gaps between tiles). Returns Sq, Skv, the tables for run(), and
    the first row and valid rows of every tile."""
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    cum = lambda w: [0] + torch.tensor(w).cumsum(0).tolist()
    if addressing == "none":
        Sq, Skv = 64 * (nqb - 1) + 17, 64 * (nkb - 1) + 50
        qo, ko = [64 * i for i in range(nqb)], [64 * i for i in range(nkb)]
        ql, kl = [min(64, Sq - o) for o in qo], [min(64, Skv - o) for o in ko]
        t = dict(q_off=None, q_len=None, kv_off=None, kv_len=None)
    elif addressing == "len":
        Sq, Skv = 64 * nqb, 64 * nkb
        qo, ko, ql, kl = [64 * i for i in range(nqb)], [64 * i for i in range(nkb)], Q_LEN, KV_LEN
        t = dict(q_off=None, q_len=i32(Q_LEN), kv_off=None, kv_len=i32(KV_LEN))
    elif addressing == "off":
        qo, ko, ql, kl = cum(Q_LEN), cum(KV_LEN), Q_LEN, KV_LEN
        Sq, Skv = qo[-1], ko[-1]
        t = dict(q_off=i32(qo), q_len=None, kv_off=i32(ko), kv_len=None)
    else:
        qo = cum([a + b for a, b in zip(Q_LEN, GAP)])
        ko = cum([a + b for a, b in zip(KV_LEN, GAP[::-1])])
        ql, kl, Sq, Skv = Q_LEN, KV_LEN, qo[-1], ko[-1]
        t = dict(q_off=i32(qo), q_len=i32(Q_LEN), kv_off=i32(ko), kv_len=i32(KV_LEN))
    t.update(nqb=nqb, nkb=nkb)
    return Sq, Skv, t, (qo[:nqb], ql), (ko[:nkb], kl)


def _block_case(kind, addressing, bcast, g, B=2, H=3, nqb=7, nkb=7):
    Sq, Skv, tiles, (qo, ql), (ko, kl) = tile_layout(addressing, nqb, nkb)
    q_block, kv_block = R.block_of_rows(Sq, qo, ql, DEV), R.block_of_rows(Skv, ko, kl, DEV)
    sel = bwd_select(nqb, nkb, bcast, g)
    visible = R.visible_mask(B, H, Sq, Skv, DEV, q_block, kv_block, sel)
    scale = 128 ** -0.5 if kind == "random" else EXACT_SCALE
    ins = R.bwd_inputs(kind, B, H, Sq, Skv, visible, g, DEV, scale)
    ins = garbage_rows(ins, q_block >= 0, kv_block >= 0, g)
    return ins, sel, visible, scale, tiles, q_block, kv_block


@pytest.mark.parametrize("addressing", ["none", "len", "off", "both"])
@pytest.mark.parametrize("bcast", ["none", "batch", "both"])
def test_sparse(addressing, bcast):
    """fvb_attention_sparse_bwd in all four tile addressings, index lists broadcast over nothing, batch or both; odd nqb and
    nkb; ragged tiles with empty kv tiles; q tile 3 sees only empty kv tiles (lse = -inf, dq exactly 0); kv tile 5 is
    selected by none (dk, dv written as zeros); owned tile pairs with identical, disjoint and empty lists; lists longer than
    their counts, the spare slots holding unselected tiles; rows outside every tile hold garbage in q, dO, k, v, and their
    dq, dk, dv keep their sentinels."""
    B, H, nqb, nkb = 2, 3, 7, 7
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"sparse/{addressing}/{bcast}".encode()))
    for kind in KINDS:
        ins, sel, visible, scale, tiles, q_block, kv_block = _block_case(kind, addressing, bcast, g)
        Sq, Skv = q_block.numel(), kv_block.numel()
        rows_q, rows_k = q_block >= 0, kv_block >= 0
        ins = place(ins, "bshd", "bhsd")
        out = Grads(B, H, Sq, Skv, seed=len(kind))
        out.mark(rows_q, rows_k)
        name = f"sparse {addressing} bcast={bcast} {kind}"
        check_case("sparse", kind, ins, out, scale, visible, rows_q, rows_k, rows_q, name, walk=(64 * nqb, 64 * nkb),
                   lists=make_lists(sel, g), tiles=tiles)
        if addressing != "none":
            assert bool((out.dq[:, q_block == 3] == 0).all()) and bool(torch.isneginf(ins[5][:, :, q_block == 3]).all()), name
        assert bool((out.dk[:, kv_block == 5] == 0).all() and (out.dv[:, kv_block == 5] == 0).all()), name
        assert bool((kv_block == 5).any()), name


@pytest.mark.parametrize("bcast", ["none", "batch", "both"])
def test_blocklist(bcast):
    """fvb_attention_blocklist_bwd (padded layout, Sq and Skv multiples of 64): ragged kv_len with 0 and 1, pad q rows with
    lse = -inf and garbage q / dO (dk, dv unaffected, dq pad rows 0), broadcast index strides, empty lists. The same inputs
    through fvb_attention_sparse_bwd with q_len / kv_len give the same bits on the exact constructions."""
    B, H, nqb, nkb = 2, 3, 7, 7
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"blocklist/{bcast}".encode()))
    for kind in KINDS:
        ins, sel, visible, scale, tiles, q_block, kv_block = _block_case(kind, "len", bcast, g)
        Sq, Skv = q_block.numel(), kv_block.numel()
        lists = make_lists(sel, g)
        allq, allk = torch.ones(Sq, dtype=torch.bool, device=DEV), torch.ones(Skv, dtype=torch.bool, device=DEV)
        name = f"blocklist bcast={bcast} {kind}"
        a = place(ins, "fused", "bshd", gapped=False)
        out = Grads(B, H, Sq, Skv, seed=3)
        out.mark(allq, allk)
        got = check_case("blocklist", kind, a, out, scale, visible, allq, allk, q_block >= 0, name,
                         walk=(64 * nqb, 64 * nkb), lists=lists, tiles=tiles)
        assert bool((out.dq[:, q_block < 0] == 0).all()), name + ": dq pad rows must be 0"
        if kind == "random":
            continue
        b = place(ins, "fused", "bshd")
        out2 = Grads(B, H, Sq, Skv, seed=4)
        rows_q, rows_k = q_block >= 0, kv_block >= 0
        out2.mark(rows_q, rows_k)
        got2 = check_case("sparse", kind, b, out2, scale, visible, rows_q, rows_k, rows_q, name + " (sparse_bwd)",
                          walk=(64 * nqb, 64 * nkb), lists=lists, tiles=tiles)
        for x, y, rs in zip(got, got2, (rows_q, rows_k, rows_k)):
            assert torch.equal(x[:, rs].view(torch.int16), y.view(torch.int16)), name + ": the two backward kernels differ"


def test_entry_points_agree_on_a_shared_case():
    """Every pair selected, Sq and Skv multiples of 64: fvb_attention_bwd, fvb_attention_sparse_bwd (64-row tiles) and
    fvb_attention_blocklist_bwd all equal the exact reference, and so each other, bit for bit."""
    B, H, Sq, Skv = 2, 3, 192, 320
    nqb, nkb = Sq // 64, Skv // 64
    g = torch.Generator(device=DEV).manual_seed(17)
    visible = R.visible_mask(B, H, Sq, Skv, DEV)
    sel = torch.ones(1, H, nqb, nkb, dtype=torch.bool, device=DEV)
    # every tile selected: the spare list slots repeat a selected tile (there is no other), which the counts exclude
    qi = torch.arange(nkb, dtype=torch.int32, device=DEV).expand(1, H, nqb, nkb).contiguous()
    ki = torch.arange(nqb, dtype=torch.int32, device=DEV).expand(1, H, nkb, nqb).contiguous()
    lists = dict(q2k=(qi, sel.sum(-1).int()), k2q=(ki, sel.sum(-2).int()), q2k_strides=(0, nqb), k2q_strides=(0, nkb))
    tiles = dict(q_off=None, q_len=None, kv_off=None, kv_len=None, nqb=nqb, nkb=nkb)
    allq, allk = torch.ones(Sq, dtype=torch.bool, device=DEV), torch.ones(Skv, dtype=torch.bool, device=DEV)
    for kind in KINDS[:3]:
        ins = R.bwd_inputs(kind, B, H, Sq, Skv, visible, g, DEV, EXACT_SCALE)
        res = []
        for mode in ("dense", "sparse", "blocklist"):
            a = place(ins, "bhsd", "fused", gapped=mode != "blocklist")
            out = Grads(B, H, Sq, Skv, seed=11)
            out.mark(allq, allk)
            res.append(check_case(mode, kind, a, out, EXACT_SCALE, visible, allq, allk, allq, f"shared {mode} {kind}",
                                  lists=lists, tiles=tiles))
        for other in res[1:]:
            assert all(torch.equal(x.view(torch.int16), y.view(torch.int16)) for x, y in zip(res[0], other)), kind
