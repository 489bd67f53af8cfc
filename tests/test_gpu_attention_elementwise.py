"""GPU: the bf16 attention forward (fvb_attention_fwd dense and pair-schedule modes, fvb_attention_blocklist_fwd) element by
element: the uniform and one-hot constructions bit for bit, random inputs against fp64 element bounds
(tests/elementwise_ref.py); o and LSE written into sentinel buffers with gaps; two calls give the same bits."""
from ctypes import c_float, c_int, c_int64
import zlib

import pytest
import torch

import elementwise_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    R.print_summary(request.config)


def _abi():
    from fastvideo_b200 import _lib, ops
    return _lib.lib(), _lib.check, _lib.ptr, _lib.stream_ptr, ops._f32p, ops._i32p


def _strides(t):
    return (c_int64 * 3)(t.stride(0), t.stride(1), t.stride(2))


class Outputs:
    """o in a [B, Sq + 2, H, 136] sentinel buffer (gaps between tokens and heads), LSE in a buffer with
    lse_stride_h = Sq + 8 and lse_stride_b = H (Sq + 8) + 16."""

    def __init__(self, B, Sq, H, seed):
        self.og = R.Guarded((B, Sq + 2, H, 136), torch.bfloat16, DEV, seed=seed)
        self.o = self.og.buf[:, 1:Sq + 1, :, :128]
        self.sh, self.sb = Sq + 8, H * (Sq + 8) + 16
        self.lg = R.Guarded((B * self.sb,), torch.float32, DEV, seed=seed + 1)
        self.lse = self.lg.buf.as_strided((B, H, Sq), (self.sb, self.sh, 1))

    def mark_rows(self, rows):
        """rows: bool [Sq], the q rows the kernel writes."""
        for r in rows.nonzero().squeeze(1).tolist():
            self.og.region(self.o[:, r])
            self.lg.region(self.lse[:, :, r])

    def untouched(self, name):
        torch.cuda.synchronize()
        self.og.assert_untouched(name + " (o)")
        self.lg.assert_untouched(name + " (lse)")


def run(mode, q, k, v, out, scale, sel=None, q_off=None, q_len=None, kv_off=None, kv_len=None, nqb=0, nkb=0):
    L, check, ptr, sp, f32p, i32p = _abi()
    B, Sq, H, _ = q.shape
    Skv = k.shape[1]
    common = (ptr(q), ptr(k), ptr(v), ptr(out.o), f32p(out.lse), _strides(q), _strides(k), _strides(v), _strides(out.o),
              c_int64(out.sb), c_int64(out.sh), c_int(B), c_int(H), c_int(Sq), c_int(Skv), c_int(128), c_float(scale))
    if mode == "dense":
        check(L.fvb_attention_fwd(*common, i32p(None), i32p(None), c_int64(0), c_int64(0), c_int(0), c_int(0), i32p(None),
                                  i32p(None), c_int(0), i32p(None), i32p(None), c_int(0), sp()))
        return
    sb_, sh_ = sel.shape[:2]
    if mode == "pairs":
        sched, cnt = pair_schedule(sel)
        npairs, cap = sched.shape[2:]
        check(L.fvb_attention_fwd(*common, i32p(sched), i32p(cnt), c_int64(0 if sb_ == 1 else sh_ * npairs),
                                  c_int64(0 if sh_ == 1 else npairs), c_int(cap), c_int(npairs), i32p(q_off), i32p(q_len),
                                  c_int(nqb), i32p(kv_off), i32p(kv_len), c_int(nkb), sp()))
        return
    idx, num = R.block_lists(sel)
    cap = idx.shape[-1]
    ws = torch.empty(256, dtype=torch.uint8, device=DEV)
    check(L.fvb_attention_blocklist_fwd(*common, i32p(idx), i32p(num), c_int64(0 if sb_ == 1 else sh_ * nqb),
                                        c_int64(0 if sh_ == 1 else nqb), c_int(cap), i32p(q_off), i32p(q_len), c_int(nqb),
                                        i32p(kv_off), i32p(kv_len), c_int(nkb), ptr(ws), c_int64(256), sp()))


def pair_schedule(sel):
    """The pair-union schedule of fvb_pair_schedule, built here: entry kv_block | flags << 24 over the ascending union of
    q blocks 2p and 2p + 1."""
    b, h, nq, nk = sel.shape
    npairs = (nq + 1) // 2
    pad = torch.zeros(b, h, 2 * npairs, nk, dtype=torch.bool, device=sel.device)
    pad[:, :, :nq] = sel
    pr = pad.view(b, h, npairs, 2, nk)
    flags = pr[:, :, :, 0].int() | (pr[:, :, :, 1].int() << 1)
    union = flags > 0
    entry = torch.arange(nk, device=sel.device, dtype=torch.int32) | (flags << 24)
    key = torch.where(union, torch.arange(nk, device=sel.device), nk)
    order = key.sort(-1).indices
    sched = entry.gather(-1, order).masked_fill(~union.gather(-1, order), 0)
    return sched.to(torch.int32).contiguous(), union.sum(-1).to(torch.int32).contiguous()


def fill(q, k, v, kind, visible, g):
    """Write one construction into the q, k, v views."""
    B, Sq, H, _ = q.shape
    Skv = k.shape[1]
    if kind == "uniform":
        q.zero_()
        k.copy_(R.rand_bf16(k.shape, g, DEV))
        v.copy_(R.grid_bf16(v.shape, g, DEV))
    elif kind == "onehot":
        qq, kk, _ = R.onehot_qk(B, H, Sq, Skv, visible, g, DEV)
        q.copy_(qq)
        k.copy_(kk)
        v.copy_(R.grid_bf16(v.shape, g, DEV))
    else:
        for t in (q, k, v):
            t.copy_(R.rand_bf16(t.shape, g, DEV))


def check_case(mode, kind, q, k, v, out, scale, visible, written, name, **kw):
    """Run, check every written element and the sentinels, then run again and compare bits."""
    run(mode, q, k, v, out, scale, **kw)
    out.untouched(name)
    w = written
    o, lse = out.o[:, w], out.lse[:, :, w]
    if kind == "random":
        oref, ob, lref, lb = R.attention_bound(q, k, v, visible, scale)
        R.assert_within(o, oref[:, w], ob[:, w], name + " o", family=f"attention {mode} o")
        R.assert_lse_within(lse, lref[:, :, w], lb[:, :, w], name + " lse", family=f"attention {mode} lse")
    else:
        oref, lref, cnt = R.tie_attention_ref(q, k, v, visible, scale)
        if kind == "onehot":  # exactly one winning key in every row that sees a key
            c = cnt[:, :, w]
            assert bool((c[c > 0] == 1).all()), name + ": one-hot construction has ties"
        R.assert_exact(o, oref[:, w], name + " o", family=f"attention {mode} o")
        R.assert_lse_tie(lse, lref[:, :, w], cnt[:, :, w], name + " lse", family=f"attention {mode} lse")
    o1, l1 = o.clone(), lse.clone()
    run(mode, q, k, v, out, scale, **kw)
    assert torch.equal(out.o[:, w], o1) and torch.equal(out.lse[:, :, w].view(torch.int32), l1.view(torch.int32)), \
        name + ": two calls differ"
    return oref


# ------------------------------------------------------------------------------------------------ dense
SIZES = [1, 63, 64, 65, 127, 128, 129, 257]
DENSE = sorted({(s, 257) for s in SIZES} | {(129, s) for s in SIZES} | {(63, 65), (257, 1)})
LAYOUTS = ["bshd", "bhsd", "fused"]


@pytest.mark.parametrize("Sq,Skv", DENSE)
def test_dense(Sq, Skv):
    """B = 2, H = 3, each (b, h) with its own content; the layout and softmax_scale vary with the case."""
    B, H = 2, 3
    i = DENSE.index((Sq, Skv))
    layout, scale = LAYOUTS[i % 3], (128 ** -0.5 if i % 2 == 0 else 0.0625)
    q, k, v = R.make_qkv(B, Sq, Skv, H, layout, DEV)
    visible = R.visible_mask(B, H, Sq, Skv, DEV)
    g = torch.Generator(device=DEV).manual_seed(Sq * 1000 + Skv)
    for kind in ("uniform", "onehot", "random"):
        fill(q, k, v, kind, visible, g)
        out = Outputs(B, Sq, H, seed=i)
        out.mark_rows(torch.ones(Sq, dtype=torch.bool, device=DEV))
        check_case("dense", kind, q, k, v, out, scale, visible, slice(None), f"dense {Sq}x{Skv} {layout} {kind}")


def test_dense_checkers_reject_defects_on_kernel_output():
    B, H, Sq, Skv = 2, 3, 129, 128
    q, k, v = R.make_qkv(B, Sq, Skv, H, "bshd", DEV)
    visible = R.visible_mask(B, H, Sq, Skv, DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    for kind in ("uniform", "onehot", "random"):
        fill(q, k, v, kind, visible, g)
        out = Outputs(B, Sq, H, seed=9)
        out.mark_rows(torch.ones(Sq, dtype=torch.bool, device=DEV))
        check_case("dense", kind, q, k, v, out, 128 ** -0.5, visible, slice(None), f"mutation base {kind}")
        o, lse = out.o.clone(), out.lse.clone()
        if kind == "random":
            oref, ob, lref, lb = R.attention_bound(q, k, v, visible, 128 ** -0.5)
            chk_o = lambda t: R.assert_within(t, oref, ob, "mutant")
            chk_l = lambda t: R.assert_lse_within(t, lref, lb, "mutant")
        else:
            oref, lref, cnt = R.tie_attention_ref(q, k, v, visible, 128 ** -0.5)
            chk_o = lambda t: R.assert_exact(t, oref, "mutant")
            chk_l = lambda t: R.assert_lse_tie(t, lref, cnt, "mutant")
        shifted = o.clone()
        shifted[1, 70] = o[1, 71]  # a row shifted by one (uniform rows of one head are equal by construction)
        head = o.clone()
        head[0, 64:128, 1] = o[0, 64:128, 2]  # one q block reading the neighbouring head
        for mutant in (head,) if kind == "uniform" else (shifted, head):
            with pytest.raises(AssertionError):
                chk_o(mutant)
        if kind == "uniform":
            # one masked key counted in one row: the row averages one more key
            vis = visible.clone()
            vis[1, 2, 100, 5] = False
            oref2, lref2, cnt2 = R.tie_attention_ref(q, k, v, vis, 128 ** -0.5)
            with pytest.raises(AssertionError):
                R.assert_exact(o, oref2, "mutant")
            with pytest.raises(AssertionError):
                R.assert_lse_tie(lse, lref2, cnt2, "mutant")
        lm = lse.clone()
        lm[0, 0, 3] = lse[0, 0, 3] + 0.25
        with pytest.raises(AssertionError):
            chk_l(lm)
        out.lg.buf.view(torch.int32)[Sq] ^= 1  # one LSE element written past Sq (b 0, h 0)
        with pytest.raises(AssertionError):
            out.untouched("mutant")


# ------------------------------------------------------------------------------------------------ block modes
KV_LEN = [64, 0, 37, 64, 1, 50, 0]
Q_LEN = [64, 30, 64, 1, 64, 63, 17]  # padded layout: rows past q_len keep their sentinels


@pytest.mark.parametrize("mode", ["blocklist", "pairs"])
@pytest.mark.parametrize("layout", ["padded", "compact"])
@pytest.mark.parametrize("bcast", ["none", "batch", "both"])
def test_block_modes(mode, layout, bcast):
    """Ragged kv_len with empty kv blocks, a q block whose every selected block is empty (zeros, -inf), q_len < 64 (padded:
    rows past it keep their sentinels; compact: q_off / kv_off), odd nqb (the last CTA has one q block), index strides
    broadcast over batch and heads."""
    B, H, nqb, nkb = 2, 3, 7, 7
    kv_len = torch.tensor(KV_LEN, dtype=torch.int32, device=DEV)
    if layout == "padded":
        Sq, Skv = 64 * nqb, 64 * nkb
        q_offs, kv_offs = [64 * i for i in range(nqb)], [64 * i for i in range(nkb)]
        q_len = torch.tensor(Q_LEN, dtype=torch.int32, device=DEV)
        kw = dict(q_len=q_len, kv_len=kv_len)
    else:
        q_offs = [0] + torch.tensor(Q_LEN).cumsum(0).tolist()
        kv_offs = [0] + torch.tensor(KV_LEN).cumsum(0).tolist()
        Sq, Skv = q_offs[-1], kv_offs[-1]
        kw = dict(q_off=torch.tensor(q_offs, dtype=torch.int32, device=DEV),
                  kv_off=torch.tensor(kv_offs, dtype=torch.int32, device=DEV))
    kw.update(nqb=nqb, nkb=nkb)
    q_block = R.block_of_rows(Sq, q_offs, Q_LEN, DEV)
    kv_block = R.block_of_rows(Skv, kv_offs, KV_LEN, DEV)
    written = q_block >= 0
    # a fixed seed per case (str hashes change from one interpreter to the next): a failure replays with the same inputs
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(f"{mode}/{layout}/{bcast}".encode()))
    for kind, topk in (("uniform", 3), ("onehot", 3), ("random", 3)):
        sel = R.select_blocks(nqb, nkb, topk, bcast, g, DEV)
        visible = R.visible_mask(B, H, Sq, Skv, DEV, q_block, kv_block, sel)
        q, k, v = R.make_qkv(B, Sq, Skv, H, "bshd", DEV)
        fill(q, k, v, kind, visible, g)
        out = Outputs(B, Sq, H, seed=topk)
        out.mark_rows(written)
        name = f"{mode} {layout} bcast={bcast} {kind}"
        check_case(mode, kind, q, k, v, out, 128 ** -0.5, visible, written, name, sel=sel, **kw)
        qb3 = written & (q_block == 3)
        assert bool((out.o[:, qb3] == 0).all()) and bool(torch.isneginf(out.lse[:, :, qb3]).all()), name
