"""GPU: the row kernels of csrc/elementwise.cu element by element, through the C ABI (tests/elementwise_ref.py, "Row
kernels"): forward rows bit for bit on exact rows against every rstd the kernel may compute, the backward column sums
bit for bit against a replay of their fixed order, and everything else against fp64 element bounds on random rows.
Outputs go into sentinel buffers with row gaps and rows before and after; inputs the kernels must not read (gaps between
modulation groups, columns past D, unselected table rows) hold NaN; workspaces get exactly the reported bytes inside a
NaN-filled guard; every case runs twice and must give the same bits. `ln_path`, `rms_path` and `bwd_path` mirror each entry
point's launch choices, so a CPU test can assert that the case lists reach every path."""
from ctypes import c_float, c_int, c_int64
import zlib

import pytest
import torch

import elementwise_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
EPS = 1e-6
NAN = float("nan")
SMEM_BUDGET, SMEM_MAX = 192 * 1024, 226 * 1024
H100_SMS = 132


# ------------------------------------------------------------------------------------------------ launch choices
def ln_path(M, D, x_f32, w, scale, mod_rows, sms=H100_SMS):
    """fvb_layernorm_modulate's choice: the warp-per-row kernel (nw warps, stages, tab_kind, grid) or one CTA per row."""
    row_bytes = D * (4 if x_f32 else 2)
    nw = min(16, SMEM_BUDGET // row_bytes)
    if not (M >= 256 and nw >= 8):
        return dict(warp=False, chunks=-(-D // 2048))
    stages = max(1, min(2, SMEM_BUDGET // (nw * row_bytes)))
    tab = 0
    if nw * stages * row_bytes + D * 8 <= SMEM_MAX:
        tab = 2 if scale and (mod_rows == 0 or mod_rows >= M) else (1 if w else 0)
    grid = min(-(-M // nw), sms)
    return dict(warp=True, nw=nw, stages=stages, tab_kind=tab, grid=grid, wraps=-(-M // (grid * nw)),
                ragged=M % (grid * nw) != 0)


def rms_path(M, D, head_dim, f64, scatter=False, sms=H100_SMS):
    """fvb_rmsnorm_rope(_scatter)'s choice: warp kernel (stages, w_tab, table row hoisted when head_dim | 256) or CTA per
    row (table slice hoisted when head_dim | 2048)."""
    if scatter or (M >= 256 and 16 * D * 2 <= SMEM_BUDGET):
        stages = max(1, min(2, SMEM_BUDGET // (16 * D * 2)))
        return dict(warp=True, stages=stages, w_tab=int(16 * stages * D * 2 + D * 4 <= SMEM_MAX),
                    hoisted=not f64 and 256 % head_dim == 0, grid=min(-(-M // 16), sms))
    return dict(warp=False, hoisted=not f64 and 2048 % head_dim == 0, chunks=-(-D // 2048))


def bwd_path(kind, M, N, R_=None):
    """Row sets of the backward column sums: ctas (block per row, 528) or parts (256) and, grouped, G and P."""
    if kind in ("rms", "ln"):
        return dict(ctas=min(M, R.RB_CTAS), chunks=-(-N // 2048))
    if kind in ("bias", "gate"):
        return dict(parts=min(M, R.BG_PARTS), col_blocks=-(-N // 1024), unrolled=M > 7 * min(M, R.BG_PARTS))
    G = -(-M // R_)
    P = R.grouped_parts(M, R_, R.RB_CTAS if kind == "ln_grouped" else R.BG_PARTS)
    last = M - (G - 1) * R_
    return dict(G=G, P=P, last=last, empty_parts=last < P)


# ------------------------------------------------------------------------------------------------ buffers
def _abi():
    from fastvideo_b200 import _lib
    return _lib.lib(), _lib.check, _lib.ptr, _lib.stream_ptr


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def nan_rows(t, gap=8, extra=1):
    """t [M, D] copied into a NaN-filled [M + 2 extra, D + gap] buffer (rows extra.., columns ..D); returns the view."""
    M, D = t.shape
    buf = torch.full((M + 2 * extra, D + gap), NAN, dtype=t.dtype, device=DEV)
    v = buf[extra:extra + M, :D]
    v.copy_(t)
    return v


def nan_groups(vec, G, stride):
    """Per-group vectors [G, D] in a NaN-filled [G, stride] buffer."""
    buf = torch.full((G, stride), NAN, dtype=torch.float32, device=DEV)
    buf[:, :vec.shape[1]] = vec
    return buf


class Out:
    """An output [M, D] view with row stride D + gap inside a guarded buffer with one row before and after."""

    def __init__(self, M, D, dtype, seed, gap=16):
        self.g = R.Guarded((M + 2, D + gap), dtype, DEV, seed=seed)
        self.v = self.g.region(self.g.buf[1:M + 1, :D])
        self.ld = D + gap


class Workspace:
    """Exactly nbytes of fp32 workspace at the start of a NaN-filled guard with 64 spare elements."""

    def __init__(self, nbytes):
        assert nbytes % 16 == 0
        self.n = nbytes // 4
        self.g = R.Guarded((self.n + 64,), torch.float32, DEV, fill=NAN)
        self.v = self.g.region(self.g.buf[:self.n])
        self.bytes = nbytes

    def check(self, name, used=None):
        """Nothing written past the workspace, and every partial that is read (the first `used` elements) written."""
        self.g.assert_untouched(f"{name} (workspace)")
        assert bool(torch.isfinite(self.v[:used]).all()), f"{name}: a workspace partial was left unwritten"


def twice(run, outs, name):
    """Run twice; the outputs (tensors) must have the same bits both times. Returns the second run's outputs."""
    run()
    first = [o.clone() for o in outs]
    run()
    torch.cuda.synchronize()
    for a, b in zip(first, outs):
        it = R._INT_VIEW[a.dtype]
        assert torch.equal(a.view(it), b.view(it)), f"{name}: two calls differ"
    return outs


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def _f32p(t):
    from fastvideo_b200 import ops
    return ops._f32p(t)


# ------------------------------------------------------------------------------------------------ LayerNorm forward
# (M, D, x_f32, affine, mod, mod_rows, round_ln, hidden)
LN_CASES = [
    (300, 1536, False, False, True, 0, 1, True),  # warp, 16 warps, 2 stages, tab 2
    (32760, 1536, True, False, True, 0, 0, True),  # Wan 1.3B 480p x 81 frames: persistent rows, ragged last wrap
    (5000, 5120, True, True, False, 0, 0, False),  # nw 9, 1 stage, tab 1, ragged
    (600, 8192, False, False, True, 0, 1, False),  # nw 12, tab 0
    (400, 6144, True, True, True, 0, 0, False),  # nw 8, tab 2 does not fit: tab 0
    (300, 8192, True, True, False, 0, 0, True),  # fp32 D 8192: nw 6 < 8 -> block path, 4 chunks
    (1000, 264, False, False, True, 333, 3, True),  # R not dividing M, bf16 modulation, tab 0
    (2048, 256, False, True, True, 0, 1, False),  # affine + modulation, tab 2
    (2047, 2048, False, True, False, 0, 0, True),  # tab 1
    (777, 2056, False, False, True, 1, 3, False),  # one modulation row per token
    (520, 1536, False, False, True, 1000, 1, False),  # mod_rows >= M: tab 2
    (77, 8, False, True, True, 0, 1, True),  # block, 1 chunk
    (129, 2056, True, False, True, 40, 0, False),  # block, 2 chunks, grouped modulation
    (255, 5120, False, False, True, 64, 3, True),  # block, 3 chunks
    (200, 2048, False, True, False, 0, 0, False),  # block, D a power of two
    (1, 1536, False, False, True, 0, 1, False),
]


def _ln_inputs(case, kind):
    M, D, x_f32, affine, mod, R_, round_ln, hidden = case
    g = _gen("ln", case, kind)
    if kind == "exact":
        x, c, qz, _ = R.exact_rows(M, D, g, DEV)
    else:
        x = torch.randn(M, D, generator=g, device=DEV) * 2 + torch.randn(M, 1, generator=g, device=DEV)
        c = qz = None
    x = x if x_f32 else x.bfloat16()
    w = b = scale = shift = None
    if affine:
        w, b = (torch.randn(D, generator=g, device=DEV) * 0.5 + 1), torch.randn(D, generator=g, device=DEV) * 0.5
    G = -(-M // R_) if R_ else 1
    if mod:
        scale, shift = (torch.randn(G, D, generator=g, device=DEV) * 0.5 for _ in range(2))
        if round_ln & 2:  # fp32 copies of bf16 values
            scale, shift = scale.bfloat16().float(), shift.bfloat16().float()
    return x, c, qz, w, b, scale, shift, G


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("case", LN_CASES, ids=lambda c: "-".join(map(str, c)))
def test_layernorm_modulate(case, kind):
    M, D, x_f32, affine, mod, R_, round_ln, hidden = case
    L, check, ptr, sp = _abi()
    x, c, qz, w, b, scale, shift, G = _ln_inputs(case, kind)
    xv = nan_rows(x)
    stride = D + 4 if R_ else 0
    sc = nan_groups(scale, G, D + 4) if mod else None
    sh = nan_groups(shift, G, D + 4) if mod else None
    out, hid = Out(M, D, torch.bfloat16, 1), (Out(M, D, torch.bfloat16, 2, gap=24) if hidden else None)
    path = ln_path(M, D, x_f32, affine, mod, R_, sms())

    def run():
        check(L.fvb_layernorm_modulate(ptr(xv), c_int(int(x_f32)), c_int64(xv.stride(0)), ptr(w), ptr(b), ptr(sc), ptr(sh),
                                       c_int(R_), c_int64(stride), c_int(round_ln), ptr(out.v), c_int64(out.ld),
                                       ptr(hid.v if hidden else None), c_int64(hid.ld if hidden else 0), c_int(M), c_int(D),
                                       c_float(EPS), sp()))

    twice(run, [out.v] + ([hid.v] if hidden else []), "layernorm_modulate")
    out.g.assert_untouched("out")
    if hidden:
        hid.g.assert_untouched("hidden_out")
        R.assert_exact(hid.v, x.bfloat16(), "hidden_out", lambda i: R.row_coords(*i), family="layernorm fwd (exact)")
    grp = (torch.arange(M, device=DEV) // R_) if R_ else torch.zeros(M, dtype=torch.int64, device=DEV)
    scr, shr = (scale[grp], shift[grp]) if mod else (None, None)
    where = lambda r, col: R.row_coords(r, col, path.get("nw"), path.get("grid"))
    if kind == "exact":
        cands = R.rstd_candidates(R.var_forms(qz, D, EPS, path["warp"]))
        chain = lambda r: R.ln_chain(x, c, r, w, b, scr, shr, round_ln)
        hit = R.assert_rows_match(out.v, chain, cands, f"layernorm {path}", where, family="layernorm fwd (exact)")
        if path["warp"] and D & (D - 1) == 0:  # exact statistics: the block path must give the same bits
            m = min(M, 255)
            blk = Out(m, D, torch.bfloat16, 3)
            check(L.fvb_layernorm_modulate(ptr(xv), c_int(int(x_f32)), c_int64(xv.stride(0)), ptr(w), ptr(b), ptr(sc),
                                           ptr(sh), c_int(R_), c_int64(stride), c_int(round_ln), ptr(blk.v),
                                           c_int64(blk.ld), None, c_int64(0), c_int(m), c_int(D), c_float(EPS), sp()))
            torch.cuda.synchronize()
            R.assert_exact(blk.v, out.v[:m], "block path vs warp path", lambda i: R.row_coords(*i),
                           family="layernorm fwd (exact)")
        return
    ref, bound = R.ln_fwd_bound(x.float(), EPS, w, b, scr, shr, round_ln)
    R.assert_within(out.v, ref, bound, f"layernorm {path}", lambda i: where(*i), family="layernorm fwd (random)")


# ------------------------------------------------------------------------------------------------ RMSNorm + RoPE forward
# (M, D, head_dim, two tensors, f64 tables, fp32 w, rope_row: none / perm, col_offsets)
RMS_CASES = [
    (300, 1536, 128, True, False, False, "none", False),  # warp, 2 stages, table row hoisted
    (9450, 5120, 128, True, False, False, "perm", False),  # warp, 1 stage
    (100, 1536, 64, False, False, False, "perm", False),  # block, hoisted
    (300, 1536, 96, True, False, False, "perm", False),  # not hoisted in either kernel
    (120, 1536, 96, False, False, False, "none", False),
    (300, 1536, 24, False, False, False, "perm", False),
    (60, 1536, 192, True, False, False, "perm", False),
    (300, 1536, 512, False, False, False, "perm", False),  # hoisted in the block kernel only
    (100, 1536, 512, False, False, False, "none", False),
    (300, 1536, 128, True, True, False, "perm", False),  # float64 tables
    (50, 1536, 128, False, True, False, "perm", False),
    (300, 1536, 128, False, False, True, "perm", False),  # fp32 weights
    (40, 3072, 128, True, False, True, "none", False),
    (300, 1536, 128, True, False, False, "perm", True),  # head-scattered rows
    (200, 1536, 128, False, False, False, "none", True),
    (300, 8192, 128, False, False, False, "perm", False),  # too wide for the warp kernel
]


def _tables(S, hd, f64, g, sel):
    """cos / sin [S + 2, hd] (NaN in every row sel does not select, and in the extra rows)."""
    ang = torch.rand(S, hd // 2, generator=g, device=DEV, dtype=torch.float64) * 6.3
    cos = torch.cos(ang).repeat_interleave(2, 1)
    sin = torch.sin(ang).repeat_interleave(2, 1)
    dt = torch.float64 if f64 else torch.float32
    out = []
    for t in (cos, sin):
        buf = torch.full((S + 2, hd), NAN, dtype=dt, device=DEV)
        buf[sel] = t[sel].to(dt)
        out.append(buf)
    return out


def _rms_inputs(M, D, w_f32, kind, g):
    if kind == "exact":
        x, _, _, qx = R.exact_rows(M, D, g, DEV)
    else:
        x = torch.randn(M, D, generator=g, device=DEV) * 3
        qx = None
    w = torch.randn(D, generator=g, device=DEV) * 0.5 + 1
    return x.bfloat16(), qx, (w if w_f32 else w.bfloat16())


def _scattered(x, perm):
    """x [M, D] placed head block by head block (128 columns) into NaN rows, block j at column offs[j] (permuted, with NaN
    between blocks); returns the buffer, its rows 1..M and the int64 offsets."""
    M, D = x.shape
    nb = D // 128
    offs = (perm * 136 + 8 * (perm % 2)).to(torch.int64)  # blocks moved apart, some 8 columns off a 128 boundary
    width = int(offs.max()) + 128 + 8
    buf = torch.full((M + 2, width + 8), NAN, dtype=x.dtype, device=DEV)
    rows = buf[1:M + 1]
    for j in range(nb):
        rows[:, int(offs[j]):int(offs[j]) + 128] = x[:, 128 * j:128 * j + 128]
    return buf, rows, offs


def _gather(rows, offs):
    return torch.cat([rows[:, int(o):int(o) + 128] for o in offs.tolist()], 1)


@pytest.mark.parametrize("kind", ["exact", "random"])
@pytest.mark.parametrize("case", RMS_CASES, ids=lambda c: "-".join(map(str, c)))
def test_rmsnorm_rope(case, kind):
    M, D, hd, two, f64, w_f32, rope, scat = case
    L, check, ptr, sp = _abi()
    path = rms_path(M, D, hd, f64, sms=sms())
    g = _gen("rms", case, kind)
    S = M + 37
    prow = torch.randperm(S, generator=g, device=DEV)[:M] if rope == "perm" else torch.arange(M, device=DEV)
    tabs = _tables(S, hd, f64, g, prow)
    rr = prow.to(torch.int32) if rope == "perm" else None
    cols = torch.arange(D, device=DEV) % hd
    ce, se = tabs[0][prow][:, cols], tabs[1][prow][:, cols]
    xs, ws, bufs = [], [], []
    for t in range(2 if two else 1):
        x, qx, w = _rms_inputs(M, D, w_f32, kind, _gen("rms", case, kind, t))
        xs.append((x, qx, ce, se))
        ws.append(w)
    perm = torch.randperm(D // 128, generator=_gen("perm", case), device=DEV) if scat else None
    for x, _, _, _ in xs:
        if scat:
            buf, rows, offs = _scattered(x, perm)
        else:
            buf = torch.full((M + 2, D + 8), NAN, dtype=torch.bfloat16, device=DEV)
            rows, offs = buf[1:M + 1], None
            rows[:, :D] = x
        bufs.append((buf, rows, offs))
    offs_t = bufs[0][2]
    flags = int(f64) | (2 * int(w_f32))
    snap = [b[0].clone() for b in bufs]

    def run():
        for b, s in zip(bufs, snap):
            b[0].copy_(s)
        x1 = bufs[1][1] if two else None
        check(L.fvb_rmsnorm_rope(ptr(bufs[0][1]), ptr(ws[0]), c_int64(bufs[0][1].stride(0)), ptr(x1),
                                 ptr(ws[1] if two else None), c_int64(x1.stride(0) if two else 0), ptr(tabs[0]),
                                 ptr(tabs[1]), c_int(flags), ptr(rr), ptr(offs_t), c_int(M), c_int(D), c_int(hd),
                                 c_float(EPS), sp()))

    twice(run, [b[0] for b in bufs], "rmsnorm_rope")
    for t, ((x, qx, ce, se), w, (buf, rows, offs)) in enumerate(zip(xs, ws, bufs)):
        got = _gather(rows, offs) if scat else rows[:, :D]
        # nothing outside the row's own elements changed (NaN stays NaN bit for bit)
        mask = torch.zeros_like(buf, dtype=torch.bool)
        if scat:
            for o in offs.tolist():
                mask[1:M + 1, o:o + 128] = True
        else:
            mask[1:M + 1, :D] = True
        before = snap[t].view(torch.int16)
        assert not bool(((buf.view(torch.int16) != before) & ~mask).any()), "rmsnorm_rope wrote outside its rows"
        name = f"rmsnorm_rope tensor {t} {path}"
        where = lambda r, col: R.row_coords(r, col)
        if kind == "exact":
            cands = R.rstd_candidates(R.var_forms(qx, D, EPS, path["warp"]))
            chain = lambda r: R.rms_rope_chain(x, r, w, w_f32, ce, se, f64)
            R.assert_rows_match(got, chain, cands, name, where, family="rmsnorm_rope fwd (exact)")
        else:
            ref, bound = R.ln_fwd_bound(x.float(), EPS, rms=True, rms_w=w, rms_w_f32=w_f32, cos=ce, sin=se)
            R.assert_within(got, ref, bound, name, lambda i: where(*i), family="rmsnorm_rope fwd (random)")


# (M, D, head_dim, mode: norm / rope_only / copy, two tensors)
SCATTER_CASES = [(1, 1536, 128, "norm", True), (300, 1536, 128, "norm", False), (77, 5120, 128, "rope_only", True),
                 (300, 1536, 64, "copy", True), (1000, 3072, 128, "norm", True)]


@pytest.mark.parametrize("case", SCATTER_CASES, ids=lambda c: "-".join(map(str, c)))
def test_rmsnorm_rope_scatter(case):
    M, D, hd, mode, two = case
    L, check, ptr, sp = _abi()
    nt = 2 if two else 1
    ins = []
    for t in range(nt):
        g = _gen("scatter", case, t)
        x, _, _, qx, = R.exact_rows(M, D, g, DEV)
        x = x.bfloat16()
        if mode == "rope_only":  # already-normalised rows: any bf16 values
            x = (torch.randn(M, D, generator=g, device=DEV)).bfloat16()
        w = (torch.randn(D, generator=g, device=DEV) * 0.5 + 1).bfloat16()
        ins.append((nan_rows(x), x, qx, w))
    g = _gen("scatter-tab", case)
    S = M + 5
    prow = torch.randperm(S, generator=g, device=DEV)[:M]
    cos, sin = _tables(S, hd, False, g, prow)
    cols = torch.arange(D, device=DEV) % hd
    ce, se = cos[prow][:, cols], sin[prow][:, cols]
    nb = D // 128
    perm = torch.randperm(nb, generator=g, device=DEV)
    offs = (perm * 136).to(torch.int64)  # blocks permuted, 8 spare columns after each
    ldy = nb * 136 + 16
    outs = [R.Guarded((M + 2, ldy), torch.bfloat16, DEV, seed=10 + t) for t in range(nt)]
    for o in outs:
        rows = o.buf[1:M + 1]
        for j in offs.tolist():
            o.region(rows[:, j:j + 128])
    tab = (None, None) if mode == "copy" else (cos, sin)
    wp = [None if mode != "norm" else i[3] for i in ins]
    rr = prow.to(torch.int32)

    def run():
        x1 = ins[1][0] if two else None
        check(L.fvb_rmsnorm_rope_scatter(ptr(ins[0][0]), ptr(wp[0]), c_int64(ins[0][0].stride(0)), ptr(x1),
                                         ptr(wp[1] if two else None), c_int64(x1.stride(0) if two else 0),
                                         ptr(outs[0].buf[1:]), ptr(outs[1].buf[1:] if two else None), c_int64(ldy), ptr(offs),
                                         ptr(tab[0]), ptr(tab[1]), c_int(0), ptr(rr), c_int(M), c_int(D),
                                         c_int(hd), c_float(EPS), sp()))

    twice(run, [o.buf for o in outs], "rmsnorm_rope_scatter")
    for t, (o, (xv, x, qx, w)) in enumerate(zip(outs, ins)):
        o.assert_untouched(f"scatter tensor {t}")
        got = _gather(o.buf[1:M + 1], offs)
        if mode == "copy":
            R.assert_exact(got, x, "scatter copy", lambda i: R.row_coords(*i), family="rmsnorm_rope fwd (exact)")
        elif mode == "rope_only":
            R.assert_exact(got, R.rms_rope_chain(x, None, None, False, ce, se), "scatter rope only",
                           lambda i: R.row_coords(*i), family="rmsnorm_rope fwd (exact)")
        else:
            cands = R.rstd_candidates(R.var_forms(qx, D, EPS, True))
            R.assert_rows_match(got, lambda r: R.rms_rope_chain(x, r, w, False, ce, se), cands, f"scatter {t}",
                                family="rmsnorm_rope fwd (exact)")


# ------------------------------------------------------------------------------------------------ RMSNorm backward
RMS_BWD_CASES = [(1, 1536, True), (527, 1536, True), (528, 256, True), (529, 2056, False), (1063, 5120, True),
                 (700, 8192, True), (530, 8, True), (300, 264, False)]


def _masked_dy(x, cands, dy, pair=False):
    """dy with 0 wherever the rstd candidates disagree on bf16(x^) (for RoPE: on either element of the pair)."""
    xh = torch.stack([x.float() * cands[:, k:k + 1] for k in range(cands.shape[1])])
    xb, ok = R.unambiguous_bf16(xh)
    if pair:
        ok2 = ok[:, 0::2] & ok[:, 1::2]
        ok = torch.stack([ok2, ok2], -1).flatten(1)
    return dy * ok, xb


def _bf16_dx_bound(o, eo):
    return eo + R.half_ulp_bf16(o.abs() + eo)


@pytest.mark.parametrize("rope", [False, True])
@pytest.mark.parametrize("case", RMS_BWD_CASES, ids=lambda c: "-".join(map(str, c)))
def test_rmsnorm_bwd(case, rope):
    M, D, has_w = case
    hd = 128 if D % 128 == 0 else 8
    if rope and not has_w:
        pytest.skip("fvb_rmsnorm_rope_bwd needs w")
    L, check, ptr, sp = _abi()
    g = _gen("rmsbwd", case, rope)
    x, _, _, qx = R.exact_rows(M, D, g, DEV)
    x = x.bfloat16()
    cands = R.rstd_candidates(R.var_forms(qx, D, EPS, False))
    dy = R.grid_bf16((M, D), g, DEV)
    w = R.grid_bf16((D,), g, DEV) if has_w else None
    S = M + 11
    prow = torch.randperm(S, generator=g, device=DEV)[:M]
    cos, sin = _tables(S, hd, False, g, prow)
    cols = torch.arange(D, device=DEV) % hd
    ce, se = cos[prow][:, cols], sin[prow][:, cols]
    dy, xb = _masked_dy(x, cands, dy.float(), pair=rope)
    dy = dy.bfloat16()
    xv, dyv = nan_rows(x), nan_rows(dy)
    dx = Out(M, D, torch.bfloat16, 4)
    dwo = R.Guarded((D + 32,), torch.bfloat16, DEV, seed=5)
    dw = dwo.region(dwo.buf[8:8 + D]) if has_w else None
    nb = L.fvb_rmsnorm_rope_bwd_workspace_bytes(M, D) if rope else L.fvb_rmsnorm_bwd_workspace_bytes(M, D)
    ws = Workspace(nb)
    rr = prow.to(torch.int32)

    def run():
        if rope:
            check(L.fvb_rmsnorm_rope_bwd(ptr(xv), c_int64(xv.stride(0)), ptr(w), ptr(dyv), c_int64(dyv.stride(0)), ptr(dx.v),
                                         c_int64(dx.ld), ptr(dw), None, c_int64(0), None, None, c_int64(0), None, c_int64(0),
                                         None, _f32p(cos), _f32p(sin), ptr(rr), _f32p(ws.v), c_int64(ws.bytes), c_int(M),
                                         c_int(D), c_int(hd), c_float(EPS), sp()))
        else:
            check(L.fvb_rmsnorm_bwd(ptr(xv), c_int64(xv.stride(0)), ptr(w), ptr(dyv), c_int64(dyv.stride(0)), ptr(dx.v),
                                    c_int64(dx.ld), ptr(dw), _f32p(ws.v), c_int64(ws.bytes), c_int(M), c_int(D),
                                    c_float(EPS), sp()))

    twice(run, [dx.v] + ([dw] if has_w else []), "rmsnorm_bwd")
    dx.g.assert_untouched("dx")
    dwo.assert_untouched("dw")
    ctas = min(M, R.RB_CTAS)
    fam = "rmsnorm_rope bwd" if rope else "rmsnorm bwd"
    dv = dy.float()
    if rope:  # dn = bf16(R^T dy), fp32 products and sums replayed
        g0, g1 = dv[:, 0::2], dv[:, 1::2]
        dn0 = (g0 * ce[:, 0::2] + g1 * se[:, 1::2]).bfloat16().float()
        dn1 = (g1 * ce[:, 1::2] - g0 * se[:, 0::2]).bfloat16().float()
        dv = torch.stack([dn0, dn1], -1).flatten(1)
    if has_w:
        ws.check(fam, ctas * D)  # fvb_rmsnorm_rope_bwd's second half belongs to x1, absent here
        ref = R.colsum_replay(dv * xb, ctas)[0].bfloat16()
        R.assert_exact(dw, ref, f"{fam} dw", lambda i: dict(col=i[0]), family=f"{fam} dw/db (exact)")
    gt = (dv * w.float()).bfloat16().float() if has_w else dv
    o, eo = R.norm_bwd_dx_bound(x.float(), gt, EPS, rms=True)
    R.assert_within(dx.v, o, _bf16_dx_bound(o, eo), f"{fam} dx", lambda i: R.row_coords(*i), family=f"{fam} dx")


# ------------------------------------------------------------------------------------------------ LayerNorm backward
# (M, D, x_f32, gain_is_scale, round_ln, gin: None / bf16 / f32)
LN_BWD_CASES = [(1, 1536, False, True, 1, None), (527, 1536, False, True, 1, "bf16"), (528, 2056, True, True, 0, "f32"),
                (529, 5120, False, False, 0, "f32"), (1063, 8192, False, True, 1, "bf16"), (600, 264, True, False, 0, None),
                (530, 8, False, True, 1, None), (1063, 256, True, True, 1, "f32")]


@pytest.mark.parametrize("case", LN_BWD_CASES, ids=lambda c: "-".join(map(str, c)))
def test_layernorm_modulate_bwd(case):
    M, D, x_f32, is_scale, round_ln, gin_kind = case
    L, check, ptr, sp = _abi()
    g = _gen("lnbwd", case)
    x, c, qz, _ = R.exact_rows(M, D, g, DEV)
    x = x if x_f32 else x.bfloat16()
    cands = R.rstd_candidates(R.var_forms(qz, D, EPS, False))
    t = torch.stack([(x.float() - c[:, None]) * cands[:, k:k + 1] for k in range(cands.shape[1])])
    tb, ok = R.unambiguous_bf16(t)
    dn = R.grid_bf16((M, D), g, DEV)
    if round_ln:
        dn = (dn.float() * ok).bfloat16()
    gain = torch.randn(D, generator=g, device=DEV) * 0.5 + (0 if is_scale else 1)
    gin = None if gin_kind is None else (torch.randn(M, D, generator=g, device=DEV) * 0.1)
    if gin_kind == "bf16":
        gin = gin.bfloat16()
    xv, dnv = nan_rows(x), nan_rows(dn)
    ginv = nan_rows(gin) if gin is not None else None
    dx = Out(M, D, torch.float32 if x_f32 else torch.bfloat16, 6)
    dgo = R.Guarded((2, D + 16), torch.float32, DEV, seed=7)
    dgain, doff = dgo.region(dgo.buf[0, :D]), dgo.region(dgo.buf[1, :D])
    ws = Workspace(L.fvb_layernorm_modulate_bwd_workspace_bytes(M, D))

    def run():
        check(L.fvb_layernorm_modulate_bwd(ptr(xv), c_int(int(x_f32)), c_int64(xv.stride(0)), ptr(dnv), c_int64(dnv.stride(0)),
                                           _f32p(gain), c_int(int(is_scale)), c_int(round_ln), ptr(ginv),
                                           c_int(int(gin_kind == "f32")), c_int64(ginv.stride(0) if gin is not None else 0),
                                           ptr(dx.v), c_int64(dx.ld), _f32p(dgain), _f32p(doff), _f32p(ws.v),
                                           c_int64(ws.bytes), c_int(M), c_int(D), c_float(EPS), sp()))

    twice(run, [dx.v, dgain, doff], "layernorm_modulate_bwd")
    dx.g.assert_untouched("dx")
    dgo.assert_untouched("d_gain / d_offset")
    ws.check("layernorm_modulate_bwd")
    ctas = min(M, R.RB_CTAS)
    dnf = dn.float()
    R.assert_exact(doff, R.colsum_replay(dnf, ctas)[0], "d_offset", lambda i: dict(col=i[0]),
                   family="layernorm bwd column sums (exact)")
    if round_ln:
        R.assert_exact(dgain, R.colsum_replay(dnf * tb, ctas)[0], "d_gain", lambda i: dict(col=i[0]),
                       family="layernorm bwd column sums (exact)")
    else:  # dn * t is not exact: fp64 bound from t's error and an M-term fp32 sum
        mean, r, rho, e_mean = R._stats64(x.float(), D, EPS, True)
        t64 = (x.double() - mean[:, None]) * r[:, None]
        et = t64.abs() * rho[:, None] + r[:, None] * e_mean[:, None] + R.U32 * t64.abs()
        ref = (dnf.double() * t64).sum(0)
        bound = (dnf.double().abs() * et).sum(0) + R.gamma(2 * M) * (dnf.double() * t64).abs().sum(0)
        R.assert_within(dgain, ref, bound, "d_gain", lambda i: dict(col=i[0]), family="layernorm bwd d_gain (random)")
    gv = (torch.ones_like(gain) + gain) if is_scale else gain
    o, eo = R.norm_bwd_dx_bound(x.float(), dnf * gv, EPS, rms=False, gin=gin)
    bound = eo if x_f32 else _bf16_dx_bound(o, eo)
    R.assert_within(dx.v, o, bound, "layernorm bwd dx", lambda i: R.row_coords(*i), family="layernorm bwd dx")


# ------------------------------------------------------------------------------------------------ column-sum backwards
BIAS_M = [255, 256, 257, 1792, 1793, 2047, 2048, 2049, 2303]
BIAS_N = [8, 1016, 1024, 1032, 5120]


@pytest.mark.parametrize("N", BIAS_N)
@pytest.mark.parametrize("M", BIAS_M)
def test_bias_grad(M, N):
    L, check, ptr, sp = _abi()
    g = _gen("bias", M, N)
    dy = R.rand_bf16((M, N), g, DEV)
    dyv = nan_rows(dy)
    dbo = R.Guarded((N + 24,), torch.bfloat16, DEV, seed=8)
    db = dbo.region(dbo.buf[8:8 + N])
    ws = Workspace(L.fvb_bias_grad_bf16_workspace_bytes(M, N))
    twice(lambda: check(L.fvb_bias_grad_bf16(ptr(dyv), c_int64(dyv.stride(0)), ptr(db), _f32p(ws.v), c_int64(ws.bytes),
                                             c_int(M), c_int(N), sp())), [db], "bias_grad")
    dbo.assert_untouched("db")
    ws.check("bias_grad")
    ref = R.colsum_replay(dy.float(), min(M, R.BG_PARTS))[0].bfloat16()
    R.assert_exact(db, ref, "db", lambda i: dict(col=i[0], col_block=i[0] // 1024), family="bias/gate column sums (exact)")


@pytest.mark.parametrize("with_db", [True, False])
@pytest.mark.parametrize("dout_f32", [False, True])
@pytest.mark.parametrize("M,N", [(255, 1032), (257, 8), (1793, 1024), (2048, 5120), (2303, 1016), (2049, 1032)])
def test_resid_gate_bwd(M, N, dout_f32, with_db):
    L, check, ptr, sp = _abi()
    g = _gen("gate", M, N, dout_f32)
    dout = R.rand_bf16((M, N), g, DEV)  # bf16-representable, also when passed as fp32
    dout = dout.float() if dout_f32 else dout
    y = R.rand_bf16((M, N), g, DEV)
    gate = torch.randn(N, generator=g, device=DEV)
    dov, yv = nan_rows(dout), nan_rows(y)
    dy = Out(M, N, torch.bfloat16, 9)
    go = R.Guarded((3 * N + 64,), torch.float32, DEV, seed=11)
    dgate = go.region(go.buf[16:16 + N])
    bo = R.Guarded((N + 24,), torch.bfloat16, DEV, seed=12)
    db = bo.region(bo.buf[8:8 + N]) if with_db else None
    ws = Workspace(L.fvb_resid_gate_bwd_workspace_bytes(M, N))
    twice(lambda: check(L.fvb_resid_gate_bwd(ptr(dov), c_int(int(dout_f32)), c_int64(dov.stride(0)), ptr(yv),
                                             c_int64(yv.stride(0)), _f32p(gate), ptr(dy.v), c_int64(dy.ld), _f32p(dgate),
                                             ptr(db), _f32p(ws.v), c_int64(ws.bytes), c_int(M), c_int(N), sp())),
          [dy.v, dgate] + ([db] if with_db else []), "resid_gate_bwd")
    dy.g.assert_untouched("dy")
    go.assert_untouched("d_gate")
    bo.assert_untouched("db")
    ws.check("resid_gate_bwd")
    fam = "bias/gate column sums (exact)"
    P = min(M, R.BG_PARTS)
    dyr = (dout.float() * gate).bfloat16()
    R.assert_exact(dy.v, dyr, "dy", lambda i: R.row_coords(*i), family=fam)
    R.assert_exact(dgate, R.colsum_replay(dout.float() * y.float(), P)[0], "d_gate", lambda i: dict(col=i[0]), family=fam)
    if with_db:
        R.assert_exact(db, R.colsum_replay(dyr.float(), P)[0].bfloat16(), "db", lambda i: dict(col=i[0]), family=fam)


# ------------------------------------------------------------------------------------------------ grouped backwards
# (M, R, D or N, gin kind / with db)
GROUPED_CASES = [(1000, 1000, 1536), (1000, 1200, 264),  # G = 1: P = min(budget, R)
                 (700, 1, 256), (600, 2, 1032),  # G > budget: P = 1
                 (40, 8, 1536), (45, 8, 2056),  # P clamped to R; last group of 5 rows < P
                 (2000, 350, 1024), (1003, 100, 5120),  # last group shorter than R and than P
                 (32760, 1560, 1536)]  # the causal shape: R = 1560, G = 21


@pytest.mark.parametrize("gin_kind", [None, "bf16", "f32"])
@pytest.mark.parametrize("case", GROUPED_CASES, ids=lambda c: "-".join(map(str, c)))
def test_layernorm_modulate_grouped_bwd(case, gin_kind):
    M, R_, D = case
    if gin_kind == "bf16" and M > 20000:
        pytest.skip("the causal shape runs with fp32 gin and without gin")
    L, check, ptr, sp = _abi()
    g = _gen("lngbwd", case, gin_kind)
    x, c, qz, _ = R.exact_rows(M, D, g, DEV)
    x = x.bfloat16()
    cands = R.rstd_candidates(R.var_forms(qz, D, EPS, False))
    t = torch.stack([(x.float() - c[:, None]) * cands[:, k:k + 1] for k in range(cands.shape[1])])
    tb, ok = R.unambiguous_bf16(t)
    dn = (R.grid_bf16((M, D), g, DEV).float() * ok).bfloat16()
    G = -(-M // R_)
    scale = (torch.randn(G, D, generator=g, device=DEV) * 0.5).bfloat16().float()
    sc = nan_groups(scale, G, D + 4)
    gin = None if gin_kind is None else torch.randn(M, D, generator=g, device=DEV) * 0.1
    if gin_kind == "bf16":
        gin = gin.bfloat16()
    xv, dnv = nan_rows(x), nan_rows(dn)
    ginv = nan_rows(gin) if gin is not None else None
    dx = Out(M, D, torch.bfloat16, 13)
    ld = D + 12
    mo = R.Guarded((2, G + 1, ld), torch.float32, DEV, seed=14)
    dsc, dsh = mo.region(mo.buf[0, :G, :D]), mo.region(mo.buf[1, :G, :D])
    ws = Workspace(L.fvb_layernorm_modulate_grouped_bwd_workspace_bytes(M, R_, D))

    def run():
        check(L.fvb_layernorm_modulate_grouped_bwd(ptr(xv), c_int64(xv.stride(0)), ptr(dnv), c_int64(dnv.stride(0)), _f32p(sc),
                                                   c_int(R_), c_int64(sc.stride(0)), ptr(ginv), c_int(int(gin_kind == "f32")),
                                                   c_int64(ginv.stride(0) if gin is not None else 0), ptr(dx.v),
                                                   c_int64(dx.ld), _f32p(dsc), _f32p(dsh), c_int64(ld), _f32p(ws.v),
                                                   c_int64(ws.bytes), c_int(M), c_int(D), c_float(EPS), sp()))

    twice(run, [dx.v, dsc, dsh], "layernorm_modulate_grouped_bwd")
    dx.g.assert_untouched("dx")
    mo.assert_untouched("d_scale / d_shift")
    ws.check("layernorm_modulate_grouped_bwd")
    fam = "grouped bwd column sums (exact)"
    where = lambda i: dict(group=i[0], col=i[1])
    dnf = dn.float()
    R.assert_exact(dsh, R.grouped_colsum_replay(dnf, R_, R.RB_CTAS)[0], "d_shift", where, family=fam)
    R.assert_exact(dsc, R.grouped_colsum_replay(dnf * tb, R_, R.RB_CTAS)[0], "d_scale", where, family=fam)
    grp = torch.arange(M, device=DEV) // R_
    gv = (torch.ones_like(scale) + scale).bfloat16().float()[grp]
    dt = (dnf * gv).bfloat16().float()
    o, eo = R.norm_bwd_dx_bound(x.float(), dt, EPS, rms=False, gin=gin)
    R.assert_within(dx.v, o, _bf16_dx_bound(o, eo), "grouped dx", lambda i: R.row_coords(*i), family="grouped bwd dx")


@pytest.mark.parametrize("with_db", [True, False])
@pytest.mark.parametrize("case", GROUPED_CASES, ids=lambda c: "-".join(map(str, c)))
def test_resid_gate_grouped_bwd(case, with_db):
    M, R_, N = case
    L, check, ptr, sp = _abi()
    g = _gen("gategrp", case, with_db)
    dout, y = R.rand_bf16((M, N), g, DEV), R.rand_bf16((M, N), g, DEV)
    G = -(-M // R_)
    gate = torch.randn(G, N, generator=g, device=DEV).bfloat16().float()
    gt = nan_groups(gate, G, N + 8)
    dov, yv = nan_rows(dout), nan_rows(y)
    dy = Out(M, N, torch.bfloat16, 15)
    ld = N + 20
    go = R.Guarded((G + 2, ld), torch.float32, DEV, seed=16)
    dgate = go.region(go.buf[1:G + 1, :N])
    bo = R.Guarded((N + 24,), torch.bfloat16, DEV, seed=17)
    db = bo.region(bo.buf[8:8 + N]) if with_db else None
    ws = Workspace(L.fvb_resid_gate_grouped_bwd_workspace_bytes(M, R_, N))
    twice(lambda: check(L.fvb_resid_gate_grouped_bwd(ptr(dov), c_int64(dov.stride(0)), ptr(yv), c_int64(yv.stride(0)),
                                                     _f32p(gt), c_int(R_), c_int64(gt.stride(0)), ptr(dy.v), c_int64(dy.ld),
                                                     _f32p(dgate), c_int64(ld), ptr(db), _f32p(ws.v), c_int64(ws.bytes),
                                                     c_int(M), c_int(N), sp())),
          [dy.v, dgate] + ([db] if with_db else []), "resid_gate_grouped_bwd")
    dy.g.assert_untouched("dy")
    go.assert_untouched("d_gate")
    bo.assert_untouched("db")
    ws.check("resid_gate_grouped_bwd")
    fam = "grouped bwd column sums (exact)"
    grp = torch.arange(M, device=DEV) // R_
    dyr = (dout.float() * gate[grp]).bfloat16()
    R.assert_exact(dy.v, dyr, "dy", lambda i: R.row_coords(*i), family=fam)
    R.assert_exact(dgate, R.grouped_colsum_replay(dout.float() * y.float(), R_, R.BG_PARTS)[0], "d_gate",
                   lambda i: dict(group=i[0], col=i[1]), family=fam)
    if with_db:
        parts = R.grouped_colsum_replay(dyr.float(), R_, R.BG_PARTS)[1]
        R.assert_exact(db, R.partial_sum(parts.flatten(0, 1)).bfloat16(), "db", lambda i: dict(col=i[0]), family=fam)


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    R.print_summary(request.config)
    name = torch.cuda.get_device_name(0)
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    cap = request.config.pluginmanager.getplugin("capturemanager")
    with cap.global_and_fixture_disabled():
        print(f"  device: {name}, power limit {pl}", flush=True)
