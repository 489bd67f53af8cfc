"""GPU: the Wan VAE decoder's row and data-movement kernels (csrc/vae_ops.cu) element by element, through the C ABI
(tests/elementwise_ref.py, "Convolutions"): the channels-last RMS norm (bf16 and e4m3 outputs) replayed bit for bit without
SiLU and held to the round-to-nearest interval of its bound with SiLU, the row softmax bit for bit on tie rows and within an
fp64 bound on random rows, upsample, transpose and clamp bit for bit. Outputs go into sentinel buffers with row gaps; row
gaps of the inputs hold NaN."""
from ctypes import c_float, c_int, c_int64
import zlib

import pytest
import torch

import elementwise_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAN = float("nan")


def _abi():
    from fastvideo_b200 import _lib, ops
    return _lib.lib(), _lib.check, _lib.ptr, _lib.stream_ptr, ops._f32p


def _gen(*key):
    return torch.Generator(device=DEV).manual_seed(zlib.crc32(repr(key).encode()))


def nan_rows(t, gap):
    """t [M, C] in a NaN-filled [M, C + gap] buffer; returns the view."""
    buf = torch.full((t.shape[0], t.shape[1] + gap), NAN, dtype=t.dtype, device=DEV)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


class Out:
    """An output [M, C] view with row stride C + gap inside a sentinel buffer with one row before and after."""

    def __init__(self, M, C, gap, dtype, seed):
        self.g = R.Guarded((M + 2, C + gap), dtype, DEV, seed=seed)
        self.v = self.g.region(self.g.buf[1:M + 1, :C])
        self.ld = C + gap


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    R.print_summary(request.config)


# (pixels, C, x gap, out gap): pixel counts off a multiple of the 8 warps of a CTA; the decoder's widths at real frame sizes
NORM_CASES = [(13, 8, 8, 8), (1001, 96, 8, 16), (999, 264, 16, 8), (517, 384, 8, 8), (480 * 832, 96, 0, 0),
              (120 * 208 + 3, 384, 8, 8), (1, 96, 0, 8)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("out", ["bf16", "bf16+beta", "e4m3", "e4m3 bound 0"])
@pytest.mark.parametrize("case", NORM_CASES, ids=lambda c: "-".join(map(str, c)))
def test_rmsnorm_silu_cl(case, out, silu):
    P, C, xg, og = case
    L, check, ptr, sp, f32p = _abi()
    g = _gen("norm", case, out, silu)
    x = R.rand_bf16((P, C), g, DEV, 2.0)
    x[0, :] = 0  # the 1e-12 floor of the norm
    xv = nan_rows(x, xg)
    gamma = 1 + 0.2 * torch.randn(C, generator=g, device=DEV)
    beta = 0.3 * torch.randn(C, generator=g, device=DEV) if out == "bf16+beta" else None
    e4m3 = out.startswith("e4m3")
    o = Out(P, C, og + (8 if e4m3 else 0), torch.float8_e4m3fn if e4m3 else torch.bfloat16, 1)
    bound = 0.0 if out.endswith("0") else R.f32(float(torch.tensor(float(C)).sqrt() * gamma.abs().max().cpu()))
    if e4m3:
        check(L.fvb_rmsnorm_silu_cl_e4m3(ptr(xv), c_int64(xv.stride(0)), f32p(gamma), ptr(o.v), c_int64(o.ld), c_int64(P),
                                         c_int(C), c_int(int(silu)), c_float(bound), sp()))
    else:
        check(L.fvb_rmsnorm_silu_cl(ptr(xv), c_int64(xv.stride(0)), f32p(gamma), f32p(beta), ptr(o.v), c_int64(o.ld),
                                    c_int64(P), c_int(C), c_int(int(silu)), sp()))
    torch.cuda.synchronize()
    o.g.assert_untouched("rmsnorm_silu_cl out")
    v = R.rownorm_replay(x, gamma, beta)
    qs = R.e4m3_qscale(bound) if e4m3 else None
    where = lambda i: dict(pixel=int(i[0]), channel=int(i[1]), lane=(int(i[1]) // 8) % 32)
    fam = f"vae rmsnorm_silu_cl {'e4m3' if e4m3 else 'bf16'}"
    if not silu:
        if e4m3:
            R.assert_exact(o.v.view(torch.uint8), R.e4m3_code(v, qs).view(torch.uint8), "rmsnorm e4m3", where, fam)
        else:
            R.assert_exact(o.v, v.bfloat16(), "rmsnorm bf16", where, fam)
        return
    ref, b = R.silu_bound(v)
    R.assert_rounds_from(o.v.float(), ref, b, "rmsnorm + SiLU", qscale=qs, where=where,
                         family=fam + " (SiLU, round-to-nearest interval)")


@pytest.mark.parametrize("shape", [(2, 7, 9, 8), (3, 5, 3, 96), (1, 60, 104, 384), (1, 1, 1, 264)])
def test_upsample2x_cl(shape):
    T, H, W, C = shape
    L, check, ptr, sp, _ = _abi()
    x = R.rand_bf16(shape, _gen("up", shape), DEV)
    n = T * 4 * H * W * C
    g = R.Guarded((n + 64,), torch.bfloat16, DEV, seed=2)
    o = g.region(g.buf[:n]).view(T, 2 * H, 2 * W, C)
    check(L.fvb_upsample2x_cl(ptr(x), ptr(o), c_int(T), c_int(H), c_int(W), c_int(C), sp()))
    torch.cuda.synchronize()
    g.assert_untouched("upsample2x out")
    R.assert_exact(o, x.repeat_interleave(2, 1).repeat_interleave(2, 2), "upsample2x", family="vae upsample2x_cl")


@pytest.mark.parametrize("shape", [(1, 1), (33, 95), (64, 31), (100, 257), (9, 1024)])
def test_transpose_bf16(shape):
    Rr, C = shape
    L, check, ptr, sp, _ = _abi()
    x = R.rand_bf16(shape, _gen("tr", shape), DEV)
    xv = nan_rows(x, 5)
    o = Out(C, Rr, 3, torch.bfloat16, 3)
    check(L.fvb_transpose_bf16(ptr(xv), c_int64(xv.stride(0)), ptr(o.v), c_int64(o.ld), c_int(Rr), c_int(C), sp()))
    torch.cuda.synchronize()
    o.g.assert_untouched("transpose out")
    R.assert_exact(o.v, x.T, "transpose", family="vae transpose_bf16")


SOFTMAX_N = [1, 255, 256, 257, 1350, 6240]


def _softmax_call(x, o):
    L, check, ptr, sp, _ = _abi()
    check(L.fvb_softmax_rows_f32(ptr(x), c_int64(x.stride(0)), ptr(o.v), c_int64(o.ld), c_int64(x.shape[0]),
                                 c_int(x.shape[1]), sp()))
    torch.cuda.synchronize()
    o.g.assert_untouched("softmax out")


@pytest.mark.parametrize("n", SOFTMAX_N)
def test_softmax_rows_f32_ties(n):
    """Integer logits at the row maximum or at least 150 below it (some -inf): p = 1 at the ties (__expf(0) = 1), 0 below
    (underflow), so the output is bf16(fl(1 / ties)) at the ties and 0 elsewhere, bit for bit."""
    g = _gen("smt", n)
    rows = 7
    top = torch.randint(-50, 50, (rows, 1), generator=g, device=DEV).float()
    below = top - 150 - torch.randint(0, 400, (rows, n), generator=g, device=DEV).float()
    tie = torch.rand(rows, n, generator=g, device=DEV) < torch.tensor([0.0, 0.01, 0.3, 1.0, 0.5, 0.05, 0.9],
                                                                      device=DEV)[:, None]
    tie[torch.arange(rows), torch.randint(0, n, (rows,), generator=g, device=DEV)] = True
    x = torch.where(tie, top, below)
    x[(torch.rand(rows, n, generator=g, device=DEV) < 0.1) & ~tie] = float("-inf")
    xv = nan_rows(x, 4)
    o = Out(rows, n, 8, torch.bfloat16, 4)
    _softmax_call(xv, o)
    cnt = tie.sum(1, keepdim=True).float()
    ref = torch.where(tie, torch.ones_like(cnt) / cnt, torch.zeros_like(x)).bfloat16()
    R.assert_exact(o.v, ref, f"softmax ties n={n}", family="vae softmax_rows_f32 (ties)")


@pytest.mark.parametrize("n", SOFTMAX_N)
def test_softmax_rows_f32_random(n):
    g = _gen("smr", n)
    rows = 9
    x = torch.randn(rows, n, generator=g, device=DEV) * 3
    x[1] = x[1] * 10
    x[2, 1::3] = float("-inf")
    xv = nan_rows(x, 8)
    o = Out(rows, n, 8, torch.bfloat16, 5)
    _softmax_call(xv, o)
    ref, b = R.softmax_bound(x)
    R.assert_within(o.v, ref, b, f"softmax random n={n}", family="vae softmax_rows_f32 (random)")


@pytest.mark.parametrize("npix,C,ld", [(1, 3, 8), (999, 3, 96), (32 * 48, 3, 3), (77, 16, 24)])
def test_clamp_to_nchw(npix, C, ld):
    L, check, ptr, sp, _ = _abi()
    x = R.rand_bf16((npix, C), _gen("clamp", npix, C), DEV, 1.5)
    xv = nan_rows(x, ld - C)
    g = R.Guarded((C * npix + 64,), torch.float32, DEV, seed=6)
    o = g.region(g.buf[:C * npix]).view(C, npix)
    check(L.fvb_clamp_to_nchw(ptr(xv), c_int64(ld), ptr(o), c_int(C), c_int64(npix), sp()))
    torch.cuda.synchronize()
    g.assert_untouched("clamp out")
    R.assert_exact(o, x.float().clamp(-1, 1).T, "clamp_to_nchw", family="vae clamp_to_nchw")
