"""GPU: the wgmma GEMM (fvb_linear_bf16 and the entry points on its kernel body) element by element, at every tile and
dispatch boundary the host code selects on.

Every case runs twice: on grid inputs, where the output is compared bit for bit with the rounding points of
include/fvb200.h, and on random inputs, where each element is held to an fp64 bound (tests/elementwise_ref.py). Every
output lives inside a sentinel buffer, and every strided operand has garbage in its gaps."""
from ctypes import c_float, c_int, c_int64
import math

import pytest
import torch

import elementwise_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
NUM_SMS = 132


@pytest.fixture(scope="module", autouse=True)
def _report(request):
    yield
    R.print_summary(request.config)


def _lib():
    from fastvideo_b200._lib import lib
    return lib()


def _check(code):
    from fastvideo_b200._lib import check
    check(code)


def _p(t):
    from fastvideo_b200._lib import ptr
    return ptr(t)


def _s():
    from fastvideo_b200._lib import stream_ptr
    return stream_ptr()


def _f32p(t):
    from fastvideo_b200.ops import _f32p
    return _f32p(t)


def bn_of(N):
    """The bf16 GEMM's tile width (gemm_impl)."""
    return 256 if N >= 256 and N % 256 == 0 else 128 if N >= 128 and N % 128 == 0 else 256 if N >= 192 else 64


def _operand(rows, cols, pad, gen, grid, scale=1.0):
    """[rows, cols] bf16 view of a [rows, cols + pad] buffer whose pad columns hold large values the GEMM must not read."""
    buf = (torch.randn(rows, cols + pad, generator=gen, device=DEV) * 1e3).bfloat16()
    v = buf[:, :cols]
    v.copy_(R.grid_bf16((rows, cols), gen, DEV) if grid else R.rand_bf16((rows, cols), gen, DEV, scale))
    return v


def _expand_gate(gate, gate_rows, M, N):
    if gate_rows == 0:
        return gate[0, :N].expand(M, N)
    return gate[torch.arange(M, device=DEV) // gate_rows, :N]


def run_linear(M, N, K, epi, bias=True, gate_rows=0, pads=(0, 0, 0, 0), gate_pad=0, seed=0, grid=True, ret=False):
    """fvb_linear_bf16 through the C ABI with x / w / resid / out views of padded buffers (pads: ldx - K, ldw - K,
    ldr - N, ldo - N_store); checks every element and the sentinels. ret: also return what the checks used."""
    g = torch.Generator(device=DEV).manual_seed(seed * 7919 + M * 31 + N * 7 + K + epi)
    N8 = (N + 7) // 8 * 8
    x = _operand(M, K, pads[0], g, grid)
    w = _operand(N, K, pads[1], g, grid, K ** -0.5)
    b = (R.grid_bf16((N,), g, DEV) if grid else R.rand_bf16((N,), g, DEV)) if bias else None
    needs_resid = epi in (R.EPI_GATE_F32, R.EPI_GATE_BF16, R.EPI_RESID_BF16, R.EPI_GATE_BF16R)
    needs_gate = needs_resid and epi != R.EPI_RESID_BF16
    resid = _operand(M, N, pads[2], g, False) if needs_resid else None
    gate = None
    if needs_gate:
        G = 1 if gate_rows == 0 else (M + gate_rows - 1) // gate_rows
        gate = torch.randn(G, N + gate_pad, generator=g, device=DEV)
    out_dt = torch.float32 if epi == R.EPI_GATE_F32 else torch.bfloat16
    ldo = N8 + pads[3]
    # rows of ldo elements from row 2 of the guard buffer: sentinels before, after and in the ldo - N_store gaps
    guard = R.Guarded(((M + 4) * ldo,), out_dt, DEV, seed=seed + 1)
    out = guard.region(guard.buf.as_strided((M, N8), (ldo, 1), 2 * ldo))
    _check(_lib().fvb_linear_bf16(_p(x), c_int64(x.stride(0)), _p(w), c_int64(w.stride(0)), _p(b), _p(out), c_int64(ldo),
                                  _p(resid), c_int64(resid.stride(0) if resid is not None else 0), _f32p(gate),
                                  c_int(gate_rows), c_int64(gate.stride(0) if gate is not None else 0), c_int(M), c_int(N),
                                  c_int(K), c_int(epi), _s()))
    name = f"linear M={M} N={N} K={K} epi={epi} bias={bias} gate_rows={gate_rows} pads={pads} {'grid' if grid else 'random'}"
    where = lambda idx: R.gemm_coords(idx, bn_of(N))
    torch.cuda.synchronize()
    guard.assert_untouched(name)
    if N8 != N:
        assert bool((out[:, N:] == 0).all()), f"{name}: columns N..N rounded to 8 must be zeros"
    got = out[:, :N]
    ge = _expand_gate(gate, gate_rows, M, N) if gate is not None else None
    e, A = R.exact_gemm(x, w)
    if grid:
        if epi == R.EPI_GELU:
            y = R.epilogue_ref(e.float(), R.EPI_BIAS, bias=b).double()
            ref, bound = R.gelu_grid_bound(y)
            R.assert_within(got, ref, bound, name, where, family="gemm bf16 forward gelu, grid inputs")
        else:
            ref = R.epilogue_ref(e.float(), epi, bias=b, resid=resid, gate=ge)
            R.assert_exact(got, ref, name, where, family="gemm bf16 forward")
    else:
        ref, bound = R.epilogue_bound(e, A, K, epi, bias=b, resid=resid, gate=ge)
        R.assert_within(got, ref, bound, name, where, family="gemm bf16 forward")
    if ret:
        return dict(x=x, w=w, b=b, resid=resid, gate=ge, out=got, guard=guard, e=e, A=A, ref=ref, name=name, where=where)


def _both(*a, **k):
    for grid in (True, False):
        run_linear(*a, grid=grid, **k)


# ------------------------------------------------------------------------------------------------ shapes and dispatch
@pytest.mark.parametrize("N", [8, 64, 72, 120, 128, 136, 184, 192, 200, 256, 264, 384])
def test_tile_width_selection(N):
    """Each BN branch (256 / 128 / 256 for ragged N >= 192 / 64) and both sides of each boundary."""
    _both(200, N, 136, R.EPI_BIAS)


@pytest.mark.parametrize("N", [1, 7, 130, 201])
@pytest.mark.parametrize("ldo_gap", [0, 16])
def test_n_not_a_multiple_of_8(N, ldo_gap):
    """Columns N .. N rounded to 8 are written as zeros; nothing past them."""
    _both(133, N, 72, R.EPI_BIAS, bias=False, pads=(0, 0, 0, ldo_gap))


@pytest.mark.parametrize("K", [8, 56, 64, 72, 200])
def test_k_tails(K):
    _both(130, 256, K, R.EPI_BIAS)


@pytest.mark.parametrize("N,K", [(256, 320), (128, 448), (64, 576)])
def test_stage_ring_wraps_within_a_tile(N, K):
    """num_k above the ring depth (4 / 6 / 8 stages for BN 256 / 128 / 64)."""
    assert bn_of(N) == N and math.ceil(K / 64) > {256: 4, 128: 6, 64: 8}[N]
    _both(256, N, K, R.EPI_BIAS)


@pytest.mark.parametrize("M,N,K", [(1000, 2432, 448), (1300, 3328, 320), (6000, 184, 576), (1921, 1152, 64)])
def test_ring_phase_carries_across_persistent_tiles(M, N, K):
    """More tiles than SMs and not a multiple of them: CTAs run a second tile with the ring phase of the first."""
    tiles = math.ceil(M / 128) * math.ceil(N / bn_of(N))
    assert tiles > NUM_SMS and tiles % NUM_SMS != 0
    _both(M, N, K, R.EPI_BIAS)


@pytest.mark.parametrize("M", [1, 127, 128, 129])
def test_m_tails(M):
    _both(M, 192, 72, R.EPI_BIAS)


RASTER = [(M, N) for M in (1920, 1921) for N in (2048, 1152, 1664)]


@pytest.mark.parametrize("M,N", RASTER)
def test_weight_stripe_raster_boundary(M, N):
    """The weight-stripe raster (stripes of 8 column tiles) runs for num_m >= 16 and num_n > 8. M = 1920 / 1921 give
    num_m = 15 / 16; N = 2048 gives 8 column tiles of 256 (row-group raster), N = 1152 and 1664 give 9 and 13 tiles of 128
    (with M = 1921: striped, with a partial last stripe of 1 and 5 tiles)."""
    num_m, num_n = math.ceil(M / 128), math.ceil(N / bn_of(N))
    assert (num_m, num_n) in {(15, 8), (16, 8), (15, 9), (16, 9), (15, 13), (16, 13)}
    _both(M, N, 64, R.EPI_BIAS)


EPI_CASES = ([(e, b, 0) for e in (0, 1, 2, 3, 4, 7) for b in (True, False)] +
             [(e, True, gr) for e in (2, 3, 7) for gr in (1, 100, 333)])


@pytest.mark.parametrize("epi,bias,gate_rows", EPI_CASES)
def test_epilogues(epi, bias, gate_rows):
    """Every public epilogue, with and without bias; gated ones with per-row-group gates (100 divides neither 64 nor 128)
    whose row stride exceeds N."""
    _both(333, 264, 200, epi, bias=bias, gate_rows=gate_rows, gate_pad=24 if gate_rows else 0)


@pytest.mark.parametrize("epi", [0, 2, 3])
def test_strided_operands_and_output(epi):
    """ldx > K, ldw > K, ldr > N, ldo > N, with garbage in the operand gaps and sentinels in the output gaps."""
    _both(300, 384, 200, epi, pads=(24, 40, 16, 32))


def test_checkers_reject_defects_on_kernel_output():
    """The checks above fail on one-tile defects edited into a copy of a passing kernel output."""
    for grid in (True, False):
        c = run_linear(300, 384, 448, R.EPI_BIAS, pads=(0, 0, 0, 16), grid=grid, ret=True)
        check = ((lambda o: R.assert_exact(o, c["ref"], "mutant")) if grid else
                 (lambda o: R.assert_within(o, c["ref"], R.epilogue_bound(c["e"], c["A"], 448, 0, bias=c["b"])[1], "mutant")))
        check(c["out"])
        # one k-block missing from one 128 x 128 tile
        drop = c["x"][128:256, 192:256].double() @ c["w"][128:256, 192:256].double().t()
        m = c["out"].clone()
        m[128:256, 128:256] = (c["e"][128:256, 128:256] - drop + c["b"][128:256].double()).float().bfloat16()
        # two 8-column groups swapped in one tile's rows; a row shifted by one
        s = c["out"].clone()
        s[0:64, 8:16], s[0:64, 16:24] = c["out"][0:64, 16:24], c["out"][0:64, 8:16]
        r = c["out"].clone()
        r[129] = c["out"][130]
        for mutant in (m, s, r):
            with pytest.raises(AssertionError):
                check(mutant)
        # one element written past N (row 0, column N of the output rows, which start at row 2 of the buffer)
        c["guard"].buf.view(torch.int16)[2 * 400 + 384] ^= 1
        with pytest.raises(AssertionError):
            c["guard"].assert_untouched("mutant")


# ------------------------------------------------------------------------------------------------ fvb_linear_bf16_sp / _aux
def _plain(x, w, b, resid, gate, epi, M, N, K):
    out = torch.empty(M, N, dtype=torch.float32 if epi == 2 else torch.bfloat16, device=DEV)
    _check(_lib().fvb_linear_bf16(_p(x), c_int64(x.stride(0)), _p(w), c_int64(w.stride(0)), _p(b), _p(out), c_int64(N),
                                  _p(resid), c_int64(N), _f32p(gate), c_int(0), c_int64(0), c_int(M), c_int(N), c_int(K),
                                  c_int(epi), _s()))
    return out


@pytest.mark.parametrize("grid", [True, False])
def test_sp_segmented_a_and_column_block_offsets(grid):
    """x read as 3 segments of 128 columns that live apart; output heads scattered through out_col_offsets into a send
    buffer: both bit-equal to the plain call, the send buffer's other slots untouched."""
    M, N, K, seg = 300, 384, 384, 128
    g = torch.Generator(device=DEV).manual_seed(11)
    mk = (lambda s: R.grid_bf16(s, g, DEV)) if grid else (lambda s: R.rand_bf16(s, g, DEV))
    x, w, b = mk((M, K)), mk((N, K)), mk((N,))
    resid, gate = R.rand_bf16((M, N), g, DEV), torch.randn(N, generator=g, device=DEV)
    for epi in (R.EPI_BIAS, R.EPI_GATE_BF16):
        ref = _plain(x, w, b, resid, gate, epi, M, N, K)
        # segmented A: [3 segments][M][136], one segment per 128 columns of x
        xs = (torch.randn(K // seg, M, seg + 8, generator=g, device=DEV) * 1e3).bfloat16()
        xs[:, :, :seg] = x.view(M, K // seg, seg).transpose(0, 1)
        # send buffer [slot][M][160]; head j goes to slot perm[j] at column 16
        perm = [2, 0, 1]
        guard = R.Guarded((3, M, 160), torch.bfloat16, DEV, seed=3)
        offs = torch.tensor([perm[j] * M * 160 + 16 for j in range(3)], dtype=torch.int64, device=DEV)
        for j in range(3):
            guard.region(guard.buf[perm[j], :, 16:144])
        # plain output rows of ldo = N + 16 from row 1 of a sentinel buffer
        plain = R.Guarded((M + 2, N + 16), torch.bfloat16, DEV, seed=4)
        plain.region(plain.buf[1:M + 1, :N])
        for seg_len, col_offsets in ((seg, None), (0, offs), (seg, offs)):
            xin, ldx, sstride = (xs, seg + 8, M * (seg + 8)) if seg_len else (x, K, 0)
            if col_offsets is None:
                out, ldo = plain.buf[1:M + 1, :N], N + 16
            else:
                out, ldo = guard.buf, 160
            _check(_lib().fvb_linear_bf16_sp(_p(xin), c_int64(ldx), c_int(seg_len), c_int64(sstride), _p(w), c_int64(K),
                                             _p(b), _p(out), c_int64(ldo), _p(col_offsets), _p(resid), c_int64(N),
                                             _f32p(gate), c_int(0), c_int64(0), c_int(M), c_int(N), c_int(K), c_int(epi), _s()))
            got = out if col_offsets is None else torch.cat([guard.buf[perm[j], :, 16:144] for j in range(3)], 1)
            R.assert_exact(got, ref, f"sp seg_len={seg_len} offsets={col_offsets is not None} epi={epi}",
                           family="gemm bf16 forward (sp = plain)")
        torch.cuda.synchronize()
        guard.assert_untouched("sp send buffer")
        plain.assert_untouched("sp segmented-A output")


def test_sp_column_offsets_need_whole_heads():
    from fastvideo_b200.ops import FvbError
    M, N, K = 64, 200, 64
    x, w = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV), torch.zeros(N, K, dtype=torch.bfloat16, device=DEV)
    out = R.Guarded((M, 256), torch.bfloat16, DEV, seed=6)  # a refused call writes nothing
    offs = torch.zeros(2, dtype=torch.int64, device=DEV)
    with pytest.raises(FvbError):
        _check(_lib().fvb_linear_bf16_sp(_p(x), c_int64(K), c_int(0), c_int64(0), _p(w), c_int64(K), _p(None), _p(out.buf),
                                         c_int64(256), _p(offs), _p(None), c_int64(0), _f32p(None), c_int(0), c_int64(0),
                                         c_int(M), c_int(N), c_int(K), c_int(0), _s()))
    torch.cuda.synchronize()
    out.assert_untouched("refused sp call")


@pytest.mark.parametrize("epi", [1, 2, 3])
def test_aux_output_and_sentinels(epi):
    """fvb_linear_bf16_aux: out equals the plain call's bits, aux the plain FVB_EPI_BIAS bits; neither writes past N."""
    M, N, K = 333, 264, 200
    g = torch.Generator(device=DEV).manual_seed(epi)
    x, w, b = R.rand_bf16((M, K), g, DEV), R.rand_bf16((N, K), g, DEV, K ** -0.5), R.rand_bf16((N,), g, DEV)
    resid, gate = R.rand_bf16((M, N), g, DEV), torch.randn(N, generator=g, device=DEV)
    if epi == 1:
        resid = gate = None
    ref = _plain(x, w, b, resid, gate, epi, M, N, K)
    y = _plain(x, w, b, None, None, 0, M, N, K)
    og = R.Guarded((M + 2, N + 8), ref.dtype, DEV, seed=1)
    ag = R.Guarded((M + 2, N + 24), torch.bfloat16, DEV, seed=2)
    out, aux = og.region(og.buf[:M, :N]), ag.region(ag.buf[:M, :N])
    _check(_lib().fvb_linear_bf16_aux(_p(x), c_int64(K), _p(w), c_int64(K), _p(b), _p(out), c_int64(N + 8), _p(resid),
                                      c_int64(N), _f32p(gate), c_int(0), c_int64(0), _p(aux), c_int64(N + 24), c_int(M),
                                      c_int(N), c_int(K), c_int(epi), _s()))
    R.assert_exact(out, ref, f"aux out epi={epi}", family="gemm bf16 forward (aux = plain)")
    R.assert_exact(aux, y, f"aux y epi={epi}", family="gemm bf16 forward (aux = plain)")
    og.assert_untouched("aux out")
    ag.assert_untouched("aux buffer")


# ------------------------------------------------------------------------------------------------ fvb_gemm_batched_bf16
BATCHED = ([(bt, 200, 136, 72, d) for bt in (1, 3, 6) for d in (0.0, 1.0, math.sqrt(128))] +
           [(6, 45, 45, 128, math.sqrt(128)), (6, 45, 128, 45, 0.0), (3, 45, 45, 8, 0.0)])


@pytest.mark.parametrize("batch,M,N,K,div", BATCHED)
def test_gemm_batched(batch, M, N, K, div):
    """Batch strides larger than the matrices, M / N / K off the tile, div in {0, 1, sqrt(128)}, and the VSA compression
    shapes (nblk x nblk x 128 scores; out_c = attn @ v_c with K = nblk)."""
    N8 = (N + 7) // 8 * 8
    lda, ldb, ldo = (K + 7) // 8 * 8 + 8, (K + 7) // 8 * 8 + 16, N8 + 8
    sa, sb, so = M * lda + 64, N * ldb + 128, (M + 3) * ldo
    epi = R.EPI_DIV if div not in (0.0, 1.0) else R.EPI_BIAS
    for grid in (True, False):
        g = torch.Generator(device=DEV).manual_seed(batch * 100 + M + N + K)
        abuf = (torch.randn(batch * sa, generator=g, device=DEV) * 1e3).bfloat16()
        bbuf = (torch.randn(batch * sb, generator=g, device=DEV) * 1e3).bfloat16()
        a = abuf.as_strided((batch, M, K), (sa, lda, 1))
        b = bbuf.as_strided((batch, N, K), (sb, ldb, 1))
        a.copy_(R.grid_bf16(a.shape, g, DEV) if grid else R.rand_bf16(a.shape, g, DEV))
        b.copy_(R.grid_bf16(b.shape, g, DEV) if grid else R.rand_bf16(b.shape, g, DEV))
        guard = R.Guarded((batch * so + 64,), torch.bfloat16, DEV, seed=batch)
        out = guard.region(guard.buf.as_strided((batch, M, N8), (so, ldo, 1)))
        _check(_lib().fvb_gemm_batched_bf16(_p(a), c_int64(lda), c_int64(sa), _p(b), c_int64(ldb), c_int64(sb), _p(out),
                                            c_int64(ldo), c_int64(so), c_int(M), c_int(N), c_int(K), c_int(batch),
                                            c_float(div), _s()))
        name = f"batched {batch}x{M}x{N}x{K} div={div:.3f} {'grid' if grid else 'random'}"
        guard.assert_untouched(name)
        assert bool((out[:, :, N:] == 0).all()), name
        e, A = R.exact_gemm(a, b)
        if grid:
            R.assert_exact(out[:, :, :N], R.epilogue_ref(e.float(), epi, div=div), name, family="gemm batched")
        else:
            ref, bound = R.epilogue_bound(e, A, K, epi, div=div)
            R.assert_within(out[:, :, :N], ref, bound, name, family="gemm batched")


# ------------------------------------------------------------------------------------------------ fvb_gemm_f32out
@pytest.mark.parametrize("HW", [1350, 1])
def test_gemm_f32out_vae_mid_block(HW):
    """The VAE mid-block logits: q and k column slices of a [HW, 3C] buffer, C = 384, HW not a multiple of 8."""
    C = 384
    N8 = (HW + 7) // 8 * 8
    scale = 1.0 / math.sqrt(C)
    for grid in (True, False):
        g = torch.Generator(device=DEV).manual_seed(HW)
        qkv = R.grid_bf16((HW, 3 * C), g, DEV) if grid else R.rand_bf16((HW, 3 * C), g, DEV)
        a, b = qkv[:, :C], qkv[:, C:2 * C]
        guard = R.Guarded((HW + 3, N8 + 8), torch.float32, DEV, seed=5)
        out = guard.region(guard.buf[1:HW + 1, :N8])
        _check(_lib().fvb_gemm_f32out(_p(a), c_int64(3 * C), _p(b), c_int64(3 * C), _f32p(out), c_int64(N8 + 8), c_int(HW),
                                      c_int(HW), c_int(C), c_float(scale), _s()))
        name = f"f32out HW={HW} {'grid' if grid else 'random'}"
        guard.assert_untouched(name)
        assert bool((out[:, HW:] == 0).all()), name
        e, A = R.exact_gemm(a, b)
        if grid:
            R.assert_exact(out[:, :HW], R.epilogue_ref(e.float(), R.EPI_SCALE_F32, scale=scale), name, family="gemm f32out")
        else:
            ref, bound = R.epilogue_bound(e, A, C, R.EPI_SCALE_F32, scale=scale)
            R.assert_within(out[:, :HW], ref, bound, name, family="gemm f32out")


# ------------------------------------------------------------------------------------------------ dgrad / wgrad / dgrad-GELU
BWD_SHAPES = [(1, 256, 512), (333, 200, 136), (1000, 64, 64), (777, 128, 128), (500, 136, 256), (600, 72, 200),
              (65, 72, 8), (129, 8, 72), (1000, 1536, 1536), (1000, 8960, 1536), (9450, 5120, 5120)]


@pytest.mark.parametrize("M,N,K", BWD_SHAPES)
def test_dgrad_wgrad_dgrad_gelu(M, N, K):
    """dx = dy w, dw = dy^T x and dh = bf16(dx) * gelu'(h) with the transposed-operand tails (N, M off the 64 grid)."""
    for grid in (True, False):
        g = torch.Generator(device=DEV).manual_seed(M + N + K + grid)
        x = _operand(M, K, 16, g, grid)
        w = _operand(N, K, 8, g, grid, K ** -0.5)
        dy = _operand(M, N, 24, g, grid)
        # h spans the GELU's cancellation region (down to -8) on its own grid
        h = (torch.randint(-32, 33, (M, K), generator=g, device=DEV) / 4.0).bfloat16() if grid else R.rand_bf16((M, K), g, DEV, 2.0)
        tag = "grid" if grid else "random"
        outs = {}
        for kind, rows in (("dgrad", M), ("wgrad", N), ("dgrad-gelu", M)):
            guard = R.Guarded((rows + 2, K + 24), torch.bfloat16, DEV, seed=rows)
            o = guard.region(guard.buf[1:rows + 1, :K])
            ldo = K + 24
            if kind == "dgrad":
                rc = _lib().fvb_linear_dgrad_bf16(_p(dy), c_int64(dy.stride(0)), _p(w), c_int64(w.stride(0)), _p(o),
                                                  c_int64(ldo), c_int(M), c_int(N), c_int(K), _s())
            elif kind == "wgrad":
                rc = _lib().fvb_linear_wgrad_bf16(_p(dy), c_int64(dy.stride(0)), _p(x), c_int64(x.stride(0)), _p(o),
                                                  c_int64(ldo), c_int(M), c_int(N), c_int(K), _s())
            else:
                rc = _lib().fvb_linear_dgrad_gelu_bf16(_p(dy), c_int64(dy.stride(0)), _p(w), c_int64(w.stride(0)), _p(h),
                                                       c_int64(K), _p(o), c_int64(ldo), c_int(M), c_int(N), c_int(K), _s())
            _check(rc)
            guard.assert_untouched(f"{kind} {M}x{N}x{K} {tag}")
            outs[kind] = o
        ed, Ad = R.exact_gemm(dy, w.t())
        ew, Aw = R.exact_gemm(dy.t(), x.t())
        where = lambda idx: R.gemm_coords(idx, bn_of(K))
        for kind, e, A, red in (("dgrad", ed, Ad, N), ("wgrad", ew, Aw, M)):
            name = f"{kind} {M}x{N}x{K} {tag}"
            if grid:
                R.assert_exact(outs[kind], e.float().bfloat16(), name, where, family=f"gemm {kind}")
            else:
                ref, bound = R.epilogue_bound(e, A, red, R.EPI_BIAS)
                R.assert_within(outs[kind], ref, bound, name, where, family=f"gemm {kind}")
        name = f"dgrad-gelu {M}x{N}x{K} {tag}"
        if grid:
            d = ed.float().bfloat16().double()
            g64 = R.gelu_grad64(h)
            ref = d * g64
            derr = d.abs() * R.gelu_grad_err(h)
            bound = R.ulp_bf16(ref.abs() + derr) + derr + 1e-38
            R.assert_within(outs["dgrad-gelu"], ref, bound, name, where, family="gemm dgrad-gelu, grid inputs")
        else:
            ref, bound = R.dgrad_gelu_bound(ed, Ad, N, h)
            R.assert_within(outs["dgrad-gelu"], ref, bound, name, where, family="gemm dgrad-gelu")
