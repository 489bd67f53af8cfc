"""Python entry points over the C ABI (include/fvb200.h). Tensors are torch CUDA tensors; outputs are
allocated here (torch is the device allocator) and every call is issued on torch's current stream."""
from __future__ import annotations

from ctypes import c_float, c_int, c_int64, c_void_p, POINTER, cast

import os

import torch

from ._lib import check, lib, ptr, stream_ptr, FvbError

EPI_BIAS = 0
EPI_BIAS_GELU_TANH = 1
EPI_RESID_GATE_F32 = 2
EPI_RESID_GATE_BF16 = 3
EPI_RESID_BF16 = 4
EPI_RESID_GATE_BF16R = 7  # bf16 gate tensors: the gated product is rounded to bf16 before the residual add


def _require_cuda_bf16(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise FvbError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != torch.bfloat16:
        raise FvbError(f"{name} must be bf16, got {t.dtype}")


def linear(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, epilogue: int = EPI_BIAS,
           resid: torch.Tensor | None = None, gate: torch.Tensor | None = None,
           out: torch.Tensor | None = None, gate_rows: int = 0) -> torch.Tensor:
    """out = epilogue(x @ w.T + bias). x: [..., K] (rows may be strided), w: [N, K].
    gate: fp32 [N], or [G, N] with gate_rows > 0 (row r uses gate[r // gate_rows])."""
    _require_cuda_bf16(x, "x")
    _require_cuda_bf16(w, "w")
    K = x.shape[-1]
    N = w.shape[0]
    x2 = x.reshape(-1, K)
    if x2.stride(1) != 1:
        x2 = x2.contiguous()
    M = x2.shape[0]
    out_dtype = torch.float32 if epilogue == EPI_RESID_GATE_F32 else torch.bfloat16
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    o2 = out.reshape(M, N)
    assert o2.dtype == out_dtype and o2.stride(1) == 1
    r2 = None
    if resid is not None:
        _require_cuda_bf16(resid, "resid")
        r2 = resid.reshape(M, N)
        assert r2.stride(1) == 1
    gate_stride = _check_grouped(gate, N, gate_rows, M, "gate")
    if bias is not None:
        _require_cuda_bf16(bias, "bias")
        assert bias.is_contiguous() and bias.numel() == N
    assert w.stride(1) == 1
    check(lib().fvb_linear_bf16(ptr(x2), c_int64(x2.stride(0)), ptr(w), c_int64(w.stride(0)), ptr(bias), ptr(o2),
                                c_int64(o2.stride(0)), ptr(r2), c_int64(r2.stride(0) if r2 is not None else 0),
                                cast(ptr(gate), POINTER(c_float)), c_int(gate_rows), c_int64(gate_stride), c_int(M), c_int(N),
                                c_int(K), c_int(epilogue), stream_ptr()))
    return out.reshape(*x.shape[:-1], N)


def linear_bwd(x: torch.Tensor, w: torch.Tensor, dy: torch.Tensor, need_dx: bool = True, need_dw: bool = True,
               need_db: bool = False):
    """Backward of y = linear(x, w, bias) (FVB_EPI_BIAS) on the bf16 wgmma GEMM: x [M, K], w [N, K], dy [M, N] bf16 2-D views
    with unit inner stride (row strides multiples of 8: column slices of fused buffers are read in place); K a multiple of
    8 for dx / dw, N for db. Returns (dx [M, K], dw [N, K], db [N]), each fp32-accumulated and rounded to bf16 once, with
    None for what was not requested (and not launched): fvb_linear_dgrad_bf16, fvb_linear_wgrad_bf16, fvb_bias_grad_bf16."""
    for n, t in (("x", x), ("w", w), ("dy", dy)):
        _require_cuda_bf16(t, n)
        if t.dim() != 2 or t.stride(1) != 1:
            raise FvbError(f"linear_bwd: {n} must be a 2-D view with unit inner stride")
    M, K = x.shape
    N = w.shape[0]
    if w.shape[1] != K or dy.shape != (M, N):
        raise FvbError(f"linear_bwd: x [M, K], w [N, K], dy [M, N] (got {tuple(x.shape)}, {tuple(w.shape)}, {tuple(dy.shape)})")
    dx = dw = db = None
    if need_dx:
        dx = torch.empty((M, K), dtype=torch.bfloat16, device=x.device)
        check(lib().fvb_linear_dgrad_bf16(ptr(dy), c_int64(dy.stride(0)), ptr(w), c_int64(w.stride(0)), ptr(dx), c_int64(K),
                                          c_int(M), c_int(N), c_int(K), stream_ptr()))
    if need_dw:
        dw = torch.empty((N, K), dtype=torch.bfloat16, device=x.device)
        check(lib().fvb_linear_wgrad_bf16(ptr(dy), c_int64(dy.stride(0)), ptr(x), c_int64(x.stride(0)), ptr(dw), c_int64(K),
                                          c_int(M), c_int(N), c_int(K), stream_ptr()))
    if need_db:
        db = torch.empty(N, dtype=torch.bfloat16, device=x.device)
        ws = _workspace(int(lib().fvb_bias_grad_bf16_workspace_bytes(c_int(M), c_int(N))), x.device)
        check(lib().fvb_bias_grad_bf16(ptr(dy), c_int64(dy.stride(0)), ptr(db), _f32p(ws), c_int64(ws.numel()), c_int(M),
                                       c_int(N), stream_ptr()))
    return dx, dw, db


class LinearFn(torch.autograd.Function):
    """y = bf16(x w^T + b) over rows of x [M, K], w bf16 [N, K], b bf16 [N] or None: forward on fvb_linear_bf16 (the output
    of the no-grad call, bit for bit), backward on linear_bwd for the inputs that need a gradient (nothing else is
    launched). An fp32 bias is cast outside, so torch differentiates the cast."""

    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        return linear(x, w, b)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dy = dy.to(torch.bfloat16)
        if dy.stride(1) != 1 or dy.stride(0) % 8 != 0:
            dy = dy.contiguous()
        need_dx, need_dw, need_db = ctx.needs_input_grad
        return linear_bwd(x, w, dy, need_dx, need_dw, need_db)


def _check_2d(t: torch.Tensor, name: str, shape, dtypes=(torch.bfloat16,)) -> None:
    if not t.is_cuda or t.dtype not in dtypes or t.dim() != 2 or t.stride(1) != 1 or tuple(t.shape) != tuple(shape):
        raise FvbError(f"{name} must be a CUDA {'/'.join(map(str, dtypes))} [{shape[0]}, {shape[1]}] view with unit inner stride")


def linear_aux(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None, epilogue: int,
               resid: torch.Tensor | None = None, gate: torch.Tensor | None = None, gate_rows: int = 0):
    """fvb_linear_bf16_aux: `linear` (bf16 weight, EPI_BIAS_GELU_TANH / EPI_RESID_GATE_F32 / EPI_RESID_GATE_BF16 /
    EPI_RESID_GATE_BF16R) that also returns the bf16 y = bf16(x @ w.T + bias) its epilogue consumes. x: [M, K] with unit
    inner stride; one gate vector (gate_rows 0), or [G, N] with gate_rows > 0 for EPI_RESID_GATE_BF16R. Returns (out, aux);
    out has the bits of `linear`, aux those of `linear` with EPI_BIAS."""
    if gate_rows != 0 and epilogue != EPI_RESID_GATE_BF16R:
        raise FvbError("linear_aux takes per-row-group gates (gate_rows > 0) with EPI_RESID_GATE_BF16R only")
    _require_cuda_bf16(x, "x")
    _require_cuda_bf16(w, "w")
    if x.dim() != 2 or x.stride(1) != 1 or w.stride(1) != 1:
        raise FvbError("linear_aux: x [M, K] and w [N, K] with unit inner stride")
    M, K = x.shape
    N = w.shape[0]
    out = torch.empty((M, N), dtype=torch.float32 if epilogue == EPI_RESID_GATE_F32 else torch.bfloat16, device=x.device)
    aux = torch.empty((M, N), dtype=torch.bfloat16, device=x.device)
    if resid is not None:
        _check_2d(resid, "resid", (M, N))
    gate_stride = _check_grouped(gate, N, gate_rows, M, "gate")
    if bias is not None:
        _require_cuda_bf16(bias, "bias")
        assert bias.is_contiguous() and bias.numel() == N
    check(lib().fvb_linear_bf16_aux(ptr(x), c_int64(x.stride(0)), ptr(w), c_int64(w.stride(0)), ptr(bias), ptr(out),
                                    c_int64(N), ptr(resid), c_int64(resid.stride(0) if resid is not None else 0), _f32p(gate),
                                    c_int(gate_rows), c_int64(gate_stride), ptr(aux), c_int64(N), c_int(M), c_int(N), c_int(K),
                                    c_int(epilogue), stream_ptr()))
    return out, aux


def linear_dgrad_gelu(dy: torch.Tensor, w: torch.Tensor, h: torch.Tensor) -> torch.Tensor:
    """fvb_linear_dgrad_gelu_bf16: dh = bf16(bf16(dy @ w) * gelu_tanh'(h)) for y = gelu_tanh(h) @ w.T (+ b). dy [M, N],
    w [N, K], h [M, K] bf16 2-D views with unit inner stride. Returns dh [M, K]."""
    M, N = dy.shape
    K = w.shape[1]
    _check_2d(dy, "dy", (M, N))
    _check_2d(w, "w", (N, K))
    _check_2d(h, "h", (M, K))
    dh = torch.empty((M, K), dtype=torch.bfloat16, device=dy.device)
    check(lib().fvb_linear_dgrad_gelu_bf16(ptr(dy), c_int64(dy.stride(0)), ptr(w), c_int64(w.stride(0)), ptr(h),
                                           c_int64(h.stride(0)), ptr(dh), c_int64(K), c_int(M), c_int(N), c_int(K), stream_ptr()))
    return dh


def resid_gate_bwd(dout: torch.Tensor, y: torch.Tensor, gate: torch.Tensor, need_db: bool = True):
    """fvb_resid_gate_bwd: backward of out = resid + y * gate (EPI_RESID_GATE_F32 / _BF16). dout fp32 or bf16 [M, N], y the
    saved bf16 [M, N] (2-D views, unit inner stride), gate fp32 [N]. Returns (dy bf16 [M, N], d_gate fp32 [N], db bf16 [N] or
    None); the residual's gradient is dout."""
    M, N = y.shape
    _check_2d(dout, "dout", (M, N), (torch.float32, torch.bfloat16))
    _check_2d(y, "y", (M, N))
    if gate.dtype != torch.float32 or not gate.is_contiguous() or gate.numel() != N:
        raise FvbError(f"resid_gate_bwd: gate must be a contiguous fp32 [{N}] tensor")
    dy = torch.empty((M, N), dtype=torch.bfloat16, device=y.device)
    d_gate = torch.empty(N, dtype=torch.float32, device=y.device)
    db = torch.empty(N, dtype=torch.bfloat16, device=y.device) if need_db else None
    ws = _workspace(int(lib().fvb_resid_gate_bwd_workspace_bytes(c_int(M), c_int(N))), y.device)
    check(lib().fvb_resid_gate_bwd(ptr(dout), c_int(int(dout.dtype == torch.float32)), c_int64(dout.stride(0)), ptr(y),
                                   c_int64(y.stride(0)), _f32p(gate), ptr(dy), c_int64(N), _f32p(d_gate), ptr(db), _f32p(ws),
                                   c_int64(ws.numel()), c_int(M), c_int(N), stream_ptr()))
    return dy, d_gate, db


def layernorm_modulate_bwd(x: torch.Tensor, dn: torch.Tensor, scale: torch.Tensor | None = None,
                           weight: torch.Tensor | None = None, round_ln: bool = False, gin: torch.Tensor | None = None,
                           eps: float = 1e-6):
    """fvb_layernorm_modulate_bwd: backward of layernorm_modulate(x, scale, shift, round_ln=...) (scale given) or of
    layernorm_modulate(x, weight=weight, bias=...) (weight given), one (scale, shift) for all rows. x bf16 or fp32 [M, D],
    dn bf16 [M, D]; gin: optional fp32 / bf16 [M, D] gradient added into dx. Returns (dx in x's dtype, d_scale or d_weight
    fp32 [D], d_shift or d_bias fp32 [D])."""
    M, D = x.shape
    _check_2d(x, "x", (M, D), (torch.float32, torch.bfloat16))
    _check_2d(dn, "dn", (M, D))
    if (scale is None) == (weight is None):
        raise FvbError("layernorm_modulate_bwd takes scale (modulation) or weight (affine), not both")
    if round_ln and weight is not None:
        raise FvbError("layernorm_modulate_bwd: round_ln is the modulation form's (the affine forward rounds after w, b)")
    gain = scale if scale is not None else weight
    if gain.dtype != torch.float32 or not gain.is_contiguous() or gain.numel() != D:
        raise FvbError(f"layernorm_modulate_bwd: scale / weight must be a contiguous fp32 [{D}] tensor")
    if gin is not None:
        _check_2d(gin, "gin", (M, D), (torch.float32, torch.bfloat16))
    dx = torch.empty((M, D), dtype=x.dtype, device=x.device)
    d_gain = torch.empty(D, dtype=torch.float32, device=x.device)
    d_off = torch.empty(D, dtype=torch.float32, device=x.device)
    ws = _workspace(int(lib().fvb_layernorm_modulate_bwd_workspace_bytes(c_int(M), c_int(D))), x.device)
    check(lib().fvb_layernorm_modulate_bwd(ptr(x), c_int(int(x.dtype == torch.float32)), c_int64(x.stride(0)), ptr(dn),
                                           c_int64(dn.stride(0)), _f32p(gain), c_int(int(scale is not None)), c_int(int(round_ln)),
                                           ptr(gin), c_int(int(gin is not None and gin.dtype == torch.float32)),
                                           c_int64(gin.stride(0) if gin is not None else 0), ptr(dx), c_int64(D), _f32p(d_gain),
                                           _f32p(d_off), _f32p(ws), c_int64(ws.numel()), c_int(M), c_int(D), c_float(eps),
                                           stream_ptr()))
    return dx, d_gain, d_off


def _check_groups(t: torch.Tensor, name: str, D: int, G: int) -> None:
    if t.dtype != torch.float32 or t.dim() != 2 or t.shape != (G, D) or t.stride(1) != 1 or t.data_ptr() % 16:
        raise FvbError(f"{name} must be an fp32 [{G}, {D}] view with unit inner stride, 16-byte aligned")


def layernorm_modulate_grouped_bwd(x: torch.Tensor, dn: torch.Tensor, scale: torch.Tensor, mod_rows: int,
                                   gin: torch.Tensor | None = None, eps: float = 1e-6):
    """fvb_layernorm_modulate_grouped_bwd: backward of layernorm_modulate(x, scale, shift, round_ln=True, mod_rows=R,
    mod_bf16=True) (one modulation row per group of R rows, bf16 arithmetic). x, dn bf16 [M, D]; scale fp32 [G, D] (G =
    ceil(M / R); any row stride that is a multiple of 4, e.g. a slice of the [F, 6, D] modulation); gin: optional fp32 /
    bf16 [M, D] gradient added into dx. Returns (dx bf16 [M, D], d_scale fp32 [G, D], d_shift fp32 [G, D])."""
    M, D = x.shape
    _check_2d(x, "x", (M, D))
    _check_2d(dn, "dn", (M, D))
    if mod_rows <= 0:
        raise FvbError("layernorm_modulate_grouped_bwd: mod_rows must be > 0")
    G = -(-M // mod_rows)
    _check_groups(scale, "scale", D, G)
    if gin is not None:
        _check_2d(gin, "gin", (M, D), (torch.float32, torch.bfloat16))
    dx = torch.empty((M, D), dtype=torch.bfloat16, device=x.device)
    d_scale = torch.empty((G, D), dtype=torch.float32, device=x.device)
    d_shift = torch.empty((G, D), dtype=torch.float32, device=x.device)
    ws = _workspace(int(lib().fvb_layernorm_modulate_grouped_bwd_workspace_bytes(c_int(M), c_int(mod_rows), c_int(D))), x.device)
    check(lib().fvb_layernorm_modulate_grouped_bwd(ptr(x), c_int64(x.stride(0)), ptr(dn), c_int64(dn.stride(0)), _f32p(scale),
                                                   c_int(mod_rows), c_int64(scale.stride(0)), ptr(gin),
                                                   c_int(int(gin is not None and gin.dtype == torch.float32)),
                                                   c_int64(gin.stride(0) if gin is not None else 0), ptr(dx), c_int64(D),
                                                   _f32p(d_scale), _f32p(d_shift), c_int64(D), _f32p(ws), c_int64(ws.numel()),
                                                   c_int(M), c_int(D), c_float(eps), stream_ptr()))
    return dx, d_scale, d_shift


def resid_gate_grouped_bwd(dout: torch.Tensor, y: torch.Tensor, gate: torch.Tensor, gate_rows: int, need_db: bool = True):
    """fvb_resid_gate_grouped_bwd: backward of out = bf16(resid + bf16(y * gate[r // gate_rows])) (EPI_RESID_GATE_BF16R with
    gate_rows > 0). dout, y bf16 [M, N] (2-D views, unit inner stride), gate fp32 [G, N] (row stride a multiple of 4).
    Returns (dy bf16 [M, N], d_gate fp32 [G, N], db bf16 [N] or None); the residual's gradient is dout."""
    M, N = y.shape
    _check_2d(dout, "dout", (M, N))
    _check_2d(y, "y", (M, N))
    if gate_rows <= 0:
        raise FvbError("resid_gate_grouped_bwd: gate_rows must be > 0")
    G = -(-M // gate_rows)
    _check_groups(gate, "gate", N, G)
    dy = torch.empty((M, N), dtype=torch.bfloat16, device=y.device)
    d_gate = torch.empty((G, N), dtype=torch.float32, device=y.device)
    db = torch.empty(N, dtype=torch.bfloat16, device=y.device) if need_db else None
    ws = _workspace(int(lib().fvb_resid_gate_grouped_bwd_workspace_bytes(c_int(M), c_int(gate_rows), c_int(N))), y.device)
    check(lib().fvb_resid_gate_grouped_bwd(ptr(dout), c_int64(dout.stride(0)), ptr(y), c_int64(y.stride(0)), _f32p(gate),
                                           c_int(gate_rows), c_int64(gate.stride(0)), ptr(dy), c_int64(N), _f32p(d_gate),
                                           c_int64(N), ptr(db), _f32p(ws), c_int64(ws.numel()), c_int(M), c_int(N), stream_ptr()))
    return dy, d_gate, db


def rmsnorm_rope_bwd(x0, w0, dy0, dx0, x1, w1, dy1, dx1, cos, sin, rope_row=None, head_dim: int = 128, eps: float = 1e-6,
                     want_dw: bool = True):
    """fvb_rmsnorm_rope_bwd: backward of rmsnorm_rope_(x0, w0, x1, w1, cos, sin, rope_row) (bf16 weights) into dx0 / dx1,
    which may be column slices of a fused gradient buffer. x*, dy*, dx*: bf16 [M, D] 2-D views with unit inner stride (x1 /
    dy1 / dx1 None: one tensor); cos / sin fp32 [S_pos, head_dim]. Returns (dw0, dw1) bf16 [D] (None without want_dw)."""
    M, D = x0.shape
    for n, t in (("x0", x0), ("dy0", dy0), ("dx0", dx0)) + ((("x1", x1), ("dy1", dy1), ("dx1", dx1)) if x1 is not None else ()):
        _check_2d(t, n, (M, D))
    for n, w in (("w0", w0), ("w1", w1 if x1 is not None else w0)):
        if w.dtype != torch.bfloat16 or not w.is_contiguous() or w.numel() != D:
            raise FvbError(f"rmsnorm_rope_bwd: {n} must be a contiguous bf16 [{D}] tensor (fp32 RMSNorm weights have no backward)")
    if cos.dtype != torch.float32 or sin.dtype != torch.float32 or not cos.is_contiguous() or not sin.is_contiguous():
        raise FvbError("rmsnorm_rope_bwd: cos / sin must be contiguous fp32 tables")
    if rope_row is not None:
        _check_i32(rope_row, "rope_row", M)
    dw0 = torch.empty(D, dtype=torch.bfloat16, device=x0.device) if want_dw else None
    dw1 = torch.empty(D, dtype=torch.bfloat16, device=x0.device) if want_dw and x1 is not None else None
    ws = _workspace(int(lib().fvb_rmsnorm_rope_bwd_workspace_bytes(c_int(M), c_int(D))), x0.device) if want_dw else None
    ld = lambda t: c_int64(t.stride(0) if t is not None else 0)
    check(lib().fvb_rmsnorm_rope_bwd(ptr(x0), ld(x0), ptr(w0), ptr(dy0), ld(dy0), ptr(dx0), ld(dx0), ptr(dw0), ptr(x1), ld(x1),
                                     ptr(w1 if x1 is not None else None), ptr(dy1), ld(dy1), ptr(dx1), ld(dx1), ptr(dw1),
                                     _f32p(cos), _f32p(sin), _i32p(rope_row), _f32p(ws),
                                     c_int64(ws.numel() if ws is not None else 0), c_int(M), c_int(D), c_int(head_dim),
                                     c_float(eps), stream_ptr()))
    return dw0, dw1


FP8_E4M3_MAX = 448.0


def quantize_fp8_rows(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """fvb_quantize_fp8_rows: bf16 [M, K] (rows may be strided; K % 8 == 0) -> (q float8_e4m3fn [M, K], scale fp32 [M])
    with x[r] ~= q[r] * scale[r]. q's row stride is K rounded up to 16 (16-byte rows, what fvb_linear_fp8 loads)."""
    _require_cuda_bf16(x, "x")
    if x.dim() != 2 or x.stride(1) != 1:
        raise FvbError("x must be a 2-D view with unit inner stride")
    M, K = x.shape
    ldq = (K + 15) // 16 * 16
    q = torch.empty((M, ldq), dtype=torch.float8_e4m3fn, device=x.device)
    scale = torch.empty((M,), dtype=torch.float32, device=x.device)
    check(lib().fvb_quantize_fp8_rows(ptr(x), c_int64(x.stride(0)), c_int(M), c_int(K), ptr(q), c_int64(ldq), _f32p(scale),
                                      stream_ptr()))
    return q[:, :K], scale


class Fp8Weight:
    """A linear weight w[N, K] held as e4m3 rows with one fp32 scale per output channel (w ~= q * scale[:, None])."""

    def __init__(self, q: torch.Tensor, scale: torch.Tensor):
        if q.dtype != torch.float8_e4m3fn or q.dim() != 2 or q.stride(1) != 1 or q.stride(0) % 16 != 0:
            raise FvbError("Fp8Weight.q must be float8_e4m3fn [N, K] with 16-byte-aligned rows")
        if scale.dtype != torch.float32 or scale.shape != (q.shape[0],) or not scale.is_contiguous():
            raise FvbError("Fp8Weight.scale must be fp32 [N] contiguous")
        self.q, self.scale = q, scale

    @classmethod
    def quantize(cls, w: torch.Tensor) -> "Fp8Weight":
        """bf16 [N, K] -> per-output-channel e4m3 (the same row quantisation as the activations)."""
        return cls(*quantize_fp8_rows(w))

    @property
    def shape(self):
        return self.q.shape

    @property
    def device(self):
        return self.q.device

    def dequantize(self) -> torch.Tensor:
        """fp32 [N, K] values the GEMM multiplies with (q * scale)."""
        return self.q.float() * self.scale[:, None]


def linear_fp8(x: torch.Tensor, w: Fp8Weight, bias: torch.Tensor | None = None, epilogue: int = EPI_BIAS,
               resid: torch.Tensor | None = None, gate: torch.Tensor | None = None,
               out: torch.Tensor | None = None, gate_rows: int = 0) -> torch.Tensor:
    """`linear` with e4m3 operands: x (bf16 [..., K]) is row-quantised here (fvb_quantize_fp8_rows), then
    out = epilogue(bf16((q_x @ q_w.T) * s_x[m] * s_w[n] + bias)) by fvb_linear_fp8. Same epilogues, gate grouping and
    output dtypes as `linear`."""
    if not isinstance(w, Fp8Weight):
        raise FvbError("linear_fp8 takes an Fp8Weight (see Fp8Weight.quantize)")
    _require_cuda_bf16(x, "x")
    K = x.shape[-1]
    N = w.shape[0]
    if w.shape[1] != K:
        raise FvbError(f"x has K={K}, weight has K={w.shape[1]}")
    x2 = x.reshape(-1, K)
    if x2.stride(1) != 1 or x2.stride(0) % 8 != 0:
        x2 = x2.contiguous()
    M = x2.shape[0]
    xq, xs = quantize_fp8_rows(x2)
    out_dtype = torch.float32 if epilogue == EPI_RESID_GATE_F32 else torch.bfloat16
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    o2 = out.reshape(M, N)
    assert o2.dtype == out_dtype and o2.stride(1) == 1
    r2 = None
    if resid is not None:
        _require_cuda_bf16(resid, "resid")
        r2 = resid.reshape(M, N)
        assert r2.stride(1) == 1
    gate_stride = _check_grouped(gate, N, gate_rows, M, "gate")
    if bias is not None:
        _require_cuda_bf16(bias, "bias")
        assert bias.is_contiguous() and bias.numel() == N
    check(lib().fvb_linear_fp8(ptr(xq), c_int64(xq.stride(0)), _f32p(xs), ptr(w.q), c_int64(w.q.stride(0)), _f32p(w.scale),
                               ptr(bias), ptr(o2), c_int64(o2.stride(0)), ptr(r2), c_int64(r2.stride(0) if r2 is not None else 0),
                               _f32p(gate), c_int(gate_rows), c_int64(gate_stride), c_int(M), c_int(N), c_int(K),
                               c_int(epilogue), stream_ptr()))
    return out.reshape(*x.shape[:-1], N)


def quantize_int8_rows(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """fvb_quantize_int8_rows: bf16 [M, K] (rows may be strided; K % 8 == 0) -> (q int8 [M, K], scale fp32 [M]) with
    x[r] ~= q[r] * scale[r], by the rule of Int8Weight.quantize. q's row stride is K rounded up to 16 (16-byte rows, what
    fvb_linear_w8a8_sp loads)."""
    _require_cuda_bf16(x, "x")
    if x.dim() != 2 or x.stride(1) != 1:
        raise FvbError("x must be a 2-D view with unit inner stride")
    M, K = x.shape
    return _quantize_int8_rows_sp(x, M, K, x.stride(0))


def _quantize_int8_rows_sp(x: torch.Tensor, M: int, K: int, ldx: int, x_seg_len: int = 0, x_seg_stride: int = 0):
    """quantize_int8_rows on a raw buffer with linear_sp's geometry (x_seg_len / x_seg_stride: fvb_linear_bf16_sp's K
    segmentation); each row comes out contiguous."""
    _require_cuda_bf16(x, "x")
    ldq = (K + 15) // 16 * 16
    q = torch.empty((M, ldq), dtype=torch.int8, device=x.device)
    scale = torch.empty((M,), dtype=torch.float32, device=x.device)
    check(lib().fvb_quantize_int8_rows(ptr(x), c_int64(ldx), c_int(x_seg_len), c_int64(x_seg_stride), c_int(M), c_int(K),
                                       ptr(q), c_int64(ldq), _f32p(scale), stream_ptr()))
    return q[:, :K], scale


class Int8Weight:
    """A linear weight w[N, K] held as int8 rows with one fp32 scale per output channel (w ~= q * scale[:, None]). The
    activations it multiplies stay bf16 (fvb_linear_w8_sp), or, with int8_activations, are quantised to int8 with one
    scale per token (quantize_int8_rows) and multiplied on the s8 tensor cores (fvb_linear_w8a8_sp)."""

    def __init__(self, q: torch.Tensor, scale: torch.Tensor, int8_activations: bool = False):
        if q.dtype != torch.int8 or q.dim() != 2 or q.stride(1) != 1 or q.stride(0) % 16 != 0:
            raise FvbError("Int8Weight.q must be int8 [N, K] with 16-byte-aligned rows")
        if scale.dtype != torch.float32 or scale.shape != (q.shape[0],) or not scale.is_contiguous():
            raise FvbError("Int8Weight.scale must be fp32 [N] contiguous")
        if q.device != scale.device:
            raise FvbError("Int8Weight.q and scale must be on the same device")
        self.q, self.scale = q, scale
        self.int8_activations = bool(int8_activations)

    @classmethod
    def quantize(cls, w: torch.Tensor, int8_activations: bool = False) -> "Int8Weight":
        """[N, K] -> per-output-channel int8, once at load (torch, on w's device): amax = max|w[n]| (fp32),
        scale = amax / 127, q = clamp(rint(w * (127 / amax)), -127, 127); an all-zero row gets scale 1 and q = 0."""
        if w.dim() != 2:
            raise FvbError("Int8Weight.quantize takes a 2-D [N, K] weight")
        N, K = w.shape
        w32 = w.detach().float()
        amax = w32.abs().amax(dim=1)
        zero = amax == 0
        one = torch.ones_like(amax)
        inv = torch.where(zero, one, torch.full_like(amax, 127.0) / torch.where(zero, one, amax))
        scale = torch.where(zero, one, amax / 127.0)
        ld = (K + 15) // 16 * 16
        q = torch.zeros((N, ld), dtype=torch.int8, device=w.device)
        q[:, :K] = torch.clamp(torch.round(w32 * inv[:, None]), -127, 127).to(torch.int8)
        return cls(q[:, :K], scale.contiguous(), int8_activations)

    def __getitem__(self, rows) -> "Int8Weight":
        """Row slice w[a:b] (q rows and scale rows, same activation mode), e.g. the Q / K / V parts of a fused QKV weight."""
        if not isinstance(rows, slice) or rows.step not in (None, 1):
            raise FvbError("Int8Weight supports contiguous row slices only")
        return Int8Weight(self.q[rows], self.scale[rows], self.int8_activations)

    @property
    def shape(self):
        return self.q.shape

    @property
    def device(self):
        return self.q.device

    @property
    def nbytes(self) -> int:
        return self.q.numel() * self.q.element_size() + self.scale.numel() * 4

    def dequantize(self) -> torch.Tensor:
        """fp32 [N, K] values the GEMM multiplies with (q * scale)."""
        return self.q.float() * self.scale[:, None]


def linear_any(x: torch.Tensor, w, bias: torch.Tensor | None = None, epilogue: int = EPI_BIAS,
               resid: torch.Tensor | None = None, gate: torch.Tensor | None = None,
               out: torch.Tensor | None = None, gate_rows: int = 0) -> torch.Tensor:
    """`linear` for whatever the weight holds: linear_fp8 for an Fp8Weight, fvb_linear_w8_sp for an Int8Weight
    (fvb_quantize_int8_rows + fvb_linear_w8a8_sp when it is marked int8_activations), `linear` for a bf16 tensor."""
    if isinstance(w, Fp8Weight):
        return linear_fp8(x, w, bias, epilogue, resid, gate, out, gate_rows)
    if not isinstance(w, Int8Weight):
        return linear(x, w, bias, epilogue, resid, gate, out, gate_rows)
    _require_cuda_bf16(x, "x")
    K = x.shape[-1]
    N = w.shape[0]
    if w.shape[1] != K:
        raise FvbError(f"x has K={K}, weight has K={w.shape[1]}")
    x2 = x.reshape(-1, K)
    if x2.stride(1) != 1:
        x2 = x2.contiguous()
    M = x2.shape[0]
    out_dtype = torch.float32 if epilogue == EPI_RESID_GATE_F32 else torch.bfloat16
    if out is None:
        out = torch.empty((M, N), dtype=out_dtype, device=x.device)
    o2 = out.reshape(M, N)
    assert o2.dtype == out_dtype and o2.stride(1) == 1
    r2 = None
    if resid is not None:
        _require_cuda_bf16(resid, "resid")
        r2 = resid.reshape(M, N)
        assert r2.stride(1) == 1
    if bias is not None:
        _require_cuda_bf16(bias, "bias")
        assert bias.is_contiguous() and bias.numel() == N
    linear_sp(x2, M, K, x2.stride(0), w, bias, o2, o2.stride(0), epilogue, resid=r2, gate=gate, gate_rows=gate_rows)
    return out.reshape(*x.shape[:-1], N)


def _check_grouped(t, D: int, rows: int, M: int, name: str) -> int:
    """Validate a per-row-group fp32 vector table ([D] when rows == 0, [G, D] otherwise); returns its group stride."""
    if t is None:
        return 0
    if t.dtype != torch.float32 or t.stride(-1) != 1:
        raise FvbError(f"{name} must be fp32 with unit inner stride")
    if rows == 0:
        if t.numel() != D:
            raise FvbError(f"{name} must have {D} elements")
        return 0
    if t.dim() != 2 or t.shape[1] != D or t.shape[0] * rows < M:
        raise FvbError(f"{name} must be [groups, {D}] covering {M} rows in groups of {rows}")
    return t.stride(0)


def linear_sp(x: torch.Tensor, M: int, K: int, ldx: int, w: torch.Tensor, bias, out: torch.Tensor, ldo: int,
              epilogue: int = EPI_BIAS, x_seg_len: int = 0, x_seg_stride: int = 0, out_col_offsets=None, resid=None,
              gate=None, gate_rows: int = 0) -> None:
    """fvb_linear_bf16_sp on raw buffers (x / out are base tensors; the logical shapes are given explicitly);
    fvb_linear_w8_sp, with the same arguments, when w is an Int8Weight; when that weight is marked int8_activations, x
    (segmented or not) is quantised to contiguous int8 rows first and fvb_linear_w8a8_sp runs on them."""
    N = w.shape[0]
    ldr = resid.stride(0) if resid is not None else 0
    gate_stride = _check_grouped(gate, N, gate_rows, M, "gate")
    if isinstance(w, Int8Weight):
        if not x.is_cuda or w.q.device != x.device:
            raise FvbError("x and the Int8Weight must be on the same CUDA device")
        if w.int8_activations:
            xq, xs = _quantize_int8_rows_sp(x, M, K, ldx, x_seg_len, x_seg_stride)
            check(lib().fvb_linear_w8a8_sp(ptr(xq), c_int64(xq.stride(0)), _f32p(xs), ptr(w.q), c_int64(w.q.stride(0)),
                                           _f32p(w.scale), ptr(bias), ptr(out), c_int64(ldo), ptr(out_col_offsets), ptr(resid),
                                           c_int64(ldr), _f32p(gate), c_int(gate_rows), c_int64(gate_stride), c_int(M), c_int(N),
                                           c_int(K), c_int(epilogue), stream_ptr()))
            return
        check(lib().fvb_linear_w8_sp(ptr(x), c_int64(ldx), c_int(x_seg_len), c_int64(x_seg_stride), ptr(w.q),
                                     c_int64(w.q.stride(0)), _f32p(w.scale), ptr(bias), ptr(out), c_int64(ldo),
                                     ptr(out_col_offsets), ptr(resid), c_int64(ldr), _f32p(gate), c_int(gate_rows),
                                     c_int64(gate_stride), c_int(M), c_int(N), c_int(K), c_int(epilogue), stream_ptr()))
        return
    check(lib().fvb_linear_bf16_sp(ptr(x), c_int64(ldx), c_int(x_seg_len), c_int64(x_seg_stride), ptr(w), c_int64(w.stride(0)),
                                   ptr(bias), ptr(out), c_int64(ldo), ptr(out_col_offsets), ptr(resid), c_int64(ldr),
                                   cast(ptr(gate), POINTER(c_float)), c_int(gate_rows), c_int64(gate_stride), c_int(M), c_int(N),
                                   c_int(K), c_int(epilogue), stream_ptr()))


def _f32p(t):
    return cast(ptr(t), POINTER(c_float))


def _i32p(t):
    from ctypes import c_int32
    return cast(ptr(t), POINTER(c_int32))


def layernorm_modulate(x: torch.Tensor, scale: torch.Tensor | None = None, shift: torch.Tensor | None = None,
                       weight: torch.Tensor | None = None, bias: torch.Tensor | None = None, round_ln: bool = False,
                       eps: float = 1e-6, want_hidden: bool = False, mod_rows: int = 0, mod_bf16: bool = False):
    """See fvb_layernorm_modulate. x: [M, D] bf16 or fp32. Returns out (bf16) [, hidden (bf16)].
    scale/shift: fp32 [D], or [G, D] with mod_rows > 0 (row r uses entry r // mod_rows)."""
    assert x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    M, D = x.shape
    out = torch.empty((M, D), dtype=torch.bfloat16, device=x.device)
    hidden = torch.empty((M, D), dtype=torch.bfloat16, device=x.device) if want_hidden else None
    for t in (weight, bias):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and t.numel() == D)
    mod_stride = _check_grouped(scale, D, mod_rows, M, "scale")
    if _check_grouped(shift, D, mod_rows, M, "shift") != mod_stride:
        raise FvbError("scale and shift must share their group stride")
    if mod_bf16 and not round_ln:
        raise FvbError("bf16 modulation arithmetic implies a bf16 LayerNorm output (round_ln)")
    check(lib().fvb_layernorm_modulate(ptr(x), c_int(int(x.dtype == torch.float32)), c_int64(x.stride(0)), _f32p(weight),
                                       _f32p(bias), _f32p(scale), _f32p(shift), c_int(mod_rows), c_int64(mod_stride),
                                       c_int(int(round_ln) | (2 if mod_bf16 else 0)), ptr(out),
                                       c_int64(out.stride(0)), ptr(hidden), c_int64(hidden.stride(0) if want_hidden else 0),
                                       c_int(M), c_int(D), c_float(eps), stream_ptr()))
    return (out, hidden) if want_hidden else out


def rmsnorm_rope_(x0: torch.Tensor, w0: torch.Tensor, x1: torch.Tensor | None = None, w1: torch.Tensor | None = None,
                  cos: torch.Tensor | None = None, sin: torch.Tensor | None = None, rope_row: torch.Tensor | None = None,
                  head_dim: int = 128, eps: float = 1e-6, col_offsets: torch.Tensor | None = None,
                  shape: tuple | None = None) -> None:
    """In-place RMSNorm(+RoPE) of the rows of x0 (and x1). x*: [M, D] bf16 views with unit inner stride."""
    _require_cuda_bf16(x0, "x0")
    if col_offsets is not None:
        # head-scattered rows: x0/x1 are base views whose row stride is stride(0); logical shape given explicitly
        M, D = shape
        assert col_offsets.dtype == torch.int64 and col_offsets.numel() == D // 128
    else:
        M, D = x0.shape
        assert x0.stride(1) == 1
        if x1 is not None:
            assert x1.shape == x0.shape and x1.stride(1) == 1
    assert w0.dtype in (torch.bfloat16, torch.float32) and w0.numel() == D and w0.is_contiguous()
    if x1 is not None:
        assert w1.dtype == w0.dtype and w1.is_contiguous()
    rope_f64 = int(cos is not None and cos.dtype == torch.float64) | (2 if w0.dtype == torch.float32 else 0)  # flag bits
    if cos is not None:
        assert cos.dtype in (torch.float32, torch.float64) and cos.is_contiguous() and cos.shape[-1] == head_dim
        assert sin.dtype == cos.dtype and sin.is_contiguous() and sin.shape == cos.shape
        assert rope_row is not None or cos.shape[0] >= M
    if rope_row is not None:
        assert rope_row.dtype == torch.int32 and rope_row.numel() == M
    check(lib().fvb_rmsnorm_rope(ptr(x0), ptr(w0), c_int64(x0.stride(0)), ptr(x1), ptr(w1),
                                 c_int64(x1.stride(0) if x1 is not None else 0), ptr(cos), ptr(sin), c_int(int(rope_f64)),
                                 _i32p(rope_row),
                                 ptr(col_offsets), c_int(M), c_int(D), c_int(head_dim), c_float(eps), stream_ptr()))


def rmsnorm_rope_scatter(x0: torch.Tensor, w0, x1, w1, y0_ptr: int, y1_ptr: int, ldy: int, out_col_offsets: torch.Tensor,
                         cos=None, sin=None, rope_row=None, head_dim: int = 128, eps: float = 1e-6) -> None:
    """fvb_rmsnorm_rope_scatter: rows of x0 (and x1) [M, D] (contiguous rows, any row stride) are normalised (+RoPE) --
    or copied unchanged when the weight is None -- and written to y*_ptr + row*ldy + out_col_offsets[head]. y pointers
    are raw device addresses (they may belong to a peer GPU's symmetric-memory buffer)."""
    from ctypes import c_void_p
    _require_cuda_bf16(x0, "x0")
    M, D = x0.shape
    assert x0.stride(1) == 1 and (x1 is None or (x1.shape == x0.shape and x1.stride(1) == 1))
    assert out_col_offsets.dtype == torch.int64 and out_col_offsets.numel() == D // 128 and out_col_offsets.is_cuda
    assert w0 is None or w0.dtype in (torch.bfloat16, torch.float32)
    assert x1 is None or w1 is None or w0 is None or w1.dtype == w0.dtype
    rope_f64 = int(cos is not None and cos.dtype == torch.float64) | (2 if (w0 is not None and w0.dtype == torch.float32) else 0)
    check(lib().fvb_rmsnorm_rope_scatter(ptr(x0), ptr(w0), c_int64(x0.stride(0)), ptr(x1), ptr(w1),
                                         c_int64(x1.stride(0) if x1 is not None else 0), c_void_p(y0_ptr),
                                         c_void_p(y1_ptr if x1 is not None else 0), c_int64(ldy), ptr(out_col_offsets),
                                         ptr(cos), ptr(sin), c_int(int(rope_f64)), _i32p(rope_row), c_int(M), c_int(D),
                                         c_int(head_dim), c_float(eps), stream_ptr()))


def _bsh_strides(t: torch.Tensor):
    """t: [B, S, H, d] view (any strides, d contiguous) -> ctypes int64[3] of (b, s, h) strides."""
    assert t.dim() == 4 and t.stride(3) == 1
    return (c_int64 * 3)(t.stride(0), t.stride(1), t.stride(2))


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, softmax_scale: float | None = None,
              out: torch.Tensor | None = None, return_lse: bool = False, sched: torch.Tensor | None = None,
              sched_cnt: torch.Tensor | None = None, q_off=None, q_len=None, kv_off=None, kv_len=None,
              nqb: int = 0, nkb: int = 0):
    """q: [B, Sq, H, 128], k/v: [B, Skv, H, 128] bf16 views (BSHD indexing; pass .transpose(1,2) of BHSD data).
    sched: int32 [B or 1, H or 1, npairs, cap] + sched_cnt [.., npairs] selects block-list mode."""
    for n, t in (("q", q), ("k", k), ("v", v)):
        _require_cuda_bf16(t, n)
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    if softmax_scale is None:
        softmax_scale = d ** -0.5
    if out is None:
        out = torch.empty((B, Sq, H, d), dtype=torch.bfloat16, device=q.device)
    lse = torch.empty((B, H, Sq), dtype=torch.float32, device=q.device) if return_lse else None
    if sched is not None:
        assert sched.dtype == torch.int32 and sched.dim() == 4 and sched.is_contiguous()
        assert sched_cnt.dtype == torch.int32 and sched_cnt.is_contiguous()
        sb, sh, npairs, cap = sched.shape
        stride_h = 0 if sh == 1 else npairs
        stride_b = 0 if sb == 1 else sh * npairs
    else:
        npairs = cap = stride_h = stride_b = 0
    check(lib().fvb_attention_fwd(ptr(q), ptr(k), ptr(v), ptr(out), _f32p(lse), _bsh_strides(q), _bsh_strides(k),
                                  _bsh_strides(v), _bsh_strides(out), c_int64(H * Sq), c_int64(Sq), c_int(B), c_int(H),
                                  c_int(Sq), c_int(Skv), c_int(d), c_float(softmax_scale), _i32p(sched), _i32p(sched_cnt),
                                  c_int64(stride_b), c_int64(stride_h), c_int(cap), c_int(npairs), _i32p(q_off),
                                  _i32p(q_len), c_int(nqb), _i32p(kv_off), _i32p(kv_len), c_int(nkb), stream_ptr()))
    return (out, lse) if return_lse else out


_WORKSPACES: dict = {}


def _workspace(nbytes: int, device) -> torch.Tensor:
    """Grow-only per-device scratch handed to kernels that need caller-allocated workspace (stream-ordered reuse: every
    user runs on the current stream). Allocated outside CUDA-graph capture by the warm-up step."""
    key = (device.type, device.index)
    buf = _WORKSPACES.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
        _WORKSPACES[key] = buf
    return buf


def attention_blocklist(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q2k_idx: torch.Tensor, q2k_num: torch.Tensor,
                        softmax_scale: float | None = None, out: torch.Tensor | None = None, return_lse: bool = False,
                        q_off=None, q_len=None, kv_off=None, kv_len=None, nkb: int | None = None):
    """Block-list attention (weight-stationary M=64 path). q: [B, Sq, H, 128], k/v: [B, Skv, H, 128] views;
    q2k_idx int32 [B or 1, H or 1, nqb, cap], q2k_num int32 [B or 1, H or 1, nqb]."""
    for n, t in (("q", q), ("k", k), ("v", v)):
        _require_cuda_bf16(t, n)
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    if softmax_scale is None:
        softmax_scale = d ** -0.5
    if out is None:
        # padded layout (q_off None, q_len given): rows past a tile's length are never stored by the kernel; the
        # reference returns defined values there, so they are zero here (ADVICE r1: no uninitialised rows leave the API)
        alloc = torch.zeros if (q_off is None and q_len is not None) else torch.empty
        out = alloc((B, Sq, H, d), dtype=torch.bfloat16, device=q.device)
    lse = None
    if return_lse:
        # padded layout: rows past a tile's length are not computed; their LSE is that of a row without keys, -inf, so
        # attention_blocklist_bwd gives them no weight
        lse = (torch.full((B, H, Sq), float("-inf"), dtype=torch.float32, device=q.device) if (q_off is None and q_len is not None)
               else torch.empty((B, H, Sq), dtype=torch.float32, device=q.device))
    assert q2k_idx.dtype == torch.int32 and q2k_idx.dim() == 4 and q2k_idx.is_contiguous()
    assert q2k_num.dtype == torch.int32 and q2k_num.is_contiguous()
    ib, ih, nqb, cap = q2k_idx.shape
    stride_h = 0 if ih == 1 else nqb
    stride_b = 0 if ib == 1 else ih * nqb
    ws = _workspace(int(lib().fvb_attention_blocklist_workspace_bytes(c_int(ib * ih), c_int(nqb), c_int(cap))), q.device)
    check(lib().fvb_attention_blocklist_fwd(ptr(q), ptr(k), ptr(v), ptr(out), _f32p(lse), _bsh_strides(q), _bsh_strides(k),
                                            _bsh_strides(v), _bsh_strides(out), c_int64(H * Sq), c_int64(Sq), c_int(B), c_int(H),
                                            c_int(Sq), c_int(Skv), c_int(d), c_float(softmax_scale), _i32p(q2k_idx),
                                            _i32p(q2k_num), c_int64(stride_b), c_int64(stride_h), c_int(cap), _i32p(q_off),
                                            _i32p(q_len), c_int(nqb), _i32p(kv_off), _i32p(kv_len),
                                            c_int(nkb if nkb is not None else cap), ptr(ws), c_int64(ws.numel()),
                                            stream_ptr()))
    return (out, lse) if return_lse else out


class Attn8bitInputs:
    """Operands of the 8-bit attention, from quantize_attention_8bit (layouts and arithmetic in include/fvb200.h,
    fvb_attention_8bit_quantize): q8 / k8 int8 [B, H, S, 128] with q_scale / k_scale fp32 [B, H, S]; vt8 float8_e4m3fn
    [B, H, nkb, 128, 64] (V transposed per 64-key block, key slots permuted) with v_scale fp32 [B, H, 128]; k_mean fp32
    [B, H, 128] (the mean key subtracted before quantising K). kv_off / kv_len / nkb: the key blocks vt8 is laid out by."""

    def __init__(self, q8, q_scale, k8, k_scale, k_mean, vt8, v_scale, kv_off, kv_len, nkb):
        self.q8, self.q_scale, self.k8, self.k_scale, self.k_mean = q8, q_scale, k8, k_scale, k_mean
        self.vt8, self.v_scale = vt8, v_scale
        self.kv_off, self.kv_len, self.nkb = kv_off, kv_len, nkb

    @property
    def shape(self):
        """(B, H, Sq, Skv)"""
        B, H, Sq, _ = self.q8.shape
        return B, H, Sq, self.k8.shape[2]


def _check_i32(t, name: str, n: int) -> None:
    if t is not None and (t.dtype != torch.int32 or not t.is_cuda or not t.is_contiguous() or t.numel() < n):
        raise FvbError(f"{name} must be a contiguous int32 CUDA tensor of at least {n} elements")


def quantize_attention_8bit(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, kv_off=None, kv_len=None,
                            nkb: int | None = None) -> Attn8bitInputs:
    """fvb_attention_8bit_quantize. q: [B, Sq, H, 128], k/v: [B, Skv, H, 128] bf16 views (any (b, s, h) strides that are
    multiples of 8, e.g. the column slices of a fused QKV buffer). kv_off int32 [nkb + 1] / kv_len int32 [nkb] define the key
    blocks (default: 64-key blocks, nkb = ceil(Skv / 64))."""
    for n, t in (("q", q), ("k", k), ("v", v)):
        _require_cuda_bf16(t, n)
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    if d != 128 or k.shape != (B, Skv, H, d) or v.shape != k.shape:
        raise FvbError("q, k, v must be [B, S, H, 128] with matching B, H and key counts")
    if kv_off is None:
        nkb = (Skv + 63) // 64 if nkb is None else nkb
    elif nkb is None:
        nkb = kv_off.numel() - 1
    _check_i32(kv_off, "kv_off", nkb + 1)
    _check_i32(kv_len, "kv_len", nkb)
    dev = q.device
    q8 = torch.empty((B, H, Sq, d), dtype=torch.int8, device=dev)
    k8 = torch.empty((B, H, Skv, d), dtype=torch.int8, device=dev)
    q_scale = torch.empty((B, H, Sq), dtype=torch.float32, device=dev)
    k_scale = torch.empty((B, H, Skv), dtype=torch.float32, device=dev)
    k_mean = torch.empty((B, H, d), dtype=torch.float32, device=dev)
    vt8 = torch.empty((B, H, nkb, d, 64), dtype=torch.float8_e4m3fn, device=dev)
    v_scale = torch.empty((B, H, d), dtype=torch.float32, device=dev)
    ws = _workspace(int(lib().fvb_attention_8bit_workspace_bytes(c_int(B), c_int(H), c_int(Skv))), dev)
    check(lib().fvb_attention_8bit_quantize(ptr(q), ptr(k), ptr(v), _bsh_strides(q), _bsh_strides(k), _bsh_strides(v), c_int(B),
                                            c_int(H), c_int(Sq), c_int(Skv), c_int(d), _i32p(kv_off), _i32p(kv_len), c_int(nkb),
                                            ptr(q8), _f32p(q_scale), ptr(k8), _f32p(k_scale), _f32p(k_mean), ptr(vt8),
                                            _f32p(v_scale), ptr(ws), c_int64(ws.numel()), stream_ptr()))
    return Attn8bitInputs(q8, q_scale, k8, k_scale, k_mean, vt8, v_scale, kv_off, kv_len, nkb)


def attention_8bit(inputs: Attn8bitInputs, softmax_scale: float | None = None, q2k_idx: torch.Tensor | None = None,
                   q2k_num: torch.Tensor | None = None, q_off=None, q_len=None, out: torch.Tensor | None = None) -> torch.Tensor:
    """fvb_attention_8bit_fwd on quantize_attention_8bit's output -> bf16 [B, Sq, H, 128] (or into `out`, a BSHD view).
    Dense keys without q2k_idx / q2k_num; otherwise per-q-block lists q2k_idx int32 [B or 1, H or 1, nqb, cap] (ascending,
    first q2k_num[..] valid) with q blocks q_off / q_len, as in attention_blocklist. The key blocks are the quantiser's."""
    if not isinstance(inputs, Attn8bitInputs):
        raise FvbError("attention_8bit takes the Attn8bitInputs of quantize_attention_8bit")
    B, H, Sq, Skv = inputs.shape
    d = 128
    if softmax_scale is None:
        softmax_scale = d ** -0.5
    if out is None:
        alloc = torch.zeros if (q2k_idx is not None and q_off is None and q_len is not None) else torch.empty
        out = alloc((B, Sq, H, d), dtype=torch.bfloat16, device=inputs.q8.device)
    _require_cuda_bf16(out, "out")
    if out.shape != (B, Sq, H, d):
        raise FvbError(f"out must be [{B}, {Sq}, {H}, {d}]")
    if (q2k_idx is None) != (q2k_num is None):
        raise FvbError("q2k_idx and q2k_num go together")
    nqb = cap = stride_b = stride_h = 0
    if q2k_idx is not None:
        if q2k_idx.dtype != torch.int32 or q2k_idx.dim() != 4 or not q2k_idx.is_contiguous():
            raise FvbError("q2k_idx must be contiguous int32 [B or 1, H or 1, nqb, cap]")
        ib, ih, nqb, cap = q2k_idx.shape
        if q2k_num.dtype != torch.int32 or not q2k_num.is_contiguous() or q2k_num.shape != (ib, ih, nqb):
            raise FvbError("q2k_num must be contiguous int32 [B or 1, H or 1, nqb]")
        stride_h = 0 if ih == 1 else nqb
        stride_b = 0 if ib == 1 else ih * nqb
        _check_i32(q_off, "q_off", nqb + 1)
        _check_i32(q_len, "q_len", nqb)
    check(lib().fvb_attention_8bit_fwd(ptr(inputs.q8), _f32p(inputs.q_scale), ptr(inputs.k8), _f32p(inputs.k_scale),
                                       ptr(inputs.vt8), _f32p(inputs.v_scale), ptr(out), None, _bsh_strides(out), c_int(B),
                                       c_int(H), c_int(Sq), c_int(Skv), c_int(d), c_float(softmax_scale), None, _i32p(q2k_idx),
                                       _i32p(q2k_num), c_int64(stride_b), c_int64(stride_h), c_int(cap), _i32p(q_off),
                                       _i32p(q_len), c_int(nqb), _i32p(inputs.kv_off), _i32p(inputs.kv_len),
                                       c_int(inputs.nkb), stream_ptr()))
    return out


def attention_blocklist_bwd(q, k, v, o, lse, dO, q2k_idx, q2k_num, k2q_idx, k2q_num, kv_len=None, softmax_scale=None):
    """Backward of attention_blocklist in the padded layout. q/k/v/o/dO: [B, S, H, 128] views; lse fp32 [B, H, Sq] contiguous;
    index tensors int32 [B or 1, H or 1, n, cap] / [.., n]. Returns (dq, dk, dv) with q's / k's / v's shapes (BSHD views)."""
    for n, t in (("q", q), ("k", k), ("v", v), ("o", o), ("dO", dO)):
        _require_cuda_bf16(t, n)
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    if softmax_scale is None:
        softmax_scale = d ** -0.5
    assert lse.dtype == torch.float32 and lse.is_contiguous() and lse.shape == (B, H, Sq)
    dq = torch.empty((B, Sq, H, d), dtype=torch.bfloat16, device=q.device)
    dk = torch.empty((B, Skv, H, d), dtype=torch.bfloat16, device=q.device)
    dv = torch.empty((B, Skv, H, d), dtype=torch.bfloat16, device=q.device)
    delta = torch.empty((B * H * Sq,), dtype=torch.float32, device=q.device)
    for t in (q2k_idx, q2k_num, k2q_idx, k2q_num):
        assert t.dtype == torch.int32 and t.is_contiguous()
    ib, ih, nqb, capq = q2k_idx.shape
    kb_, kh_, nkb, capk = k2q_idx.shape
    sb = lambda nb, nh, n: (0 if nb == 1 else nh * n, 0 if nh == 1 else n)
    isb, ish = sb(ib, ih, nqb)
    ksb, ksh = sb(kb_, kh_, nkb)
    check(lib().fvb_attention_blocklist_bwd(ptr(q), ptr(k), ptr(v), ptr(o), ptr(dO), _f32p(lse), ptr(dq), ptr(dk), ptr(dv),
                                            _f32p(delta), _bsh_strides(q), _bsh_strides(k), _bsh_strides(v), _bsh_strides(o),
                                            _bsh_strides(dO), _bsh_strides(dq), _bsh_strides(dk), _bsh_strides(dv), c_int(B),
                                            c_int(H), c_int(Sq), c_int(Skv), c_int(d), c_float(softmax_scale), _i32p(q2k_idx),
                                            _i32p(q2k_num), c_int(capq), _i32p(k2q_idx), _i32p(k2q_num), c_int(capk),
                                            c_int64(isb), c_int64(ish), c_int64(ksb), c_int64(ksh), _i32p(kv_len), stream_ptr()))
    return dq, dk, dv


def attention_sparse_bwd(q, k, v, o, lse, dO, q2k_idx, q2k_num, k2q_idx, k2q_num, q_off=None, q_len=None, kv_off=None,
                         kv_len=None, softmax_scale=None, out=None):
    """fvb_attention_sparse_bwd: backward of attention_blocklist in either layout, on the wgmma kernels. q/k/v/o/dO:
    [B, S, H, 128] bf16 views (strided ok, as the forward takes them); lse fp32 [B, H, Sq] (unit stride along Sq) as
    attention_blocklist(..., return_lse=True) returns it; q2k_idx int32 [B or 1, H or 1, nqb, capq] / q2k_num [.., nqb] and the
    inverse k2q lists [.., nkb, capk] / [.., nkb]. q_off / q_len / kv_off / kv_len: the forward's tile tables (None: 64-row
    tiles). Returns (dq, dk, dv) with q's / k's / v's shapes (BSHD); rows outside every tile (pad rows) are zero.
    out = (dq, dk, dv) views to write into instead ((b, s, h) strides multiples of 8): only tile rows are written there."""
    for n, t in (("q", q), ("k", k), ("v", v), ("o", o), ("dO", dO)):
        _require_cuda_bf16(t, n)
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    if softmax_scale is None:
        softmax_scale = d ** -0.5
    if (k.shape != (B, Skv, H, d) or v.shape != k.shape or o.shape != q.shape or dO.shape != q.shape
            or lse.dtype != torch.float32 or lse.shape != (B, H, Sq) or lse.stride(2) != 1):
        raise FvbError("attention_sparse_bwd: q/o/dO [B, Sq, H, 128], k/v [B, Skv, H, 128], lse fp32 [B, H, Sq]")
    for t in (q2k_idx, q2k_num, k2q_idx, k2q_num):
        if t.dtype != torch.int32 or not t.is_contiguous():
            raise FvbError("attention_sparse_bwd: index lists must be contiguous int32")
    ib, ih, nqb, capq = q2k_idx.shape
    kb_, kh_, nkb, capk = k2q_idx.shape
    for name, t, n in (("q_off", q_off, nqb + 1), ("q_len", q_len, nqb), ("kv_off", kv_off, nkb + 1), ("kv_len", kv_len, nkb)):
        if t is not None:
            _check_i32(t, name, n)
    # without tile offsets, rows past a tile's length (pad rows) belong to no tile and are not written: zero them
    if out is None:
        alloc = lambda off, lens: torch.zeros if (off is None and lens is not None) else torch.empty
        dq = alloc(q_off, q_len)((B, Sq, H, d), dtype=torch.bfloat16, device=q.device)
        dk = alloc(kv_off, kv_len)((B, Skv, H, d), dtype=torch.bfloat16, device=q.device)
        dv = alloc(kv_off, kv_len)((B, Skv, H, d), dtype=torch.bfloat16, device=q.device)
    else:
        dq, dk, dv = out
        for n, t, want in (("dq", dq, q.shape), ("dk", dk, k.shape), ("dv", dv, k.shape)):
            _require_cuda_bf16(t, n)
            if t.shape != want:
                raise FvbError(f"attention_sparse_bwd: {n} must have shape {tuple(want)}")
    delta = torch.empty((B * H * Sq,), dtype=torch.float32, device=q.device)
    sb = lambda nb, nh, n: (0 if nb == 1 else nh * n, 0 if nh == 1 else n)
    isb, ish = sb(ib, ih, nqb)
    ksb, ksh = sb(kb_, kh_, nkb)
    check(lib().fvb_attention_sparse_bwd(ptr(q), ptr(k), ptr(v), ptr(o), ptr(dO), _f32p(lse), c_int64(lse.stride(0)),
                                         c_int64(lse.stride(1)), ptr(dq), ptr(dk), ptr(dv), _f32p(delta), _bsh_strides(q),
                                         _bsh_strides(k), _bsh_strides(v), _bsh_strides(o), _bsh_strides(dO), _bsh_strides(dq),
                                         _bsh_strides(dk), _bsh_strides(dv), c_int(B), c_int(H), c_int(Sq), c_int(Skv), c_int(d),
                                         c_float(softmax_scale), _i32p(q2k_idx), _i32p(q2k_num), c_int(capq), _i32p(k2q_idx),
                                         _i32p(k2q_num), c_int(capk), c_int64(isb), c_int64(ish), c_int64(ksb), c_int64(ksh),
                                         _i32p(q_off), _i32p(q_len), c_int(nqb), _i32p(kv_off), _i32p(kv_len), c_int(nkb),
                                         stream_ptr()))
    return dq, dk, dv


def attention_bwd(q, k, v, o, lse, dO, softmax_scale=None):
    """fvb_attention_bwd: backward of the dense attention(). q/o/dO: [B, Sq, H, 128], k/v: [B, Skv, H, 128] bf16 views ((b, s, h)
    strides multiples of 8, as the forward takes them); lse fp32 [B, H, Sq] (unit stride along Sq), as attention(...,
    return_lse=True) returns it. Returns contiguous (dq, dk, dv) with q's / k's / v's shapes (BSHD)."""
    for n, t in (("q", q), ("k", k), ("v", v), ("o", o), ("dO", dO)):
        _require_cuda_bf16(t, n)
    B, Sq, H, d = q.shape
    Skv = k.shape[1]
    if softmax_scale is None:
        softmax_scale = d ** -0.5
    if (k.shape != (B, Skv, H, d) or v.shape != k.shape or o.shape != q.shape or dO.shape != q.shape
            or lse.dtype != torch.float32 or lse.shape != (B, H, Sq) or lse.stride(2) != 1):
        raise FvbError("attention_bwd: q/o/dO [B, Sq, H, 128], k/v [B, Skv, H, 128], lse fp32 [B, H, Sq]")
    dq = torch.empty((B, Sq, H, d), dtype=torch.bfloat16, device=q.device)
    dk = torch.empty((B, Skv, H, d), dtype=torch.bfloat16, device=q.device)
    dv = torch.empty((B, Skv, H, d), dtype=torch.bfloat16, device=q.device)
    delta = torch.empty((B * H * Sq,), dtype=torch.float32, device=q.device)
    check(lib().fvb_attention_bwd(ptr(q), ptr(k), ptr(v), ptr(o), ptr(dO), _f32p(lse), c_int64(lse.stride(0)),
                                  c_int64(lse.stride(1)), ptr(dq), ptr(dk), ptr(dv), _f32p(delta), _bsh_strides(q),
                                  _bsh_strides(k), _bsh_strides(v), _bsh_strides(o), _bsh_strides(dO), _bsh_strides(dq),
                                  _bsh_strides(dk), _bsh_strides(dv), c_int(B), c_int(H), c_int(Sq), c_int(Skv), c_int(d),
                                  c_float(softmax_scale), stream_ptr()))
    return dq, dk, dv


def rmsnorm_bwd(x: torch.Tensor, w: torch.Tensor | None, dy: torch.Tensor, eps: float = 1e-6, want_dw: bool = True):
    """fvb_rmsnorm_bwd: backward of rmsnorm_rope_(x, w) without RoPE. x, dy: [M, D] bf16 with unit inner stride; w: bf16 [D]
    or None (ones). Returns (dx bf16 [M, D], dw bf16 [D], or None without w or with want_dw=False)."""
    _require_cuda_bf16(x, "x")
    _require_cuda_bf16(dy, "dy")
    M, D = x.shape
    if x.stride(1) != 1 or dy.shape != (M, D) or dy.stride(1) != 1:
        raise FvbError("rmsnorm_bwd: x and dy must be [M, D] with unit inner stride")
    if w is not None and (w.dtype != torch.bfloat16 or not w.is_contiguous() or w.numel() != D):
        raise FvbError("rmsnorm_bwd: w must be a contiguous bf16 [D] tensor")
    dx = torch.empty((M, D), dtype=torch.bfloat16, device=x.device)
    want_dw = want_dw and w is not None
    dw = torch.empty(D, dtype=torch.bfloat16, device=x.device) if want_dw else None
    ws = _workspace(int(lib().fvb_rmsnorm_bwd_workspace_bytes(c_int(M), c_int(D))), x.device) if want_dw else None
    check(lib().fvb_rmsnorm_bwd(ptr(x), c_int64(x.stride(0)), ptr(w), ptr(dy), c_int64(dy.stride(0)), ptr(dx),
                                c_int64(dx.stride(0)), ptr(dw), _f32p(ws), c_int64(ws.numel() if ws is not None else 0),
                                c_int(M), c_int(D), c_float(eps), stream_ptr()))
    return dx, dw


# ---------------------------------------------------------------- index / mask construction
def vsa_tile_index(seq_shape, tile_size, device="cuda"):
    """Returns dict of device tensors: tile_partition, reverse_partition, non_pad, untile_combined (int64 [S]),
    variable_block_sizes (int32 [n_tiles]), block_offsets (int32 [n_tiles+1])."""
    import math
    T, H, W = seq_shape
    ts, hs, ws = tile_size
    S = T * H * W
    nt = math.ceil(T / ts) * math.ceil(H / hs) * math.ceil(W / ws)
    out = {k: torch.empty(S, dtype=torch.int64, device=device)
           for k in ("tile_partition", "reverse_partition", "non_pad", "untile_combined")}
    out["variable_block_sizes"] = torch.empty(nt, dtype=torch.int32, device=device)
    out["block_offsets"] = torch.empty(nt + 1, dtype=torch.int32, device=device)
    check(lib().fvb_vsa_tile_index(c_int(T), c_int(H), c_int(W), c_int(ts), c_int(hs), c_int(ws), ptr(out["tile_partition"]),
                                   ptr(out["reverse_partition"]), ptr(out["non_pad"]), ptr(out["untile_combined"]),
                                   ptr(out["variable_block_sizes"]), ptr(out["block_offsets"]), stream_ptr()))
    return out


def topk_mask(scores: torch.Tensor, topk: int) -> torch.Tensor:
    """scores [..., n] bf16/fp32 (last dim contiguous) -> bool mask with exactly min(topk, n) True per row."""
    assert scores.is_cuda and scores.dtype in (torch.bfloat16, torch.float32)
    n = scores.shape[-1]
    s2 = scores.reshape(-1, n)
    if s2.stride(1) != 1:
        s2 = s2.contiguous()
    mask = torch.empty(s2.shape, dtype=torch.bool, device=scores.device)
    check(lib().fvb_topk_mask(ptr(s2), c_int(0 if scores.dtype == torch.bfloat16 else 1), c_int64(s2.stride(0)), ptr(mask),
                              c_int64(n), c_int64(s2.shape[0]), c_int(n), c_int(topk), stream_ptr()))
    return mask.reshape(scores.shape)


def topk_index(scores: torch.Tensor, topk: int, want_mask: bool = False):
    """scores [..., nq, n] bf16 -> (q2k_idx int32 [..., nq, n] ascending, -1 padded; q2k_num int32 [..., nq]; bool mask or
    None): topk_mask + map_to_index in one pass (one warp per row when n % 4 == 0 and n <= 2048)."""
    assert scores.is_cuda and scores.dtype == torch.bfloat16
    n = scores.shape[-1]
    s2 = scores.reshape(-1, n)
    if s2.stride(1) != 1:
        s2 = s2.contiguous()
    rows = s2.shape[0]
    fast = (n % 4 == 0 and n <= 2048 and s2.stride(0) % 4 == 0 and s2.data_ptr() % 8 == 0
            and os.environ.get("FVB_TOPK_WARP", "1") != "0")  # else the library needs the mask as its intermediate
    mask = torch.empty(s2.shape, dtype=torch.bool, device=s2.device) if (want_mask or not fast) else None
    idx = torch.empty(s2.shape, dtype=torch.int32, device=s2.device)
    num = torch.empty(rows, dtype=torch.int32, device=s2.device)
    check(lib().fvb_topk_index(ptr(s2), c_int64(s2.stride(0)), ptr(mask), c_int64(n), ptr(idx), ptr(num), c_int64(rows), c_int(n),
                               c_int(topk), stream_ptr()))
    return (idx.reshape(scores.shape), num.reshape(scores.shape[:-1]),
            mask.reshape(scores.shape) if (mask is not None and want_mask) else None)


def map_to_index(block_map: torch.Tensor):
    """bool [..., nq, nkv] -> (q2k_idx int32 same shape, -1 padded ascending; q2k_num int32 [..., nq])."""
    assert block_map.is_cuda and block_map.dtype == torch.bool
    n = block_map.shape[-1]
    m2 = block_map.reshape(-1, n).contiguous()
    idx = torch.empty(m2.shape, dtype=torch.int32, device=m2.device)
    num = torch.empty(m2.shape[0], dtype=torch.int32, device=m2.device)
    check(lib().fvb_map_to_index(ptr(m2), c_int64(n), ptr(idx), ptr(num), c_int64(m2.shape[0]), c_int(n), stream_ptr()))
    return idx.reshape(block_map.shape), num.reshape(block_map.shape[:-1])


def pair_schedule(block_map: torch.Tensor, cap: int | None = None):
    """bool [B, H, nq, nkv] (or [H, nq, nkv]) -> (sched int32 [B, H, npairs, cap], cnt int32 [B, H, npairs])."""
    assert block_map.is_cuda and block_map.dtype == torch.bool
    if block_map.dim() == 3:
        block_map = block_map.unsqueeze(0)
    B, H, nq, nkv = block_map.shape
    m = block_map.contiguous()
    npairs = (nq + 1) // 2
    cap = cap or nkv
    sched = torch.empty((B, H, npairs, cap), dtype=torch.int32, device=m.device)
    cnt = torch.empty((B, H, npairs), dtype=torch.int32, device=m.device)
    check(lib().fvb_pair_schedule(ptr(m), c_int64(nq * nkv), c_int64(nkv), c_int(B * H), c_int(nq), c_int(nkv), ptr(sched),
                                  ptr(cnt), c_int(cap), stream_ptr()))
    return sched, cnt


def sta_map(canvas_tiles, windows, device="cuda") -> torch.Tensor:
    """windows: list of (t,h,w) per head -> bool [heads, n_tiles, n_tiles]."""
    ct, ch, cw = canvas_tiles
    n = ct * ch * cw
    win = torch.tensor(windows, dtype=torch.int32, device=device).contiguous()
    heads = win.shape[0]
    m = torch.empty((heads, n, n), dtype=torch.bool, device=device)
    check(lib().fvb_sta_map(c_int(ct), c_int(ch), c_int(cw), ptr(win), c_int(heads), ptr(m), stream_ptr()))
    return m


# ---------------------------------------------------------------- VSA compression branch
def gemm_batched(a: torch.Tensor, b: torch.Tensor, div: float = 0.0) -> torch.Tensor:
    """a: [batch, M, K], b: [batch, N, K] (bf16, inner stride 1) -> bf16 [batch, M, N] = a @ b^T (/ div)."""
    _require_cuda_bf16(a, "a")
    _require_cuda_bf16(b, "b")
    batch, M, K = a.shape
    N = b.shape[1]
    assert b.shape[0] == batch and b.shape[2] == K and a.stride(2) == 1 and b.stride(2) == 1
    ldo = (N + 7) // 8 * 8
    out = torch.empty((batch, M, ldo), dtype=torch.bfloat16, device=a.device)
    check(lib().fvb_gemm_batched_bf16(ptr(a), c_int64(a.stride(1)), c_int64(a.stride(0)), ptr(b), c_int64(b.stride(1)),
                                      c_int64(b.stride(0)), ptr(out), c_int64(ldo), c_int64(M * ldo), c_int(M), c_int(N),
                                      c_int(K), c_int(batch), c_float(div), stream_ptr()))
    return out[:, :, :N]


def block_mean(x: torch.Tensor, nblk: int, block_off=None, block_len=None, block_rows: int = 64,
               want_transposed: bool = False):
    """x: [B, S, H, 128] view -> [B, H, nblk, 128] bf16 (and [B, H, 128, ldt] if want_transposed)."""
    _require_cuda_bf16(x, "x")
    B, S, H, d = x.shape
    assert d == 128
    out = torch.empty((B, H, nblk, 128), dtype=torch.bfloat16, device=x.device)
    ldt = (nblk + 7) // 8 * 8
    out_t = torch.zeros((B, H, 128, ldt), dtype=torch.bfloat16, device=x.device) if want_transposed else None
    check(lib().fvb_block_mean(ptr(x), _bsh_strides(x), _i32p(block_off), _i32p(block_len), c_int(block_rows), c_int(B),
                               c_int(H), c_int(S), c_int(nblk), ptr(out), ptr(out_t), c_int64(ldt), stream_ptr()))
    return (out, out_t[..., :nblk]) if want_transposed else out


def softmax_rows(x: torch.Tensor, pad_to: int = 8) -> torch.Tensor:
    """Row softmax; the result's row stride is rounded up to `pad_to` elements (zero padded) so it can feed a GEMM."""
    _require_cuda_bf16(x, "x")
    n = x.shape[-1]
    assert x.stride(-1) == 1
    x2 = x.reshape(-1, n) if x.is_contiguous() else x
    if x2.dim() != 2:
        # strided batch of rows (e.g. a column-sliced [batch, M, ld] buffer): collapse leading dims by hand
        lead = x.shape[:-1]
        assert all(x.stride(i) == x.stride(i + 1) * x.shape[i + 1] for i in range(len(lead) - 1))
        x2 = x.as_strided((int(torch.tensor(lead).prod()), n), (x.stride(-2), 1))
    ld = (n + pad_to - 1) // pad_to * pad_to
    out = (torch.zeros if ld != n else torch.empty)((x2.shape[0], ld), dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_softmax_rows(ptr(x2), c_int64(x2.stride(0)), ptr(out), c_int64(ld), c_int64(x2.shape[0]), c_int(n),
                                 stream_ptr()))
    return out.reshape(*x.shape[:-1], ld)[..., :n]


def vsa_combine(out_s: torch.Tensor, out_c: torch.Tensor, gate: torch.Tensor | None, row_block=None,
                block_rows: int = 64, out: torch.Tensor | None = None, out_segments=None) -> torch.Tensor | None:
    """out_s/gate: [B, S, H, 128] views; out_c: [B, H, nblk, 128] contiguous. With out_segments = (int64 device table of
    base addresses, rows per segment, (b, s, h) element strides) row `tok` is stored at
    table[tok // seg_rows] + (tok % seg_rows) * stride_s + h * stride_h instead of into `out` (returns None)."""
    B, S, H, d = out_s.shape
    nblk = out_c.shape[2]
    assert out_c.is_contiguous()
    seg_tab, seg_rows, o_str = None, 0, None
    if out_segments is not None:
        seg_tab, seg_rows, st3 = out_segments
        assert seg_tab.dtype == torch.int64 and seg_tab.is_cuda and B == 1
        o_str = (c_int64 * 3)(*st3)
        out = None
    elif out is None:
        out = torch.empty((B, S, H, d), dtype=torch.bfloat16, device=out_s.device)
    check(lib().fvb_vsa_combine(ptr(out_s), _bsh_strides(out_s), ptr(gate), _bsh_strides(gate) if gate is not None else None,
                                ptr(out_c), _i32p(row_block), c_int(block_rows), ptr(out),
                                o_str if o_str is not None else _bsh_strides(out), c_int(B),
                                c_int(S), c_int(H), c_int(nblk), ptr(seg_tab), c_int(seg_rows), stream_ptr()))
    return out


# ---------------------------------------------------------------- VSA backward (padded layout: 64-row tiles; or compact)
def vsa_combine_bwd(dO: torch.Tensor, out_c: torch.Tensor, gate: torch.Tensor | None, block_len: torch.Tensor,
                    d_gate: torch.Tensor | None = None, block_off: torch.Tensor | None = None):
    """Backward of vsa_combine (fvb_vsa_combine_bwd). dO/gate/d_gate: [B, S, H, 128] views, S = 64 * nblk; out_c
    [B, H, nblk, 128] contiguous; block_len int32 [nblk]. d_gate (output, written when given) = dO * out_c on the valid
    rows and 0 on the pad rows (pad rows are not tokens: dO there counts as zero).
    Returns (d_out_c bf16 [B, H, nblk, 128], the same transposed [B, H, 128, nblk] as a view of a [.., ldt] buffer):
    d_out_c = sum over each tile's valid rows of dO * gate (of dO without a gate), fp32 in a fixed order.
    block_off (int32 [nblk + 1]): the compact layout instead (fvb_vsa_combine_bwd_compact): tile i is rows
    [block_off[i], block_off[i + 1]), every row a token; block_len is then not read."""
    for n, t in (("dO", dO), ("out_c", out_c), ("gate", gate), ("d_gate", d_gate)):
        if t is not None:
            _require_cuda_bf16(t, n)
    B, S, H, d = dO.shape
    nblk = out_c.shape[2]
    if d != 128 or (block_off is None and S != 64 * nblk) or out_c.shape != (B, H, nblk, d) or not out_c.is_contiguous():
        raise FvbError("dO must be [B, 64 * nblk, H, 128] and out_c contiguous [B, H, nblk, 128]")
    if d_gate is not None and gate is None:
        raise FvbError("d_gate needs the gate")
    if block_off is None:
        _check_i32(block_len, "block_len", nblk)
    else:
        _check_i32(block_off, "block_off", nblk + 1)
    d_out_c = torch.empty((B, H, nblk, d), dtype=torch.bfloat16, device=dO.device)
    ldt = (nblk + 7) // 8 * 8
    d_out_c_t = torch.empty((B, H, d, ldt), dtype=torch.bfloat16, device=dO.device)
    fn = lib().fvb_vsa_combine_bwd if block_off is None else lib().fvb_vsa_combine_bwd_compact
    check(fn(ptr(dO), _bsh_strides(dO), ptr(gate), _bsh_strides(gate) if gate is not None else None, ptr(out_c),
             _i32p(block_len if block_off is None else block_off), c_int(B), c_int(S), c_int(H), c_int(nblk), ptr(d_gate),
             _bsh_strides(d_gate) if d_gate is not None else None, ptr(d_out_c), ptr(d_out_c_t), c_int64(ldt), stream_ptr()))
    return d_out_c, d_out_c_t[..., :nblk]


def softmax_rows_bwd(p: torch.Tensor, dp: torch.Tensor, scale: float = 1.0, want_transposed: bool = False):
    """Backward of softmax_rows over square blocks (fvb_softmax_rows_bwd). p (the softmax output) and dp: [batch, n, n] bf16
    views of [batch, n, ld] buffers with the same ld (a multiple of 8), like softmax_rows' and gemm_batched's outputs.
    Returns ds = bf16(p * (dp - rowsum(dp * p)) * scale) [batch, n, n] (a view of a [.., ld] buffer), and with
    want_transposed also ds^T and p^T in that layout: the K-major operands of the products that contract over rows."""
    _require_cuda_bf16(p, "p")
    _require_cuda_bf16(dp, "dp")
    batch, n, n2 = p.shape
    ld = p.stride(1)
    ok = (n == n2 and dp.shape == p.shape and p.stride(2) == 1 and dp.stride(2) == 1 and dp.stride(1) == ld and ld % 8 == 0
          and p.stride(0) == n * ld and dp.stride(0) == n * ld)
    if not ok:
        raise FvbError("p and dp must be [batch, n, n] views of [batch, n, ld] buffers with one ld (a multiple of 8)")
    alloc = lambda: torch.empty((batch, n, ld), dtype=torch.bfloat16, device=p.device)
    ds = alloc()
    ds_t, p_t = (alloc(), alloc()) if want_transposed else (None, None)
    check(lib().fvb_softmax_rows_bwd(ptr(p), ptr(dp), c_int64(ld), c_int(batch), c_int(n), c_float(scale), ptr(ds), ptr(ds_t),
                                     ptr(p_t), stream_ptr()))
    if want_transposed:
        return ds[..., :n], ds_t[..., :n], p_t[..., :n]
    return ds[..., :n]


def block_mean_bwd(dx_s: torch.Tensor, d_mean: torch.Tensor, block_len: torch.Tensor, out: torch.Tensor | None = None,
                   block_off: torch.Tensor | None = None, row_block: torch.Tensor | None = None):
    """Backward of block_mean in the padded layout added to dx_s (fvb_block_mean_bwd): dx = dx_s + d_mean / len on the valid
    rows of each 64-row tile, 0 on its pad rows. dx_s / out: [B, S, H, 128] views, S = 64 * nblk (out may be dx_s: in place);
    d_mean [B, H, nblk, 128] contiguous; block_len int32 [nblk].
    block_off (int32 [nblk + 1]) with row_block (int32 [S]): the compact layout instead (fvb_block_mean_bwd_compact): every
    row is a token of tile row_block[t], len = block_off[tile + 1] - block_off[tile]; block_len is then not read."""
    _require_cuda_bf16(dx_s, "dx_s")
    _require_cuda_bf16(d_mean, "d_mean")
    B, S, H, d = dx_s.shape
    nblk = d_mean.shape[2]
    if d != 128 or (block_off is None and S != 64 * nblk) or d_mean.shape != (B, H, nblk, d) or not d_mean.is_contiguous():
        raise FvbError("dx_s must be [B, 64 * nblk, H, 128] and d_mean contiguous [B, H, nblk, 128]")
    if (block_off is None) != (row_block is None):
        raise FvbError("the compact layout needs both block_off and row_block")
    if out is None:
        out = torch.empty((B, S, H, d), dtype=torch.bfloat16, device=dx_s.device)
    _require_cuda_bf16(out, "out")
    if block_off is None:
        _check_i32(block_len, "block_len", nblk)
        check(lib().fvb_block_mean_bwd(ptr(dx_s), _bsh_strides(dx_s), ptr(d_mean), _i32p(block_len), c_int(B), c_int(H),
                                       c_int(S), c_int(nblk), ptr(out), _bsh_strides(out), stream_ptr()))
    else:
        _check_i32(block_off, "block_off", nblk + 1)
        _check_i32(row_block, "row_block", S)
        check(lib().fvb_block_mean_bwd_compact(ptr(dx_s), _bsh_strides(dx_s), ptr(d_mean), _i32p(block_off), _i32p(row_block),
                                               c_int(B), c_int(H), c_int(S), c_int(nblk), ptr(out), _bsh_strides(out),
                                               stream_ptr()))
    return out


def scatter_rows_to_segments(x: torch.Tensor, seg_table: torch.Tensor, seg_rows: int, dst_ld: int | None = None) -> None:
    """x: [S, width] bf16 (row stride any multiple of 8): row r is copied to seg_table[r // seg_rows] + (r % seg_rows) *
    dst_ld elements. One launch for the whole return path of dense attention under sequence parallelism."""
    _require_cuda_bf16(x, "x")
    assert x.dim() == 2 and x.stride(1) == 1 and seg_table.dtype == torch.int64
    S, width = x.shape
    check(lib().fvb_scatter_rows_to_segments(ptr(x), c_int64(x.stride(0)), c_int64(S), c_int(width), ptr(seg_table),
                                             c_int(seg_rows), c_int64(dst_ld if dst_ld is not None else width), stream_ptr()))


def gather_rows(x: torch.Tensor, idx: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """x: [B, S, W] (bf16, W contiguous, W % 8 == 0); out[b, i] = x[b, idx[i]] (idx < 0 -> zeros)."""
    _require_cuda_bf16(x, "x")
    assert x.dim() == 3 and x.stride(2) == 1 and idx.dtype in (torch.int64, torch.int32) and idx.is_contiguous()
    B, S, W = x.shape
    n = idx.numel()
    if out is None:
        out = torch.empty((B, n, W), dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_gather_rows(ptr(x), c_int64(x.stride(0)), c_int64(x.stride(1)), ptr(idx), c_int(int(idx.dtype == torch.int64)),
                                ptr(out), c_int64(out.stride(0)), c_int64(out.stride(1)), c_int64(n), c_int(W), c_int(B),
                                stream_ptr()))
    return out


# ---------------------------------------------------------------- Wan VAE decode (channels-last frames)
def pack_conv_weight(w: torch.Tensor):
    """[Cout, Cin, kt, kh, kw] or [Cout, Cin, kh, kw] -> (bf16 [Cout, ntaps * Cin_pad], Cin_pad, (kt, kh, kw))."""
    if w.dim() == 4:
        w = w.unsqueeze(2)
    Cout, Cin, kt, kh, kw = w.shape
    Cin_pad = Cin if Cin % 64 == 0 else (Cin + 31) // 32 * 32  # 64-channel k-blocks when possible, else 32
    packed = torch.zeros((Cout, kt * kh * kw, Cin_pad), dtype=torch.bfloat16, device=w.device)
    packed[:, :, :Cin] = w.permute(0, 2, 3, 4, 1).reshape(Cout, kt * kh * kw, Cin).to(torch.bfloat16)
    return packed.reshape(Cout, -1).contiguous(), Cin_pad, (kt, kh, kw)


def conv3d_cl(x: torch.Tensor, w_packed: torch.Tensor, cin_pad: int, k: tuple, bias=None, resid=None, out=None,
              T_out: int | None = None, t_off: int = 0, interleave_c: int = 0) -> torch.Tensor:
    """x: [T_in, H, W, Cin] bf16 contiguous. Returns [T_out(*2 if interleave), H, W, Cout(/2)]."""
    _require_cuda_bf16(x, "x")
    assert x.is_contiguous() and x.dim() == 4
    T_in, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    kt, kh, kw = k
    if T_out is None:
        T_out = T_in - t_off
    if out is None:
        shape = (2 * T_out, H, W, interleave_c) if interleave_c else (T_out, H, W, Cout)
        out = torch.empty(shape, dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_conv3d_cl(ptr(x), c_int(T_in), c_int(H), c_int(W), c_int(Cin), ptr(w_packed), c_int(cin_pad), c_int(Cout),
                              c_int(kt), c_int(kh), c_int(kw), ptr(bias), ptr(resid),
                              c_int64(resid.shape[-1] if resid is not None else 0), ptr(out), c_int64(out.shape[-1]),
                              c_int(T_out), c_int(t_off), c_int(interleave_c), stream_ptr()))
    return out


CONV_NORM_MAX_COUT = 192  # fvb_conv3d_cl_norm: one N tile must hold a pixel's whole channel row


def conv3d_cl_norm(x: torch.Tensor, w_packed: torch.Tensor, cin_pad: int, k: tuple, gamma: torch.Tensor, bias=None, resid=None,
                   want_raw: bool = True, silu: bool = True, T_out: int | None = None, t_off: int = 0, norm_out=None):
    """conv3d_cl with the consumer's RMS-norm (+ SiLU) fused into the epilogue. Returns (raw or None, normed), both
    [T_out, H, W, Cout] bf16; norm_out may be a preallocated [T_out, H, W, Cout] view (e.g. inside the consumer's
    feature-cache buffer)."""
    _require_cuda_bf16(x, "x")
    assert x.is_contiguous() and x.dim() == 4
    T_in, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    kt, kh, kw = k
    if T_out is None:
        T_out = T_in - t_off
    assert gamma.dtype == torch.float32 and gamma.numel() == Cout and gamma.is_cuda
    raw = torch.empty((T_out, H, W, Cout), dtype=torch.bfloat16, device=x.device) if want_raw else None
    if norm_out is None:
        norm_out = torch.empty((T_out, H, W, Cout), dtype=torch.bfloat16, device=x.device)
    assert norm_out.shape == (T_out, H, W, Cout) and norm_out.is_contiguous() and norm_out.dtype == torch.bfloat16
    check(lib().fvb_conv3d_cl_norm(ptr(x), c_int(T_in), c_int(H), c_int(W), c_int(Cin), ptr(w_packed), c_int(cin_pad),
                                   c_int(Cout), c_int(kt), c_int(kh), c_int(kw), ptr(bias), ptr(resid),
                                   c_int64(resid.shape[-1] if resid is not None else 0), ptr(raw), c_int64(Cout), c_int(T_out),
                                   c_int(t_off), _f32p(gamma), ptr(norm_out), c_int64(Cout), c_int(int(silu)), stream_ptr()))
    return raw, norm_out


def rmsnorm_silu_cl(x: torch.Tensor, gamma: torch.Tensor, beta=None, silu: bool = True, out=None) -> torch.Tensor:
    _require_cuda_bf16(x, "x")
    C = x.shape[-1]
    assert x.is_contiguous() and gamma.dtype == torch.float32 and gamma.numel() == C
    if out is None:
        out = torch.empty_like(x)
    assert out.shape == x.shape and out.is_contiguous() and out.dtype == torch.bfloat16
    npix = x.numel() // C
    check(lib().fvb_rmsnorm_silu_cl(ptr(x), c_int64(C), _f32p(gamma), _f32p(beta), ptr(out), c_int64(out.shape[-1]),
                                    c_int64(npix), c_int(C), c_int(int(silu)), stream_ptr()))
    return out


# ---------------------------------------------------------------- FP8 (e4m3) residual-block convolutions
def rms_norm_e4m3_bound(gamma: torch.Tensor) -> float:
    """Static e4m3 scale bound of a WanRMS_norm (+ SiLU) output: |v_c| <= sqrt(C) * max|gamma| (fp32)."""
    C = gamma.numel()
    return float(torch.tensor(C, dtype=torch.float32).sqrt() * gamma.detach().float().abs().max().cpu())


def e4m3_x_scale(bound: float) -> float:
    """The dequantisation scale a convolution applies to an input quantised against `bound`: bound / 448 (fp32), 1 if 0."""
    if bound == 0.0:
        return 1.0
    return float(torch.tensor(bound, dtype=torch.float32) / torch.tensor(FP8_E4M3_MAX, dtype=torch.float32))


def pack_conv_weight_fp8(w: torch.Tensor):
    """pack_conv_weight, then one e4m3 scale per output channel (fvb_quantize_fp8_rows of the packed bf16 rows; the zero
    padding does not change the amax) -> (q float8_e4m3fn [Cout, ntaps * Cin_pad], scale fp32 [Cout], Cin_pad, k)."""
    packed, cin_pad, k = pack_conv_weight(w)
    q, scale = quantize_fp8_rows(packed)
    return q.contiguous(), scale, cin_pad, k


def _require_e4m3(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise FvbError(f"{name} must be a CUDA tensor (no CPU fallback)")
    if t.dtype != torch.float8_e4m3fn:
        raise FvbError(f"{name} must be float8_e4m3fn, got {t.dtype}")


def _norm_out(norm_out, shape, norm_bound, device):
    dt = torch.bfloat16 if norm_bound is None else torch.float8_e4m3fn
    if norm_out is None:
        norm_out = torch.empty(shape, dtype=dt, device=device)
    assert norm_out.shape == shape and norm_out.is_contiguous() and norm_out.dtype == dt
    return norm_out


def conv3d_cl_fp8(x: torch.Tensor, wq: torch.Tensor, w_scale: torch.Tensor, cin_pad: int, k: tuple, x_scale: float,
                  bias=None, resid=None, out=None, T_out: int | None = None, t_off: int = 0) -> torch.Tensor:
    """conv3d_cl on e4m3 operands (fvb_conv3d_cl_fp8): x float8_e4m3fn [T_in, H, W, Cin] read as x * x_scale, wq / w_scale
    from pack_conv_weight_fp8. Output bf16 [T_out, H, W, Cout]."""
    _require_e4m3(x, "x")
    _require_e4m3(wq, "wq")
    assert x.is_contiguous() and x.dim() == 4
    T_in, H, W, Cin = x.shape
    Cout = wq.shape[0]
    kt, kh, kw = k
    if T_out is None:
        T_out = T_in - t_off
    if out is None:
        out = torch.empty((T_out, H, W, Cout), dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_conv3d_cl_fp8(ptr(x), c_int(T_in), c_int(H), c_int(W), c_int(Cin), c_float(x_scale), ptr(wq), _f32p(w_scale),
                                  c_int(cin_pad), c_int(Cout), c_int(kt), c_int(kh), c_int(kw), ptr(bias), ptr(resid),
                                  c_int64(resid.shape[-1] if resid is not None else 0), ptr(out), c_int64(out.shape[-1]),
                                  c_int(T_out), c_int(t_off), stream_ptr()))
    return out


def conv3d_cl_fp8_norm(x: torch.Tensor, wq: torch.Tensor, w_scale: torch.Tensor, cin_pad: int, k: tuple, x_scale: float,
                       gamma: torch.Tensor, bias=None, resid=None, want_raw: bool = True, silu: bool = True,
                       T_out: int | None = None, t_off: int = 0, norm_out=None, norm_bound: float | None = None):
    """conv3d_cl_fp8 with the consumer's RMS-norm (+ SiLU) fused (fvb_conv3d_cl_fp8_norm). Returns (raw bf16 or None,
    normed): normed is bf16, or e4m3 quantised against norm_bound when one is given."""
    _require_e4m3(x, "x")
    _require_e4m3(wq, "wq")
    assert x.is_contiguous() and x.dim() == 4
    T_in, H, W, Cin = x.shape
    Cout = wq.shape[0]
    kt, kh, kw = k
    if T_out is None:
        T_out = T_in - t_off
    assert gamma.dtype == torch.float32 and gamma.numel() == Cout and gamma.is_cuda
    raw = torch.empty((T_out, H, W, Cout), dtype=torch.bfloat16, device=x.device) if want_raw else None
    norm_out = _norm_out(norm_out, (T_out, H, W, Cout), norm_bound, x.device)
    check(lib().fvb_conv3d_cl_fp8_norm(ptr(x), c_int(T_in), c_int(H), c_int(W), c_int(Cin), c_float(x_scale), ptr(wq),
                                       _f32p(w_scale), c_int(cin_pad), c_int(Cout), c_int(kt), c_int(kh), c_int(kw), ptr(bias),
                                       ptr(resid), c_int64(resid.shape[-1] if resid is not None else 0), ptr(raw), c_int64(Cout),
                                       c_int(T_out), c_int(t_off), _f32p(gamma), ptr(norm_out), c_int64(Cout), c_int(int(silu)),
                                       c_int(int(norm_bound is not None)), c_float(norm_bound or 0.0), stream_ptr()))
    return raw, norm_out


def conv3d_cl_norm_e4m3(x: torch.Tensor, w_packed: torch.Tensor, cin_pad: int, k: tuple, gamma: torch.Tensor,
                        norm_bound: float, bias=None, resid=None, want_raw: bool = True, silu: bool = True,
                        T_out: int | None = None, t_off: int = 0, norm_out=None):
    """conv3d_cl_norm (bf16 operands) writing the normalised output as e4m3 against norm_bound (fvb_conv3d_cl_norm_e4m3)."""
    _require_cuda_bf16(x, "x")
    assert x.is_contiguous() and x.dim() == 4
    T_in, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    kt, kh, kw = k
    if T_out is None:
        T_out = T_in - t_off
    assert gamma.dtype == torch.float32 and gamma.numel() == Cout and gamma.is_cuda
    raw = torch.empty((T_out, H, W, Cout), dtype=torch.bfloat16, device=x.device) if want_raw else None
    norm_out = _norm_out(norm_out, (T_out, H, W, Cout), norm_bound, x.device)
    check(lib().fvb_conv3d_cl_norm_e4m3(ptr(x), c_int(T_in), c_int(H), c_int(W), c_int(Cin), ptr(w_packed), c_int(cin_pad),
                                        c_int(Cout), c_int(kt), c_int(kh), c_int(kw), ptr(bias), ptr(resid),
                                        c_int64(resid.shape[-1] if resid is not None else 0), ptr(raw), c_int64(Cout),
                                        c_int(T_out), c_int(t_off), _f32p(gamma), ptr(norm_out), c_int64(Cout), c_int(int(silu)),
                                        c_float(norm_bound), stream_ptr()))
    return raw, norm_out


def rmsnorm_silu_cl_e4m3(x: torch.Tensor, gamma: torch.Tensor, bound: float, silu: bool = True, out=None) -> torch.Tensor:
    """rmsnorm_silu_cl (no beta) written as e4m3: q = satfinite(v * 448 / bound) (fvb_rmsnorm_silu_cl_e4m3)."""
    _require_cuda_bf16(x, "x")
    C = x.shape[-1]
    assert x.is_contiguous() and gamma.dtype == torch.float32 and gamma.numel() == C
    out = _norm_out(out, tuple(x.shape), bound, x.device)
    npix = x.numel() // C
    check(lib().fvb_rmsnorm_silu_cl_e4m3(ptr(x), c_int64(C), _f32p(gamma), ptr(out), c_int64(C), c_int64(npix), c_int(C),
                                         c_int(int(silu)), c_float(bound), stream_ptr()))
    return out


def upsample2x_cl(x: torch.Tensor) -> torch.Tensor:
    T, H, W, C = x.shape
    out = torch.empty((T, 2 * H, 2 * W, C), dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_upsample2x_cl(ptr(x.contiguous()), ptr(out), c_int(T), c_int(H), c_int(W), c_int(C), stream_ptr()))
    return out


def transpose_bf16(x: torch.Tensor) -> torch.Tensor:
    R, C = x.shape
    ld = (R + 7) // 8 * 8
    out = torch.zeros((C, ld), dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_transpose_bf16(ptr(x), c_int64(x.stride(0)), ptr(out), c_int64(ld), c_int(R), c_int(C), stream_ptr()))
    return out[:, :R]


def gemm_f32out(a: torch.Tensor, b: torch.Tensor, scale: float) -> torch.Tensor:
    """fp32 [M, N] = (a [M, K] @ b [N, K]^T) * scale."""
    M, K = a.shape
    N = b.shape[0]
    ldo = (N + 7) // 8 * 8
    out = torch.empty((M, ldo), dtype=torch.float32, device=a.device)
    check(lib().fvb_gemm_f32out(ptr(a), c_int64(a.stride(0)), ptr(b), c_int64(b.stride(0)), _f32p(out), c_int64(ldo), c_int(M),
                                c_int(N), c_int(K), c_float(scale), stream_ptr()))
    return out[:, :N]


def softmax_rows_f32(x: torch.Tensor) -> torch.Tensor:
    rows, n = x.shape
    ld = (n + 7) // 8 * 8
    out = (torch.zeros if ld != n else torch.empty)((rows, ld), dtype=torch.bfloat16, device=x.device)
    check(lib().fvb_softmax_rows_f32(_f32p(x), c_int64(x.stride(0)), ptr(out), c_int64(ld), c_int64(rows), c_int(n), stream_ptr()))
    return out[:, :n]


def clamp_to_nchw(x: torch.Tensor, C: int) -> torch.Tensor:
    """x: [T, H, W, ld] bf16 -> fp32 [C, T, H, W] clamped to [-1, 1]."""
    T, H, W, ld = x.shape
    out = torch.empty((C, T, H, W), dtype=torch.float32, device=x.device)
    check(lib().fvb_clamp_to_nchw(ptr(x), c_int64(ld), _f32p(out), c_int(C), c_int64(T * H * W), stream_ptr()))
    return out
