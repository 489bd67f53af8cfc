"""GPU: the dense attention backward (fvb_attention_bwd through attention._DenseAttnFn / B200AttentionImpl) and the RMSNorm
backward (fvb_rmsnorm_bwd through plugin.rms_norm_forward_cuda). fp32 autograd is the truth; bf16 torch autograd of the
same formula stands in for the reference's bf16 rounding. Rule: relL2(ours, fp32) <= relL2(bf16 autograd, fp32) + 2e-3."""
import types
from ctypes import c_float, c_int, c_int64

import pytest
import torch

from util import rel_l2
import rmsnorm_bwd_ref

pytestmark = pytest.mark.gpu

TOL = 2e-3


def _inputs(B, H, Sq, Skv, seed):
    g = torch.Generator().manual_seed(seed)
    q, dO = (torch.randn(B, Sq, H, 128, generator=g).bfloat16() for _ in range(2))
    k, v = (torch.randn(B, Skv, H, 128, generator=g).bfloat16() for _ in range(2))
    return q, k, v, dO


def _torch_grads(q, k, v, dO, scale, dtype):
    leaves = [t.cuda().to(dtype).requires_grad_(True) for t in (q, k, v)]
    qh, kh, vh = (t.transpose(1, 2) for t in leaves)
    p = torch.softmax((qh @ kh.transpose(-1, -2)) * scale, dim=-1)
    (p @ vh).transpose(1, 2).backward(dO.cuda().to(dtype))
    return [t.grad for t in leaves]


def _ours(q, k, v, dO, scale=None):
    """(out, [dq, dk, dv]) through the public dense backend on the given CUDA views."""
    from fastvideo_b200.attention import B200AttentionImpl
    impl = B200AttentionImpl(q.shape[2], 128, softmax_scale=scale)
    out = impl.forward(q, k, v)
    out.backward(dO)
    return out.detach()


def _check(q, k, v, dO, grads, scale):
    truth = _torch_grads(q, k, v, dO, scale, torch.float32)
    floor = _torch_grads(q, k, v, dO, scale, torch.bfloat16)
    for name, ours, t, f in zip(("dq", "dk", "dv"), grads, truth, floor):
        assert torch.isfinite(ours.float()).all(), name
        if t.norm() == 0:  # Skv = 1: P = 1, dP = delta, so dS and dq are exactly 0; ours holds the rounding residue of ex2
            assert ours.float().abs().max() < 1e-5, name
            continue
        e, fl = rel_l2(ours, t), rel_l2(f, t)
        assert e <= fl + TOL, f"{name}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + {TOL}"


def _leaves(q, k, v):
    return [t.cuda().requires_grad_(True) for t in (q, k, v)]


@pytest.mark.parametrize("B,H,Sq,Skv", [(2, 2, 200, 77), (1, 2, 4096, 4096), (1, 12, 3000, 512), (1, 40, 1560, 257),
                                        (1, 2, 1, 64), (1, 2, 64, 1)])
def test_grads_match_autograd(B, H, Sq, Skv):
    q, k, v, dO = _inputs(B, H, Sq, Skv, seed=Sq + Skv)
    lq, lk, lv = _leaves(q, k, v)
    _ours(lq, lk, lv, dO.cuda())
    _check(q, k, v, dO, [lq.grad, lk.grad, lv.grad], 128 ** -0.5)


def test_softmax_scale():
    q, k, v, dO = _inputs(1, 3, 333, 190, seed=5)
    lq, lk, lv = _leaves(q, k, v)
    _ours(lq, lk, lv, dO.cuda(), scale=0.05)
    _check(q, k, v, dO, [lq.grad, lk.grad, lv.grad], 0.05)


def test_bhsd_views_and_fused_qkv():
    B, H, S = 2, 4, 321
    q, k, v, dO = _inputs(B, H, S, S, seed=9)
    # BHSD storage, passed as BSHD views
    bh = [t.cuda().transpose(1, 2).contiguous().requires_grad_(True) for t in (q, k, v)]
    _ours(*(t.transpose(1, 2) for t in bh), dO.cuda().transpose(1, 2).contiguous().transpose(1, 2))
    _check(q, k, v, dO, [t.grad.transpose(1, 2) for t in bh], 128 ** -0.5)
    # one fused [B, S, 3 H 128] buffer
    qkv = torch.cat([t.reshape(B, S, H * 128) for t in (q, k, v)], dim=-1).cuda().requires_grad_(True)
    views = [qkv[..., i * H * 128:(i + 1) * H * 128].view(B, S, H, 128) for i in range(3)]
    _ours(*views, dO.cuda())
    g = qkv.grad.view(B, S, 3, H, 128)
    _check(q, k, v, dO, [g[:, :, i] for i in range(3)], 128 ** -0.5)


def test_agrees_with_blocklist_kernel():
    from fastvideo_b200 import ops
    B, H, S = 1, 2, 320
    q, k, v, dO = _inputs(B, H, S, S, seed=3)
    qc, kc, vc, dc = (t.cuda() for t in (q, k, v, dO))
    out, lse = ops.attention(qc, kc, vc, return_lse=True)
    n = S // 64
    idx = torch.arange(n, dtype=torch.int32, device="cuda").expand(B, H, n, n).contiguous()
    num = torch.full((B, H, n), n, dtype=torch.int32, device="cuda")
    old = ops.attention_blocklist_bwd(qc, kc, vc, out, lse, dc, idx, num, idx, num)
    new = ops.attention_bwd(qc, kc, vc, out, lse, dc)
    _check(q, k, v, dO, new, 128 ** -0.5)
    _check(q, k, v, dO, old, 128 ** -0.5)
    for a, b in zip(new, old):
        assert rel_l2(a, b) <= 4e-3


def test_forward_unchanged_and_backward_deterministic():
    from fastvideo_b200 import ops
    from fastvideo_b200.attention import B200AttentionImpl
    q, k, v, dO = (t.cuda() for t in _inputs(2, 3, 300, 150, seed=11))
    impl = B200AttentionImpl(3, 128)
    with torch.no_grad():
        plain = impl.forward(q, k, v)
    assert torch.equal(plain, ops.attention(q, k, v, softmax_scale=128 ** -0.5))  # the no-grad path is the parent's call
    runs = []
    for _ in range(2):
        leaves = [t.clone().requires_grad_(True) for t in (q, k, v)]
        out = impl.forward(*leaves)
        assert out.grad_fn is not None and torch.equal(out.detach(), plain)
        out.backward(dO)
        runs.append([t.grad for t in leaves])
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_rows_past_sq_are_not_written():
    from fastvideo_b200 import ops
    from fastvideo_b200._lib import check, lib, ptr, stream_ptr
    B, H, Sq, Skv = 1, 2, 100, 70
    q, k, v, dO = (t.cuda() for t in _inputs(B, H, Sq, Skv, seed=2))
    out, lse = ops.attention(q, k, v, return_lse=True)
    sentinel = -12345.0
    bufs = [torch.full((B, S + 64, H, 128), sentinel, dtype=torch.bfloat16, device="cuda") for S in (Sq, Skv, Skv)]
    views = [bufs[0][:, :Sq], bufs[1][:, :Skv], bufs[2][:, :Skv]]
    delta = torch.empty(B * H * Sq, dtype=torch.float32, device="cuda")
    st = ops._bsh_strides
    check(lib().fvb_attention_bwd(ptr(q), ptr(k), ptr(v), ptr(out), ptr(dO), ops._f32p(lse), c_int64(H * Sq), c_int64(Sq),
                                  *(ptr(t) for t in views), ops._f32p(delta), st(q), st(k), st(v), st(out), st(dO),
                                  *(st(t) for t in views), c_int(B), c_int(H), c_int(Sq), c_int(Skv), c_int(128),
                                  c_float(128 ** -0.5), stream_ptr()))
    ref = ops.attention_bwd(q, k, v, out, lse, dO)
    for buf, view, r, S in zip(bufs, views, ref, (Sq, Skv, Skv)):
        assert (buf[:, S:] == sentinel).all()
        assert torch.equal(view, r)


def test_zero_do_rows():
    from fastvideo_b200 import ops
    B, H, Sq, Skv, keep = 1, 4, 230, 190, 150
    q, k, v, dO = (t.cuda() for t in _inputs(B, H, Sq, Skv, seed=4))
    dO[:, keep:] = 0
    out, lse = ops.attention(q, k, v, return_lse=True)
    dq, dk, dv = ops.attention_bwd(q, k, v, out, lse, dO)
    assert (dq[:, keep:] == 0).all()
    out2, lse2 = ops.attention(q[:, :keep], k, v, return_lse=True)
    dq2, dk2, dv2 = ops.attention_bwd(q[:, :keep], k, v, out2, lse2, dO[:, :keep])
    assert rel_l2(dq[:, :keep], dq2) < 1e-3
    assert rel_l2(dk, dk2) < 1e-3 and rel_l2(dv, dv2) < 1e-3


# ---------------------------------------------------------------- RMSNorm (plugin.rms_norm_forward_cuda)
def _rms_self(weight, eps=1e-6):
    """A stand-in for the reference RMSNorm module: the attributes rms_norm_forward_cuda reads and layernorm.py's
    forward_native."""
    self = types.SimpleNamespace(weight=weight, variance_epsilon=eps, hidden_size=weight.numel(), has_weight=True,
                                 variance_size_override=None)

    def forward_native(x, residual=None):
        orig = x.dtype
        xf = x.to(torch.float32)
        xf = xf * torch.rsqrt(xf.pow(2).mean(dim=-1, keepdim=True) + eps)
        return xf.to(orig) * self.weight

    self.forward_native = forward_native
    return self


def _rms_case(D, wdtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(2, 1000, D, generator=g) * 3).bfloat16().cuda()
    w = (1 + 0.2 * torch.randn(D, generator=g)).to(wdtype).cuda()
    dy = torch.randn(2, 1000, D, generator=g).bfloat16().cuda()
    return x, w, dy


def _rms_grads(fn_self, x, dy, cast):
    xl = x.to(cast).detach().requires_grad_(True)
    out = fn_self.forward_native(xl)
    out.backward(dy.to(out.dtype))
    return xl.grad, fn_self.weight.grad


@pytest.mark.parametrize("D", [1536, 5120])
@pytest.mark.parametrize("wdtype", [torch.bfloat16, torch.float32])
def test_rmsnorm_grads(D, wdtype):
    from fastvideo_b200 import plugin
    x, w, dy = _rms_case(D, wdtype, seed=D)
    ours_self = _rms_self(w.clone().requires_grad_(True))
    xl = x.clone().requires_grad_(True)
    out = plugin.rms_norm_forward_cuda(ours_self, xl)
    with torch.no_grad():
        plain = plugin.rms_norm_forward_cuda(ours_self, x)
    assert torch.equal(out.detach(), plain)  # forward with grad is the no-grad forward
    out.backward(dy.to(out.dtype))
    truth_self = _rms_self(w.float().clone().requires_grad_(True))
    tdx, tdw = _rms_grads(truth_self, x, dy, torch.float32)
    floor_self = _rms_self(w.clone().requires_grad_(True))
    fdx, fdw = _rms_grads(floor_self, x, dy, torch.bfloat16)
    for name, ours, t, f in (("dx", xl.grad, tdx, fdx), ("dw", ours_self.weight.grad, tdw, fdw)):
        e, fl = rel_l2(ours, t), rel_l2(f, t)
        assert e <= fl + TOL, f"{name}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + {TOL}"


def test_rmsnorm_kernel_matches_restatement_and_is_deterministic():
    from fastvideo_b200 import ops
    x, w, dy = _rms_case(1536, torch.bfloat16, seed=1)
    x2, dy2 = x.view(-1, 1536), dy.view(-1, 1536)
    dx, dw = ops.rmsnorm_bwd(x2, w, dy2, 1e-6)
    dx_r, dw_r = rmsnorm_bwd_ref.rmsnorm_bwd(x2.cpu(), w.cpu(), dy2.cpu(), 1e-6, bf16_points=True)
    assert rel_l2(dx, dx_r) < 2e-3 and rel_l2(dw, dw_r) < 2e-3
    for _ in range(2):
        dx_b, dw_b = ops.rmsnorm_bwd(x2, w, dy2, 1e-6)
        assert torch.equal(dx_b, dx) and torch.equal(dw_b, dw)
