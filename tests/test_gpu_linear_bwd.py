"""GPU: the backward of the bf16 linear (fvb_linear_dgrad_bf16 / fvb_linear_wgrad_bf16 / fvb_bias_grad_bf16 through
ops.linear_bwd and plugin.linear_forward) against fp32 matmuls of the same bf16 inputs, and the gradient of a whole Wan
block routed through every differentiable piece of the plug-in against fp32 autograd."""
import os
import types
from ctypes import c_int, c_int64

import pytest
import torch

from elementwise_ref import ulp_bf16 as _ulp_bf16
from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu

TOL = 2e-3  # the end-to-end rule of the dense-attention backward: relL2(ours, fp32) <= relL2(bf16 autograd, fp32) + TOL


def _inputs(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    dy = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    return x, w, dy


def _check_grad(got, ref32, name):
    ref_rounded = ref32.bfloat16()
    assert_bf16_parity(got, ref32, ref_rounded, name=name)
    # the single bf16 rounding of an fp32 sum: only last-bit flips from the summation order
    assert (got.float() != ref_rounded.float()).float().mean().item() < 0.02, name


# (M, N, K): K is the output width of dx and dw (BN 64 / 128 / 256 and the 192-or-wider partial tile), N the dgrad
# reduction, M the wgrad reduction
SHAPES = [(1, 256, 512), (1000, 1536, 1536), (333, 200, 136), (1000, 64, 64), (777, 128, 128), (500, 136, 256),
          (600, 72, 200), (1000, 8960, 1536), (1000, 1536, 8960), (9450, 5120, 5120), (512, 10240, 5120),
          (1000, 13824, 5120), (1000, 5120, 13824)]


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_dgrad_wgrad_match_fp32(M, N, K):
    from fastvideo_b200 import ops
    x, w, dy = _inputs(M, N, K, seed=M + N + K)
    dx, dw, db = ops.linear_bwd(x, w, dy, need_dx=True, need_dw=True, need_db=False)
    assert db is None
    _check_grad(dx, dy.float() @ w.float(), f"dx {M}x{N}x{K}")
    _check_grad(dw, dy.float().t() @ x.float(), f"dw {M}x{N}x{K}")


def test_strided_x_and_dy():
    """x a column slice of a fused buffer (row stride 768), dy a column slice of a wider gradient buffer."""
    from fastvideo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(7)
    big = torch.randn(700, 3 * 256, device="cuda", generator=g).bfloat16()
    x = big[:, 256:512]
    w = (torch.randn(320, 256, device="cuda", generator=g) / 16).bfloat16()
    dbig = torch.randn(700, 320 + 96, device="cuda", generator=g).bfloat16()
    dy = dbig[:, 48:48 + 320]
    dx, dw, db = ops.linear_bwd(x, w, dy, True, True, True)
    _check_grad(dx, dy.float() @ w.float(), "dx strided")
    _check_grad(dw, dy.float().t() @ x.float(), "dw strided")
    assert torch.equal(db, ops.linear_bwd(x, w, dy.contiguous(), False, False, True)[2])
    assert torch.equal(dx, ops.linear_bwd(x.contiguous(), w, dy.contiguous(), True, False, False)[0])


@pytest.mark.parametrize("M,N", [(1, 64), (333, 1536), (9450, 5120), (75600, 5120), (1000, 13824)])
def test_bias_grad_within_one_ulp(M, N):
    """Column sums kept away from zero (dy has a positive mean), so the fp32 summation error stays far below a bf16 ulp and
    only the final rounding can differ from the fp64 sum's."""
    from fastvideo_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(M + N)
    dy = (torch.randn(M, N, device="cuda", generator=g) + 0.5).bfloat16()
    x = torch.zeros(M, 8, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(N, 8, dtype=torch.bfloat16, device="cuda")
    _, _, db = ops.linear_bwd(x, w, dy, False, False, True)
    ref = dy.double().sum(0).bfloat16().double()
    err = (db.double() - ref).abs()
    assert (err <= _ulp_bf16(ref)).all(), f"max error {err.max().item():.3e}"


def test_backward_is_deterministic():
    from fastvideo_b200 import ops
    x, w, dy = _inputs(9450, 5120, 5120, seed=1)
    a = ops.linear_bwd(x, w, dy, True, True, True)
    b = ops.linear_bwd(x, w, dy, True, True, True)
    for t, u in zip(a, b):
        assert torch.equal(t, u)


def test_outputs_untouched_outside_their_shape():
    from fastvideo_b200 import ops
    from fastvideo_b200._lib import check, lib, ptr, stream_ptr
    M, N, K = 333, 200, 136
    x, w, dy = _inputs(M, N, K, seed=5)
    ref_dx, ref_dw, ref_db = ops.linear_bwd(x, w, dy, True, True, True)
    sentinel = -12345.0
    dx = torch.full((M + 40, K + 56), sentinel, dtype=torch.bfloat16, device="cuda")
    dw = torch.full((N + 40, K + 56), sentinel, dtype=torch.bfloat16, device="cuda")
    db = torch.full((N + 24,), sentinel, dtype=torch.bfloat16, device="cuda")
    L = lib()
    check(L.fvb_linear_dgrad_bf16(ptr(dy), c_int64(N), ptr(w), c_int64(K), ptr(dx), c_int64(K + 56), c_int(M), c_int(N),
                                  c_int(K), stream_ptr()))
    check(L.fvb_linear_wgrad_bf16(ptr(dy), c_int64(N), ptr(x), c_int64(K), ptr(dw), c_int64(K + 56), c_int(M), c_int(N),
                                  c_int(K), stream_ptr()))
    ws = torch.empty(int(L.fvb_bias_grad_bf16_workspace_bytes(c_int(M), c_int(N))) // 4, dtype=torch.float32, device="cuda")
    check(L.fvb_bias_grad_bf16(ptr(dy), c_int64(N), ptr(db), ops._f32p(ws), c_int64(ws.numel() * 4), c_int(M), c_int(N),
                               stream_ptr()))
    for buf, ref, rows in ((dx, ref_dx, M), (dw, ref_dw, N)):
        assert torch.equal(buf[:rows, :K], ref)
        assert (buf[rows:] == sentinel).all() and (buf[:, K:] == sentinel).all()
    assert torch.equal(db[:N], ref_db) and (db[N:] == sentinel).all()


def test_output_width_must_be_a_multiple_of_8():
    from fastvideo_b200 import ops
    x, w, dy = _inputs(64, 64, 72, seed=2)
    x, w = x[:, :68], w[:, :68]  # row strides stay multiples of 8; the output width K = 68 is not
    with pytest.raises(ops.FvbError):
        ops.linear_bwd(x, w, dy, True, False, False)
    with pytest.raises(ops.FvbError):
        ops.linear_bwd(x, w, dy, False, True, False)


# ---------------------------------------------------------------- the autograd Function (plugin.linear_forward)
@pytest.mark.parametrize("shape,with_bias", [((2, 300, 512), True), ((700, 256), False), ((1, 1, 128), True)])
def test_linear_forward_autograd(shape, with_bias):
    from fastvideo_b200 import ops, plugin
    K, N = shape[-1], 384
    g = torch.Generator(device="cuda").manual_seed(K)
    x = torch.randn(*shape, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g).bfloat16() if with_bias else None
    dy = torch.randn(*shape[:-1], N, device="cuda", generator=g).bfloat16()
    plain = plugin.linear_forward(x, w, b)
    assert plain.grad_fn is None and plain.shape == (*shape[:-1], N)
    with torch.no_grad():
        assert torch.equal(plugin.linear_forward(x.clone().requires_grad_(True), w, b), plain)
    leaves = [x.detach().clone().requires_grad_(True), w.clone().requires_grad_(True)]
    if with_bias:
        leaves.append(b.clone().requires_grad_(True))
    out = plugin.linear_forward(*leaves, *([] if with_bias else [None]))
    assert out.grad_fn is not None and torch.equal(out.detach(), plain)
    out.backward(dy)
    dx, dw, db = ops.linear_bwd(x.detach().reshape(-1, K), w, dy.reshape(-1, N), True, True, with_bias)
    assert torch.equal(leaves[0].grad, dx.view(shape))
    assert torch.equal(leaves[1].grad, dw)
    if with_bias:
        assert torch.equal(leaves[2].grad, db)


def test_linear_forward_only_x_requires_grad():
    from fastvideo_b200 import ops, plugin
    x, w, dy = _inputs(300, 256, 512, seed=3)
    b = torch.randn(256, device="cuda").bfloat16()
    wl, bl = w.clone(), b.clone()  # no requires_grad: no dw / db is produced
    xl = x.clone().requires_grad_(True)
    plugin.linear_forward(xl, wl, bl).backward(dy)
    assert wl.grad is None and bl.grad is None
    assert torch.equal(xl.grad, ops.linear_bwd(x, w, dy, True, False, False)[0])


# ---------------------------------------------------------------- a Wan block through the plug-in, end to end
def _rms_self(weight, eps):
    """A stand-in for the reference RMSNorm module: the attributes rms_norm_forward_cuda reads."""
    return types.SimpleNamespace(weight=weight, variance_epsilon=eps, hidden_size=weight.numel(), has_weight=True,
                                 variance_size_override=None)


def _block_grads(g, dtype, dy, route_linear_norm, route_attention):
    """Gradients of x, ctx, temb6 and every parameter, plus "out:<bias>" = the gradient of the output of each key-projection
    linear (KEY_BIASES), through the oracle block, optionally routed through the plug-in's pieces."""
    from oracle import wan_ref
    from fastvideo_b200 import plugin
    from fastvideo_b200.attention import B200AttentionImpl
    D, H = g["x"].shape[-1], g["heads"]
    d = D // H
    sd = {k: v.cuda().to(dtype).requires_grad_(True) for k, v in g["sd"].items()}
    ins = {k: g[k].cuda().to(dtype).requires_grad_(True) for k in ("x", "ctx", "temb6")}
    cos, sin = (t.cuda() for t in wan_ref.rotary_tables(g["seq"], [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)]))
    saved = wan_ref.linear, wan_ref.rmsnorm
    attn_fn = B200AttentionImpl(H, d).forward if route_attention else None
    if route_linear_norm:
        wan_ref.linear = plugin.linear_forward
        wan_ref.rmsnorm = lambda x, w, eps=1e-6: plugin.rms_norm_forward_cuda(_rms_self(w, eps), x)
    outs, lin = {}, wan_ref.linear

    def keep_key_outputs(x, w, b):
        y = lin(x, w, b)
        for k in KEY_BIASES:
            if k in sd and b is sd[k]:
                y.retain_grad()
                outs["out:" + k] = y
        return y

    wan_ref.linear = keep_key_outputs
    try:
        # the oracle builds ScaleResidualLayerNormScaleShift's null shift / scale with a device-less torch.tensor([0]): the
        # CUDA default device puts it next to the block's CUDA tensors
        with torch.device("cuda"):
            y = wan_ref.wan_block(ins["x"], ins["ctx"], ins["temb6"], sd, "", H, cos, sin, attn_fn=attn_fn)
    finally:
        wan_ref.linear, wan_ref.rmsnorm = saved
    y.backward(dy.to(y.dtype))
    return {**{k: t.grad for k, t in ins.items()}, **{k: t.grad for k, t in sd.items()},
            **{k: t.grad for k, t in outs.items()}}


# Key-projection biases: softmax is invariant to a shift shared by every key, so the exact gradient of a bias added to all
# keys cancels except for what the QK RMSNorm lets through. It is ~3-5 % of the sum of the per-token gradient magnitudes,
# which amplifies any rounding difference upstream (attention backward, RMSNorm backward) 20-30x: the bias gradients sit
# at relL2 2-4e-2 from fp32, and two equally accurate bf16 pipelines (bf16 torch autograd and the plug-in) land a few e-3
# apart there, in either direction, from one dy or one run to the next (torch's own floor moves by 3e-4 between runs).
# For these biases the rule is applied where the error is made -- the gradient of the linear's output, which the bias
# gradient sums -- and the bias gradient is held to that sum: fp32 summation error plus one bf16 rounding.
KEY_BIASES = ("to_k.bias", "attn2.to_k.bias", "attn2.add_k_proj.bias")


@pytest.mark.parametrize("name", ["wan_block_dense", "wan_block_i2v"])
def test_wan_block_gradient_end_to_end(golden_dir, name):
    g = torch.load(os.path.join(golden_dir, f"{name}.pt"))
    dy = torch.randn(g["x"].shape, generator=torch.Generator().manual_seed(0)).bfloat16().cuda()
    truth = _block_grads(g, torch.float32, dy, False, False)
    floor = _block_grads(g, torch.bfloat16, dy, False, False)
    ours = _block_grads(g, torch.bfloat16, dy, True, True)
    checked = 0
    for k, t in truth.items():
        if k.startswith("out:"):  # checked with their bias below
            continue
        if t is None:  # a parameter the block does not use (attn2.norm_added_q)
            assert ours[k] is None, k
            continue
        assert ours[k] is not None, f"{k}: no gradient through the plug-in"
        assert torch.isfinite(ours[k].float()).all(), k
        if k in KEY_BIASES:
            up = "out:" + k
            e, fl = rel_l2(ours[up], truth[up]), rel_l2(floor[up], truth[up])
            assert e <= fl + TOL, f"{up}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + {TOL}"
            terms = ours[up].double().reshape(-1, ours[up].shape[-1])
            ref = terms.sum(0)
            bound = _ulp_bf16(ref.bfloat16().double()) + terms.shape[0] * 2.0 ** -24 * terms.abs().sum(0)
            assert ((ours[k].double() - ref).abs() <= bound).all(), f"{k}: not the column sum of its output gradient"
            checked += 1
            continue
        e, fl = rel_l2(ours[k], t), rel_l2(floor[k], t)
        assert e <= fl + TOL, f"{k}: relL2 {e:.3e} > bf16 autograd {fl:.3e} + {TOL}"
        checked += 1
    assert checked == len(g["sd"]) + 3 - (1 if name == "wan_block_i2v" else 0)
