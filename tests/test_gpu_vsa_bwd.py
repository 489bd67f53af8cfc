"""GPU: the backward of video_sparse_attn (reference signature, padded layout) against torch autograd of the VSA composite
(tests/vsa_bwd_ref.py) on the same block map. fp32 autograd is the truth; bf16 autograd of the same composite stands in for
the reference's bf16 rounding. Rule of tests/test_gpu_attention_bwd.py: relL2(ours, fp32) <= relL2(bf16 composite, fp32)
+ 2e-3 for dq, dk, dv and d_gate. Plus pad rows, empty q blocks, bit-identity of the forward with and without grad,
determinism, and one test per new kernel against its formula."""
import os

import pytest
import torch

from conftest import GOLDEN
from oracle import vsa_index
from oracle.gen_golden_gpu import padded_inputs
from util import rel_l2
import vsa_bwd_ref as ref

pytestmark = pytest.mark.gpu

SMALL = torch.load(os.path.join(GOLDEN, "vsa_gpu_small.pt"))
# the three grids of vsa_gpu_small.pt (2 heads) and one at Wan 14B width: 40 heads of 128
GRIDS = [(fx["shape"], fx["heads"], fx["topk"], fx["seed"]) for fx in SMALL.values()]
GRIDS.append(((9, 13, 10), 40, 8, 14))
GRID_IDS = ["x".join(map(str, g[0])) + f"_h{g[1]}" for g in GRIDS]


def _do(shape, H, seed):
    q, k, v, gate, vbs, valid = padded_inputs(tuple(shape), H, seed)
    g = torch.Generator().manual_seed(seed + 1000)
    dO = (torch.randn(q.shape, generator=g) * valid[None, None, :, None]).bfloat16()
    return q, k, v, gate, vbs, valid, dO


def _ours(q, k, v, gate, vbs, topk, dO, block_map=None):
    """(out, [dq, dk, dv, d_gate]) through the public entry point, or through the autograd Function with a fixed block map."""
    from fastvideo_b200 import vsa
    leaves = [t.cuda().requires_grad_(True) for t in ((q, k, v) if gate is None else (q, k, v, gate))]
    g = leaves[3] if gate is not None else None
    if block_map is None:
        out = vsa.video_sparse_attn(*leaves[:3], vbs.cuda(), vbs.cuda(), topk, compress_attn_weight=g)
    else:
        out = vsa._VideoSparseAttnFn.apply(*leaves[:3], g, vbs.cuda(), topk, block_map.cuda())
    out.backward(dO.cuda())
    return out.detach(), [t.grad for t in leaves]


def _block_map(q, k, v, vbs, topk):
    from fastvideo_b200 import vsa
    _, aux = vsa.video_sparse_attn_bshd(*(t.cuda().transpose(1, 2) for t in (q, k, v)), vbs.cuda(), topk, return_aux=True)
    return aux["mask"].cpu()


def _composite_grads(q, k, v, gate, vbs, block_map, dO, dtype):
    leaves = [t.cuda().to(dtype).requires_grad_(True) for t in ((q, k, v) if gate is None else (q, k, v, gate))]
    out = ref.composite(*leaves[:3], leaves[3] if gate is not None else None, vbs, block_map.cuda())
    out.backward(dO.cuda().to(dtype))
    return [t.grad for t in leaves]


def _check_parity(ours, vbs, q, k, v, gate, block_map, dO):
    truth = _composite_grads(q, k, v, gate, vbs, block_map, dO, torch.float32)
    bf16 = _composite_grads(q, k, v, gate, vbs, block_map, dO, torch.bfloat16)
    report = {}
    for name, mine, t32, t16 in zip(("dq", "dk", "dv", "d_gate"), ours, truth, bf16):
        assert torch.isfinite(mine).all(), name
        e_mine, e_bf16 = rel_l2(mine, t32), rel_l2(t16, t32)
        report[name] = (e_mine, e_bf16)
        assert e_mine <= e_bf16 + 2e-3, (name, e_mine, e_bf16)
    print("relL2 from fp32 (ours, bf16 composite):", {n: (f"{a:.2e}", f"{b:.2e}") for n, (a, b) in report.items()})
    return report


@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_gradients_against_fp32_composite(grid):
    shape, H, topk, seed = grid
    q, k, v, gate, vbs, valid, dO = _do(shape, H, seed)
    out, grads = _ours(q, k, v, gate, vbs, topk, dO)
    _check_parity(grads, vbs, q, k, v, gate, _block_map(q, k, v, vbs, topk), dO)
    # pad rows (the 4x16x16 grid has none): dO is zero there, so every gradient is exactly zero there
    pad = ~valid.cuda()
    for t in grads:
        assert not t[:, :, pad].any()


def test_gradients_without_gate():
    shape, H, topk, seed = GRIDS[1]
    q, k, v, _, vbs, valid, dO = _do(shape, H, seed)
    _, grads = _ours(q, k, v, None, vbs, topk, dO)
    assert len(grads) == 3
    _check_parity(grads, vbs, q, k, v, None, _block_map(q, k, v, vbs, topk), dO)


def test_empty_q_block_lists():
    """q blocks whose list is empty (a fixed block map; top-k with topk >= 1 never gives one): their rows get only the
    compression branch's gradient, and everything stays within the parity rule."""
    shape, H, topk, seed = GRIDS[2]
    q, k, v, gate, vbs, valid, dO = _do(shape, H, seed)
    block_map = _block_map(q, k, v, vbs, topk)
    block_map[0, 0, 3] = False
    block_map[0, 1, 0] = False
    block_map[0, 1, 7] = False
    _, grads = _ours(q, k, v, gate, vbs, topk, dO, block_map=block_map)
    _check_parity(grads, vbs, q, k, v, gate, block_map, dO)


@pytest.mark.parametrize("with_gate", [True, False])
def test_forward_with_grad_is_bit_identical(with_gate):
    from fastvideo_b200 import vsa
    shape, H, topk, seed = GRIDS[0]
    q, k, v, gate, vbs, _, _ = _do(shape, H, seed)
    qd, kd, vd, gd, vb = q.cuda(), k.cuda(), v.cuda(), gate.cuda() if with_gate else None, vbs.cuda()
    with torch.no_grad():
        ref_out = vsa.video_sparse_attn(qd, kd, vd, vb, vb, topk, compress_attn_weight=gd)
    qg = qd.clone().requires_grad_(True)
    out = vsa.video_sparse_attn(qg, kd, vd, vb, vb, topk, compress_attn_weight=gd)
    assert out.requires_grad
    assert torch.equal(out.detach(), ref_out)


def test_backward_is_deterministic():
    shape, H, topk, seed = GRIDS[3]
    q, k, v, gate, vbs, _, dO = _do(shape, H, seed)
    out1, g1 = _ours(q, k, v, gate, vbs, topk, dO)
    out2, g2 = _ours(q, k, v, gate, vbs, topk, dO)
    assert torch.equal(out1, out2)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------- one test per new kernel
def _bf16_close(got, exact, name):
    """got: a bf16 rounding of `exact` (fp64) after fp32 arithmetic: within one bf16 step of it everywhere."""
    got, exact = got.double().cpu(), exact.double().cpu()
    tol = exact.abs() * 2.0 ** -7 + exact.abs().max() * 1e-5  # + fp32 summation error where the sum cancels
    bad = (got - exact).abs() > tol
    assert not bad.any(), (name, int(bad.sum()), float((got - exact).abs().max()))


@pytest.mark.parametrize("with_gate", [True, False])
def test_kernel_vsa_combine_bwd(with_gate):
    from fastvideo_b200 import ops
    torch.manual_seed(1)
    vbs = torch.tensor([64, 16, 64, 4, 64, 33, 1], dtype=torch.int32)
    B, H, nblk = 2, 3, vbs.numel()
    S = 64 * nblk
    dO, gate = (torch.randn(B, H, S, 128).bfloat16() for _ in range(2))
    out_c = torch.randn(B, H, nblk, 128).bfloat16()
    dg = torch.full_like(dO, float("nan")).cuda() if with_gate else None
    d_out_c, d_out_c_t = ops.vsa_combine_bwd(dO.cuda().transpose(1, 2), out_c.cuda(), gate.cuda().transpose(1, 2) if with_gate else None,
                                             vbs.cuda(), d_gate=dg.transpose(1, 2) if with_gate else None)
    want_dg, want_doc = ref.combine_bwd(dO.double(), out_c.double(), gate.double() if with_gate else None, vbs)
    if with_gate:
        # a product of two bf16 values is exact in fp32: one rounding, so bit-exact
        assert torch.equal(dg.cpu(), want_dg.bfloat16())
    _bf16_close(d_out_c, want_doc, "d_out_c")
    assert torch.equal(d_out_c_t, d_out_c.transpose(-1, -2))


@pytest.mark.parametrize("n,batch", [(36, 3), (1440, 2), (8, 1)])
def test_kernel_softmax_rows_bwd(n, batch):
    from fastvideo_b200 import ops
    torch.manual_seed(n)
    scores = (torch.randn(batch, n, n) * 3).bfloat16().cuda()
    p = ops.softmax_rows(scores)  # [batch, n, n] view of a [.., ld] buffer, as in the forward
    dp_full = torch.randn(batch, n, p.stride(1)).bfloat16().cuda()
    dp = dp_full[..., :n]
    scale = 128 ** -0.5
    ds, ds_t, p_t = ops.softmax_rows_bwd(p, dp, scale=scale, want_transposed=True)
    _bf16_close(ds, ref.softmax_rows_bwd(p.double(), dp.double(), scale), "ds")
    assert torch.equal(ds_t, ds.transpose(-1, -2))
    assert torch.equal(p_t, p.transpose(-1, -2))
    assert torch.equal(ops.softmax_rows_bwd(p, dp, scale=scale), ds)


def test_kernel_block_mean_bwd():
    from fastvideo_b200 import ops
    torch.manual_seed(2)
    vbs = torch.tensor([64, 16, 64, 4, 64, 33, 1], dtype=torch.int32)
    B, H, nblk = 2, 3, vbs.numel()
    S = 64 * nblk
    dx_s = torch.randn(B, H, S, 128).bfloat16()
    d_mean = torch.randn(B, H, nblk, 128).bfloat16()
    got = ops.block_mean_bwd(dx_s.cuda().transpose(1, 2), d_mean.cuda(), vbs.cuda())
    # fp32 division then fp32 addition, one rounding to bf16: bit-exact with the same fp32 steps
    want = ref.block_mean_bwd(dx_s.float(), d_mean.float(), vbs).bfloat16()
    assert torch.equal(got.transpose(1, 2).cpu(), want)
    # in place, as the autograd backward calls it
    buf = dx_s.cuda().transpose(1, 2).contiguous()
    ops.block_mean_bwd(buf, d_mean.cuda(), vbs.cuda(), out=buf)
    assert torch.equal(buf.transpose(1, 2).cpu(), want)
