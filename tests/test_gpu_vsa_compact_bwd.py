"""GPU: the VSA backward in the compact layout (tile-major order, no pad rows) -- VideoSparseAttentionImpl.forward, its
tile / untile permutations, and the kernels under them (fvb_attention_sparse_bwd, fvb_vsa_combine_bwd_compact,
fvb_block_mean_bwd_compact). A compact tensor is the padded one (oracle.gen_golden_gpu.padded_inputs) restricted to its
valid rows; torch autograd of the padded VSA composite (tests/vsa_bwd_ref.py) restricted to those rows is the truth.
Rule of tests/test_gpu_vsa_bwd.py: relL2(ours, fp32) <= relL2(bf16 composite, fp32) + 2e-3."""
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN
from oracle.gen_golden_gpu import padded_inputs
from util import rel_l2
import vsa_bwd_ref as ref

pytestmark = pytest.mark.gpu

SMALL = torch.load(os.path.join(GOLDEN, "vsa_gpu_small.pt"))
# the three grids of vsa_gpu_small.pt (2 heads) and one at Wan 14B width: 40 heads of 128
GRIDS = [(fx["shape"], fx["heads"], fx["topk"], fx["seed"]) for fx in SMALL.values()]
GRIDS.append(((9, 13, 10), 40, 8, 14))
GRID_IDS = ["x".join(map(str, g[0])) + f"_h{g[1]}" for g in GRIDS]
SENTINEL = -12345.0


def _tables(vbs):
    vbs = vbs.to(torch.int32).cuda()
    off = torch.zeros(vbs.numel() + 1, dtype=torch.int32, device="cuda")
    off[1:] = torch.cumsum(vbs, 0)
    row_block = torch.repeat_interleave(torch.arange(vbs.numel(), device="cuda", dtype=torch.int32), vbs.long())
    return vbs, off, row_block


def _compact(x, valid):
    """[1, H, S_pad, 128] padded -> [1, S, H, 128] compact (the valid rows, tile-major)."""
    return x[:, :, valid].transpose(1, 2).contiguous()


def _case(shape, H, seed):
    q, k, v, gate, vbs, valid = padded_inputs(tuple(shape), H, seed)
    g = torch.Generator().manual_seed(seed + 1000)
    dO = (torch.randn(q.shape, generator=g) * valid[None, None, :, None]).bfloat16()
    return q, k, v, gate, vbs, valid, dO


def _md(vbs, topk):
    """the fields VideoSparseAttentionImpl.forward reads; the sparsity gives exactly `topk` blocks per row"""
    vbs, off, row_block = _tables(vbs)
    n = vbs.numel()
    return SimpleNamespace(VSA_sparsity=1.0 - (topk - 0.5) / n, variable_block_sizes=vbs, block_offsets=off,
                           row_block=row_block)


def _impl():
    from fastvideo_b200.attention import VideoSparseAttentionImpl
    return VideoSparseAttentionImpl(num_heads=1, head_size=128)


def _ours_compact(qc, kc, vc, gc, dOc, vbs, topk, block_map=None):
    """(out, grads) on compact [1, S, H, 128] tensors through VideoSparseAttentionImpl.forward, or through the autograd
    Function with a fixed block map."""
    from fastvideo_b200 import vsa
    md = _md(vbs, topk)
    leaves = [t.cuda().requires_grad_(True) for t in ((qc, kc, vc) if gc is None else (qc, kc, vc, gc))]
    g = leaves[3] if gc is not None else None
    if block_map is None:
        out = _impl().forward(*leaves[:3], g, md)
    else:
        out = vsa._VideoSparseAttnFn.apply(*leaves[:3], g, md.variable_block_sizes, topk, block_map.cuda(),
                                           md.block_offsets, md.row_block)
    out.backward(dOc.cuda())
    return out.detach(), [t.grad for t in leaves]


def _block_map(qc, kc, vc, vbs, topk):
    from fastvideo_b200 import vsa
    v32, off, rb = _tables(vbs)
    _, aux = vsa.video_sparse_attn_bshd(qc.cuda(), kc.cuda(), vc.cuda(), v32, topk, block_off=off, row_block=rb,
                                        return_aux=True)
    return aux["mask"].cpu()


def _composite_grads(q, k, v, gate, vbs, block_map, dO, dtype):
    leaves = [t.cuda().to(dtype).requires_grad_(True) for t in ((q, k, v) if gate is None else (q, k, v, gate))]
    out = ref.composite(*leaves[:3], leaves[3] if gate is not None else None, vbs, block_map.cuda())
    out.backward(dO.cuda().to(dtype))
    return [t.grad for t in leaves]


def _check_parity(ours_c, valid, q, k, v, gate, vbs, block_map, dO):
    """ours_c: compact gradients; the composite's padded gradients restricted to the valid rows are the truth"""
    truth = _composite_grads(q, k, v, gate, vbs, block_map, dO, torch.float32)
    bf16 = _composite_grads(q, k, v, gate, vbs, block_map, dO, torch.bfloat16)
    vd = valid.cuda()
    report = {}
    for name, mine, t32, t16 in zip(("dq", "dk", "dv", "d_gate"), ours_c, truth, bf16):
        assert torch.isfinite(mine).all(), name
        t32c, t16c = _compact(t32, vd), _compact(t16, vd)
        e_mine, e_bf16 = rel_l2(mine, t32c), rel_l2(t16c, t32c)
        report[name] = (e_mine, e_bf16)
        assert e_mine <= e_bf16 + 2e-3, (name, e_mine, e_bf16)
    print("relL2 from fp32 (ours, bf16 composite):", {n: (f"{a:.2e}", f"{b:.2e}") for n, (a, b) in report.items()})


def _compact_case(grid, with_gate=True):
    shape, H, topk, seed = grid
    q, k, v, gate, vbs, valid, dO = _case(shape, H, seed)
    qc, kc, vc, gc, dOc = (_compact(t, valid) for t in (q, k, v, gate, dO))
    return (q, k, v, gate if with_gate else None, vbs, valid, dO), (qc, kc, vc, gc if with_gate else None, dOc), topk


# ------------------------------------------------------------------------------------------- 1 + 2: impl gradients
@pytest.mark.parametrize("grid", GRIDS, ids=GRID_IDS)
def test_impl_gradients_against_fp32_composite(grid):
    (q, k, v, gate, vbs, valid, dO), (qc, kc, vc, gc, dOc), topk = _compact_case(grid)
    _, grads = _ours_compact(qc, kc, vc, gc, dOc, vbs, topk)
    _check_parity(grads, valid, q, k, v, gate, vbs, _block_map(qc, kc, vc, vbs, topk), dO)


def test_impl_gradients_without_gate():
    (q, k, v, _, vbs, valid, dO), (qc, kc, vc, _, dOc), topk = _compact_case(GRIDS[1], with_gate=False)
    _, grads = _ours_compact(qc, kc, vc, None, dOc, vbs, topk)
    assert len(grads) == 3
    _check_parity(grads, valid, q, k, v, None, vbs, _block_map(qc, kc, vc, vbs, topk), dO)


def test_empty_q_and_k_lists():
    """a fixed block map with q tiles that attend nothing and kv tiles that nobody attends (empty k -> q lists)"""
    (q, k, v, gate, vbs, valid, dO), (qc, kc, vc, gc, dOc), topk = _compact_case(GRIDS[2])
    block_map = _block_map(qc, kc, vc, vbs, topk)
    block_map[0, 0, 3] = False
    block_map[0, 1, 0] = False
    block_map[0, 1, 7] = False
    block_map[0, 0, :, 5] = False
    block_map[0, 1, :, 2] = False
    _, grads = _ours_compact(qc, kc, vc, gc, dOc, vbs, topk, block_map=block_map)
    _check_parity(grads, valid, q, k, v, gate, vbs, block_map, dO)


def test_full_plugin_path_is_a_permutation_of_the_compact_gradients():
    """preprocess_qkv -> chunk -> forward -> postprocess_output on a stacked q/k/v/gate in original token order: tile and
    untile are pure permutations, so the gradients are the compact ones permuted, bit for bit."""
    from fastvideo_b200.attention import VideoSparseAttentionMetadataBuilder, compute_topk
    shape = GRIDS[1][0]
    (_, _, _, _, vbs, _, _), (qc, kc, vc, gc, dOc), topk = _compact_case(GRIDS[1])
    md = VideoSparseAttentionMetadataBuilder().build(0, tuple(shape), (1, 1, 1), 1.0 - (topk - 0.5) / vbs.numel(),
                                                     torch.device("cuda"))
    assert compute_topk(md.VSA_sparsity, md.variable_block_sizes.numel()) == topk
    assert torch.equal(md.variable_block_sizes.cpu(), vbs.to(torch.int32))
    _, want = _ours_compact(qc, kc, vc, gc, dOc, vbs, topk)
    tp, rev = md.tile_partition_indices, md.reverse_tile_partition_indices
    # original order: x[j] = compact[rev[j]] (tile gathers compact[i] = x[tp[i]])
    stack = torch.cat([t.cuda() for t in (qc, kc, vc, gc)])[:, rev].contiguous().requires_grad_(True)
    impl = _impl()
    tiled = impl.preprocess_qkv(stack, md)
    q, k, v, g = tiled.chunk(4, dim=0)
    out = impl.postprocess_output(impl.forward(q, k, v, g, md), md)
    assert out.grad_fn is not None
    out.backward(dOc.cuda()[:, rev])
    for i, w in enumerate(want):
        assert torch.equal(stack.grad[i:i + 1][:, tp], w), i


# ------------------------------------------------------------------------------------------- 5: forward, determinism
@pytest.mark.parametrize("with_gate", [True, False])
def test_forward_with_grad_is_bit_identical(with_gate):
    (_, _, _, _, vbs, _, _), (qc, kc, vc, gc, _), topk = _compact_case(GRIDS[0], with_gate)
    md = _md(vbs, topk)
    qd, kd, vd = qc.cuda(), kc.cuda(), vc.cuda()
    gd = gc.cuda() if with_gate else None
    with torch.no_grad():
        ref_out = _impl().forward(qd, kd, vd, gd, md)
    assert ref_out.grad_fn is None
    out = _impl().forward(qd.clone().requires_grad_(True), kd, vd, gd, md)
    assert out.requires_grad
    assert torch.equal(out.detach(), ref_out)


def test_backward_is_deterministic():
    (_, _, _, _, vbs, _, _), (qc, kc, vc, gc, dOc), topk = _compact_case(GRIDS[3])
    out1, g1 = _ours_compact(qc, kc, vc, gc, dOc, vbs, topk)
    out2, g2 = _ours_compact(qc, kc, vc, gc, dOc, vbs, topk)
    assert torch.equal(out1, out2)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------- 3 + 4: the kernel alone
RAGGED = torch.tensor([64, 16, 64, 4, 64, 33, 1, 50, 64], dtype=torch.int32)


def _lists(block_map):
    from fastvideo_b200 import ops
    q2k = ops.map_to_index(block_map.cuda().contiguous())
    k2q = ops.map_to_index(block_map.cuda().transpose(-1, -2).contiguous())
    return q2k, k2q


def _sentinel_views(B, S, H, pad=96):
    """three [B, S, H, 128] views into sentinel-filled buffers with `pad` rows of margin on each side"""
    bufs = [torch.full((B, S + 2 * pad, H, 128), SENTINEL, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
    return bufs, [b[:, pad:pad + S] for b in bufs]


def _masked_attention_grads(q, k, v, keep, dO, dtype, scale):
    leaves = [t.to(dtype).requires_grad_(True) for t in (q, k, v)]
    qh, kh, vh = (t.transpose(1, 2) for t in leaves)
    p = ref.masked_softmax((qh @ kh.transpose(-1, -2)) * scale, keep)
    (p @ vh).transpose(1, 2).backward(dO.to(dtype))
    return [t.grad for t in leaves]


def _kernel_inputs(S, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn(1, S, H, 128, device="cuda", generator=g).bfloat16() for _ in range(4)]


def test_kernel_compact_against_masked_attention():
    from fastvideo_b200 import ops
    vbs, off, _ = _tables(RAGGED)
    nblk, S, H = RAGGED.numel(), int(RAGGED.sum()), 2
    q, k, v, dO = _kernel_inputs(S, H, 5)
    g = torch.Generator().manual_seed(6)
    block_map = torch.rand(1, H, nblk, nblk, generator=g) < 0.45
    block_map[0, 0, 2] = False       # a q tile without keys
    block_map[0, 1, :, 4] = False    # a kv tile nobody attends
    (q2k_idx, q2k_num), (k2q_idx, k2q_num) = _lists(block_map)
    o, lse = ops.attention_blocklist(q, k, v, q2k_idx, q2k_num, q_off=off, kv_off=off, q_len=vbs, kv_len=vbs, nkb=nblk,
                                     return_lse=True)
    bufs, outs = _sentinel_views(1, S, H)
    dq, dk, dv = ops.attention_sparse_bwd(q, k, v, o, lse, dO, q2k_idx, q2k_num, k2q_idx, k2q_num, q_off=off, q_len=vbs,
                                          kv_off=off, kv_len=vbs, out=outs)
    for b in bufs:  # nothing outside [0, S) is written, every row inside is
        assert (b[:, :96] == SENTINEL).all() and (b[:, 96 + S:] == SENTINEL).all()
        assert not (b[:, 96:96 + S] == SENTINEL).all(-1).any()
    tile = torch.repeat_interleave(torch.arange(nblk), RAGGED.long())
    keep = block_map[:, :, tile][:, :, :, tile].cuda()
    truth = _masked_attention_grads(q, k, v, keep, dO, torch.float32, 128 ** -0.5)
    bf16 = _masked_attention_grads(q, k, v, keep, dO, torch.bfloat16, 128 ** -0.5)
    for name, mine, t32, t16 in zip(("dq", "dk", "dv"), (dq, dk, dv), truth, bf16):
        e_mine, e_bf16 = rel_l2(mine, t32), rel_l2(t16, t32)
        assert e_mine <= e_bf16 + 2e-3, (name, e_mine, e_bf16)
    # the empty q tile gets exact zeros in dq, the unattended kv tile in dk and dv
    assert not dq[0, int(off[2]):int(off[3]), 0].any()
    assert not dk[0, int(off[4]):int(off[5]), 1].any() and not dv[0, int(off[4]):int(off[5]), 1].any()


def test_kernel_padded_agrees_with_mma_sync_kernel():
    """same lists, padded layout (64-row tiles, variable_block_sizes valid rows): the wgmma kernel against
    fvb_attention_blocklist_bwd within the parity rule; pad rows are never written"""
    from fastvideo_b200 import ops
    shape, H, topk, seed = GRIDS[2]
    q, k, v, gate, vbs, valid, dO = _case(shape, H, seed)
    qt, kt, vt, dOt = (t.cuda().transpose(1, 2) for t in (q, k, v, dO))
    nblk = vbs.numel()
    v32 = vbs.to(torch.int32).cuda()
    g = torch.Generator().manual_seed(seed)
    block_map = torch.rand(1, H, nblk, nblk, generator=g) < 0.3
    block_map[0, 0, 1] = False
    (q2k_idx, q2k_num), (k2q_idx, k2q_num) = _lists(block_map)
    o, lse = ops.attention_blocklist(qt, kt, vt, q2k_idx, q2k_num, q_len=v32, kv_len=v32, nkb=nblk, return_lse=True)
    old = ops.attention_blocklist_bwd(qt, kt, vt, o, lse, dOt, q2k_idx, q2k_num, k2q_idx, k2q_num, kv_len=v32)
    bufs, outs = _sentinel_views(1, 64 * nblk, H)
    new = ops.attention_sparse_bwd(qt, kt, vt, o, lse, dOt, q2k_idx, q2k_num, k2q_idx, k2q_num, q_len=v32, kv_len=v32,
                                   out=outs)
    vd = valid.cuda()
    keep = ref.token_keep(block_map, vbs).cuda() & vd[None, None, None, :]
    truth = _masked_attention_grads(qt, kt, vt, keep, dOt, torch.float32, 128 ** -0.5)
    bf16 = _masked_attention_grads(qt, kt, vt, keep, dOt, torch.bfloat16, 128 ** -0.5)
    for name, a, b, t32, t16 in zip(("dq", "dk", "dv"), new, old, truth, bf16):
        a_v, b_v, t32_v, t16_v = a[:, vd], b[:, vd], t32[:, vd], t16[:, vd]
        e_bf16 = rel_l2(t16_v, t32_v)
        assert rel_l2(a_v, t32_v) <= e_bf16 + 2e-3, name
        assert rel_l2(a_v, b_v) <= e_bf16 + 2e-3, (name, rel_l2(a_v, b_v), e_bf16)
        assert (a[:, ~vd] == SENTINEL).all(), name
    for b in bufs:
        assert (b[:, :96] == SENTINEL).all() and (b[:, -96:] == SENTINEL).all()


# ------------------------------------------------------------------------------------------- 6: compact row kernels
def _bf16_close(got, exact, name):
    got, exact = got.double().cpu(), exact.double().cpu()
    tol = exact.abs() * 2.0 ** -7 + exact.abs().max() * 1e-5
    bad = (got - exact).abs() > tol
    assert not bad.any(), (name, int(bad.sum()), float((got - exact).abs().max()))


@pytest.mark.parametrize("with_gate", [True, False])
def test_kernel_vsa_combine_bwd_compact(with_gate):
    from fastvideo_b200 import ops
    torch.manual_seed(1)
    vbs, off, _ = _tables(RAGGED)
    B, H, nblk, S = 2, 3, RAGGED.numel(), int(RAGGED.sum())
    dO, gate = (torch.randn(B, S, H, 128).bfloat16() for _ in range(2))
    out_c = torch.randn(B, H, nblk, 128).bfloat16()
    dg = torch.full((B, S, H, 128), float("nan"), dtype=torch.bfloat16, device="cuda") if with_gate else None
    d_out_c, d_out_c_t = ops.vsa_combine_bwd(dO.cuda(), out_c.cuda(), gate.cuda() if with_gate else None, vbs, d_gate=dg,
                                             block_off=off)
    tile = torch.repeat_interleave(torch.arange(nblk), RAGGED.long())
    oc_rows = out_c.double()[:, :, tile].transpose(1, 2)  # [B, S, H, 128]
    if with_gate:
        # a product of two bf16 values is exact in fp32: one rounding, so bit-exact
        assert torch.equal(dg.cpu(), (dO.double() * oc_rows).bfloat16())
    prod = dO.double() * (gate.double() if with_gate else 1.0)
    want = torch.zeros(B, nblk, H, 128, dtype=torch.float64).index_add_(1, tile, prod).transpose(1, 2)
    _bf16_close(d_out_c, want, "d_out_c")
    assert torch.equal(d_out_c_t, d_out_c.transpose(-1, -2))


def test_kernel_block_mean_bwd_compact():
    from fastvideo_b200 import ops
    torch.manual_seed(2)
    vbs, off, row_block = _tables(RAGGED)
    B, H, nblk, S = 2, 3, RAGGED.numel(), int(RAGGED.sum())
    dx_s = torch.randn(B, S, H, 128).bfloat16()
    d_mean = torch.randn(B, H, nblk, 128).bfloat16()
    got = ops.block_mean_bwd(dx_s.cuda(), d_mean.cuda(), vbs, block_off=off, row_block=row_block)
    tile = torch.repeat_interleave(torch.arange(nblk), RAGGED.long())
    # fp32 division then fp32 addition, one rounding to bf16: bit-exact with the same fp32 steps
    per_row = (d_mean.float() / RAGGED.float().view(1, 1, -1, 1))[:, :, tile].transpose(1, 2)
    want = (dx_s.float() + per_row).bfloat16()
    assert torch.equal(got.cpu(), want)
    buf = dx_s.cuda().clone()
    ops.block_mean_bwd(buf, d_mean.cuda(), vbs, out=buf, block_off=off, row_block=row_block)
    assert torch.equal(buf.cpu(), want)
