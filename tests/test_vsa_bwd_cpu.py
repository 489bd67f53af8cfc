"""CPU: the restated VSA backward formulas (tests/vsa_bwd_ref.py), which the GPU kernels are held to, against torch autograd
of the VSA composite in fp64, with the dense masked formula standing in for the block-sparse branch."""
import pytest
import torch

from oracle import vsa_index
import vsa_bwd_ref as ref

CASES = {
    # a ragged token grid: tiles of 64, 32, 16, ... valid rows
    "grid_5x6x7": lambda: torch.from_numpy(vsa_index.variable_block_sizes((5, 6, 7), (4, 4, 4))).to(torch.int32),
    # very short tiles, including a 4-row one
    "ragged": lambda: torch.tensor([64, 16, 64, 4, 64, 32], dtype=torch.int32),
}


def inputs(vbs, H, seed, empty_block=None):
    g = torch.Generator().manual_seed(seed)
    nblk = vbs.numel()
    S = 64 * nblk
    m = ref.valid_rows(vbs)[None, None, :, None].double()
    q, k, v, gate, dO = ((torch.randn(1, H, S, 128, generator=g, dtype=torch.float64) * m) for _ in range(5))
    block_map = torch.rand(1, H, nblk, nblk, generator=g) < 0.5
    block_map[..., torch.arange(nblk), torch.arange(nblk)] = True
    if empty_block is not None:
        block_map[0, 0, empty_block] = False
    return q, k, v, gate, dO, block_map


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("with_gate", [True, False])
@pytest.mark.parametrize("empty_block", [None, 2])
def test_restated_backward_matches_autograd_fp64(case, with_gate, empty_block):
    vbs = CASES[case]()
    q, k, v, gate, dO, block_map = inputs(vbs, H=2, seed=7, empty_block=empty_block)
    gate = gate if with_gate else None
    leaves = [t.clone().requires_grad_(True) for t in ((q, k, v, gate) if with_gate else (q, k, v))]
    out = ref.composite(*leaves[:3], leaves[3] if with_gate else None, vbs, block_map)
    assert torch.isfinite(out).all()
    out.backward(dO)
    mine = ref.backward(q, k, v, gate, vbs, block_map, dO)
    for name, got, leaf in zip(("dq", "dk", "dv", "d_gate"), mine, leaves):
        want = leaf.grad
        err = float((got - want).norm() / want.norm())
        assert err < 1e-12, (name, err)
    if not with_gate:
        assert mine[3] is None


def test_pad_rows_and_empty_blocks_get_zero_gradient():
    vbs = CASES["ragged"]()
    q, k, v, gate, dO, block_map = inputs(vbs, H=2, seed=11, empty_block=2)
    dq, dk, dv, d_gate = ref.backward(q, k, v, gate, vbs, block_map, dO)
    pad = ~ref.valid_rows(vbs)
    for t in (dq, dk, dv, d_gate):
        assert float(t[:, :, pad].abs().max()) == 0.0
    # q block 2 of head 0 attends nothing: its rows get only the compression branch's share
    dq_s, _, _ = ref.sparse_bwd(q, k, v, dO, ref.token_keep(block_map, vbs), 128 ** -0.5)
    assert float(dq_s[0, 0, 128:192].abs().max()) == 0.0
    assert float(dq_s[0, 1, 128:192].abs().max()) > 0.0


def test_grad_path_refuses_the_pair_union_kernel(monkeypatch):
    """The backward needs the block-list kernel's LSE; with the pair-union sparse kernel selected, a call that needs
    gradients is refused instead of silently running another kernel than the no-grad call would."""
    from fastvideo_b200 import ops, vsa
    monkeypatch.setattr(vsa, "SPARSE_KERNEL", "union")
    q = torch.zeros(1, 1, 64, 128, dtype=torch.bfloat16, requires_grad=True)
    vbs = torch.tensor([64], dtype=torch.int32)
    with pytest.raises(ops.FvbError):
        vsa.video_sparse_attn(q, q, q, vbs, vbs, 1)


def test_softmax_rows_bwd_is_the_softmax_jacobian_product():
    g = torch.Generator().manual_seed(3)
    s = torch.randn(3, 9, 9, generator=g, dtype=torch.float64, requires_grad=True)
    dp = torch.randn(3, 9, 9, generator=g, dtype=torch.float64)
    p = torch.softmax(s / 2.0, -1)
    p.backward(dp)
    got = ref.softmax_rows_bwd(p.detach(), dp, scale=0.5)
    assert float((got - s.grad).abs().max()) < 1e-14
