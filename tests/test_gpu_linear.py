"""GPU: wgmma GEMM + fused epilogues against an fp32 torch reference of the same op (rounding mirrored)."""
import pytest
import torch
import torch.nn.functional as F

from util import assert_bf16_parity, rel_l2

pytestmark = pytest.mark.gpu


def ref_linear(x, w, b, epi, resid, gate):
    acc = x.float() @ w.float().t()
    if b is not None:
        acc = acc + b.float()
    y = acc.bfloat16()  # F.linear's bf16 output (fastvideo/layers/linear.py:146-156)
    if epi == 0: return acc, y
    if epi == 1: return F.gelu(acc, approximate="tanh"), F.gelu(y.float(), approximate="tanh").bfloat16()
    if epi == 2: return resid.float() + acc * gate, resid.float() + y.float() * gate
    if epi == 3: return resid.float() + acc * gate, (resid.float() + y.float() * gate).bfloat16()
    if epi == 4: return resid.float() + acc, (resid.float() + y.float()).bfloat16()


@pytest.mark.parametrize("M,N,K,epi", [(128, 256, 64, 0), (256, 512, 512, 0), (1000, 1536, 1536, 0), (333, 128, 192, 0),
                                       (200, 64, 512, 0), (1, 1536, 256, 0), (1000, 8960, 1536, 1), (1000, 1536, 8960, 2),
                                       (777, 1536, 1536, 3), (777, 1536, 1536, 4), (9450, 5120, 5120, 0), (512, 13824, 5120, 1)])
def test_linear_matches_reference(M, N, K, epi):
    from fastvideo_b200 import ops
    torch.manual_seed(M + N + K + epi)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    resid = torch.randn(M, N, device="cuda").bfloat16() if epi >= 2 else None
    gate = torch.randn(N, device="cuda") if epi in (2, 3) else None
    out = ops.linear(x, w, b, epi, resid, gate)
    ref32, ref_rounded = ref_linear(x, w, b, epi, resid, gate)
    if epi == 2:  # fp32 output: only the bf16 rounding of y separates us from the un-rounded formula
        assert rel_l2(out, ref_rounded) < 1e-3
    else:
        assert_bf16_parity(out, ref32, ref_rounded, name=f"linear epi{epi}")
        # and we reproduce the reference's rounding points almost everywhere
        assert (out.float() != ref_rounded.float()).float().mean().item() < 0.02


def test_linear_strided_rows_and_no_bias():
    from fastvideo_b200 import ops
    torch.manual_seed(3)
    big = torch.randn(300, 3 * 256, device="cuda").bfloat16()
    x = big[:, 256:512]  # a column slice of a fused buffer: row stride 768
    w = (torch.randn(128, 256, device="cuda") / 16).bfloat16()
    out = ops.linear(x, w)
    ref = x.float() @ w.float().t()
    assert_bf16_parity(out, ref, name="strided")


def test_gemm_batched_div():
    from fastvideo_b200 import ops
    torch.manual_seed(4)
    a = torch.randn(6, 200, 128, device="cuda").bfloat16()
    b = torch.randn(6, 136, 128, device="cuda").bfloat16()
    out = ops.gemm_batched(a, b, div=128 ** 0.5)
    ref = (torch.matmul(a.float(), b.float().transpose(1, 2)).bfloat16().float() / (128 ** 0.5)).bfloat16()
    assert (out.float() != ref.float()).float().mean().item() < 0.01
    assert rel_l2(out, ref) < 1e-3
