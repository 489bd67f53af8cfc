"""CPU: the restatement of the RMSNorm backward (tests/rmsnorm_bwd_ref.py) against fp64 torch autograd of the reference
formula x * rsqrt(mean(x^2) + eps) * w (fastvideo/layers/layernorm.py:73-79 without its bf16 casts)."""
import pytest
import torch

import rmsnorm_bwd_ref


@pytest.mark.parametrize("D,weight", [(64, True), (1536, True), (1536, False)])
def test_restatement_matches_fp64_autograd(D, weight):
    g = torch.Generator().manual_seed(D)
    x = (torch.randn(37, D, generator=g, dtype=torch.float64) * 2).requires_grad_(True)
    w = (1 + 0.3 * torch.randn(D, generator=g, dtype=torch.float64)).requires_grad_(True) if weight else None
    dy = torch.randn(37, D, generator=g, dtype=torch.float64)
    eps = 1e-6
    y = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
    if weight:
        y = y * w
    y.backward(dy)
    dx, dw = rmsnorm_bwd_ref.rmsnorm_bwd(x.detach(), None if w is None else w.detach(), dy, eps)
    assert torch.allclose(dx, x.grad, rtol=1e-12, atol=1e-12)
    if weight:
        assert torch.allclose(dw, w.grad, rtol=1e-12, atol=1e-10)
    else:
        assert dw is None
