"""CPU: the differentiable bf16 linear has no CPU fallback, with or without grad."""
import pytest
import torch


def test_linear_forward_refuses_cpu_tensors():
    from fastvideo_b200 import ops, plugin
    x = torch.randn(4, 64).bfloat16()
    w = torch.randn(32, 64).bfloat16()
    b = torch.randn(32).bfloat16()
    with pytest.raises(ops.FvbError):
        plugin.linear_forward(x, w, b)
    with torch.no_grad(), pytest.raises(ops.FvbError):
        plugin.linear_forward(x, w, b)
    with pytest.raises(ops.FvbError):
        plugin.linear_forward(x.requires_grad_(True), w.requires_grad_(True), b.requires_grad_(True))


def test_linear_bwd_refuses_cpu_tensors():
    from fastvideo_b200 import ops
    x, w, dy = torch.zeros(8, 64).bfloat16(), torch.zeros(16, 64).bfloat16(), torch.zeros(8, 16).bfloat16()
    with pytest.raises(ops.FvbError):
        ops.linear_bwd(x, w, dy, True, True, True)
