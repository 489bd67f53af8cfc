"""Restatement of fvb_rmsnorm_bwd (include/fvb200.h), the backward of n = bf16(bf16(x * r) * w), r = rsqrt(mean(x^2) + eps):
    g = dy * w,  x^ = x * r,  s = sum_c g * x,  dx = r * (g - x^ * (r * s) / D),  dw = sum_m dy * x^.
With bf16_points=True the kernel's roundings are applied (g and x^ in dw to bf16, dx and dw rounded once, fp32 arithmetic);
otherwise the formula is evaluated exactly in the inputs' dtype (fp64 in tests/test_rmsnorm_bwd_cpu.py)."""
import torch


def rmsnorm_bwd(x, w, dy, eps, bf16_points=False):
    """x, dy: [M, D]; w: [D] or None. Returns (dx, dw or None)."""
    if bf16_points:
        x, dy = x.float(), dy.float()
        w = None if w is None else w.float()
    rnd = (lambda t: t.bfloat16().float()) if bf16_points else (lambda t: t)
    D = x.shape[-1]
    r = torch.rsqrt(x.pow(2).sum(-1, keepdim=True) / D + eps)
    g = dy if w is None else rnd(dy * w)
    xh = x * r
    s = (g * x).sum(-1, keepdim=True)
    dx = r * (g - xh * ((r * s) / D))
    dw = None if w is None else (dy * rnd(xh)).sum(0)
    if bf16_points:
        dx = dx.bfloat16()
        dw = None if dw is None else dw.bfloat16()
    return dx, dw
