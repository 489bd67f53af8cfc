"""GPU check of the wgmma GEMM against torch."""
import sys, time, json
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import ops

def ref(x, w, b, epi, resid, gate):
    acc = x.float() @ w.float().t()
    if b is not None: acc = acc + b.float()
    y = acc.bfloat16()
    if epi == 0: return y
    if epi == 1: return torch.nn.functional.gelu(y.float(), approximate="tanh").bfloat16()
    if epi == 2: return resid.float() + y.float() * gate
    if epi == 3: return (resid.float() + y.float() * gate).bfloat16()
    if epi == 4: return (resid.float() + y.float()).bfloat16()

def relerr(a, b):
    a = a.float(); b = b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item(), (a - b).abs().max().item()

def main():
    torch.manual_seed(0)
    dev = "cuda"
    cases = [(128, 256, 64, 0), (128, 256, 256, 0), (256, 512, 512, 0), (1000, 1536, 1536, 0), (4096, 5120, 5120, 0),
             (333, 128, 192, 0), (200, 64, 512, 0), (1000, 8960, 1536, 1), (1000, 1536, 8960, 2), (777, 1536, 1536, 3),
             (777, 1536, 1536, 4), (75600 // 8, 5120, 5120, 0)]
    res = []
    for (M, N, K, epi) in cases:
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        w = (torch.randn(N, K, device=dev) / K ** 0.5).bfloat16()
        b = torch.randn(N, device=dev).bfloat16()
        resid = torch.randn(M, N, device=dev).bfloat16() if epi >= 2 else None
        gate = torch.randn(N, device=dev) if epi in (2, 3) else None
        out = ops.linear(x, w, b, epi, resid, gate)
        torch.cuda.synchronize()
        r = ref(x, w, b, epi, resid, gate)
        rel, mx = relerr(out, r)
        nz = (out.float() != r.float()).float().mean().item()
        print(f"gemm M={M} N={N} K={K} epi={epi}: rel={rel:.3e} maxabs={mx:.3e} mismatch_frac={nz:.4f}", flush=True)
        res.append(dict(M=M, N=N, K=K, epi=epi, rel=rel, maxabs=mx, mismatch=nz))
    # timing at the flagship shapes
    for (M, N, K, epi) in [(75600, 5120, 5120, 0), (75600, 13824, 5120, 1), (75600, 5120, 13824, 3), (75600, 15360, 5120, 0),
                           (32760, 1536, 1536, 0), (32760, 8960, 1536, 1)]:
        x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        w = (torch.randn(N, K, device=dev) / K ** 0.5).bfloat16()
        b = torch.randn(N, device=dev).bfloat16()
        resid = torch.randn(M, N, device=dev).bfloat16() if epi >= 2 else None
        gate = torch.randn(N, device=dev) if epi in (2, 3) else None
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        for _ in range(3): ops.linear(x, w, b, epi, resid, gate, out=out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize(); e0.record()
        for _ in range(10): ops.linear(x, w, b, epi, resid, gate, out=out)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        tf = 2 * M * N * K / ms / 1e9
        for _ in range(3): torch.nn.functional.linear(x, w, b)
        torch.cuda.synchronize(); e0.record()
        for _ in range(10): torch.nn.functional.linear(x, w, b)
        e1.record(); torch.cuda.synchronize()
        ms_t = e0.elapsed_time(e1) / 10
        print(f"time M={M} N={N} K={K} epi={epi}: {ms:.3f} ms = {tf:.0f} TFLOP/s | cuBLAS F.linear {ms_t:.3f} ms = {2*M*N*K/ms_t/1e9:.0f} TFLOP/s", flush=True)
        res.append(dict(M=M, N=N, K=K, epi=epi, ms=ms, tflops=tf, cublas_ms=ms_t))
    json.dump(res, open("tool_out/gemm_check.json", "w"), indent=1)

if __name__ == "__main__":
    main()
