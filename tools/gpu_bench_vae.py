"""Wan VAE decode throughput on H100 (BASELINE.json config #5 geometry: 1080p latent 135x240, 8x spatial / 4x temporal),
random-init decoder at the real widths (base_dim 96). Reports output voxels/s, TFLOP/s against the 8.44 MFLOP/voxel
model and GB/s against the 5.59 KB/voxel unfused-conv traffic model (SURVEY.md section 8d)."""
import json, sys, time
import torch
sys.path.insert(0, ".")
from fastvideo_b200 import wan_vae

def rand_sd(base=96, mult=(1, 2, 4, 4), nrb=2, tds=(False, True, True), dev="cuda"):
    g = torch.Generator(device=dev).manual_seed(0)
    dims = [base * u for u in [mult[-1]] + list(mult[::-1])]
    sd = {}
    def conv(name, co, ci, k):
        fan = ci * k[0] * k[1] * k[2]
        sd[name + ".weight"] = (torch.randn(co, ci, *k, generator=g, device=dev) * (1.0 / fan ** 0.5)).bfloat16()
        sd[name + ".bias"] = torch.zeros(co, device=dev).bfloat16()
    def res(p, ci, co):
        sd[p + "norm1.gamma"] = torch.ones(ci, 1, 1, 1, device=dev); sd[p + "norm2.gamma"] = torch.ones(co, 1, 1, 1, device=dev)
        conv(p + "conv1", co, ci, (3, 3, 3)); conv(p + "conv2", co, co, (3, 3, 3))
        if ci != co: conv(p + "conv_shortcut", co, ci, (1, 1, 1))
    conv("post_quant_conv", 16, 16, (1, 1, 1)); conv("decoder.conv_in", dims[0], 16, (3, 3, 3))
    res("decoder.mid_block.resnets.0.", dims[0], dims[0]); res("decoder.mid_block.resnets.1.", dims[0], dims[0])
    sd["decoder.mid_block.attentions.0.norm.gamma"] = torch.ones(dims[0], 1, 1, device=dev)
    for n, co in (("to_qkv", 3 * dims[0]), ("proj", dims[0])):
        sd[f"decoder.mid_block.attentions.0.{n}.weight"] = (torch.randn(co, dims[0], 1, 1, generator=g, device=dev) / dims[0] ** 0.5).bfloat16()
        sd[f"decoder.mid_block.attentions.0.{n}.bias"] = torch.zeros(co, device=dev).bfloat16()
    t_up = list(tds)[::-1]
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        if i > 0: ci = ci // 2
        cur = ci
        for j in range(nrb + 1):
            res(f"decoder.up_blocks.{i}.resnets.{j}.", cur, co); cur = co
        if i != len(mult) - 1:
            p = f"decoder.up_blocks.{i}.upsamplers.0."
            sd[p + "resample.1.weight"] = (torch.randn(co // 2, co, 3, 3, generator=g, device=dev) / (9 * co) ** 0.5).bfloat16()
            sd[p + "resample.1.bias"] = torch.zeros(co // 2, device=dev).bfloat16()
            if t_up[i]: conv(p + "time_conv", 2 * co, co, (3, 1, 1))
    sd["decoder.norm_out.gamma"] = torch.ones(dims[-1], 1, 1, 1, device=dev)
    conv("decoder.conv_out", 3, dims[-1], (3, 3, 3))
    return sd

def main():
    T = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    h, w = (int(sys.argv[2]), int(sys.argv[3])) if len(sys.argv) > 3 else (135, 240)
    dec = wan_vae.WanVAEDecoder(wan_vae.WanVAEConfig(), rand_sd())
    z = torch.randn(1, 16, T, h, w, device="cuda").bfloat16()
    iters = int(sys.argv[4]) if len(sys.argv) > 4 else 10
    for _ in range(2):
        y = dec.decode(z)
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); y = dec.decode(z); e1.record(); torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    ms = sorted(times)[len(times) // 2]
    vox = y.shape[2] * y.shape[3] * y.shape[4]
    # steady-state per-voxel models are for frames after the first (4 output frames per latent frame)
    res = dict(latent=[T, h, w], out=list(y.shape), iters=iters, ms_all=[round(t, 2) for t in times], ms=ms, voxels_per_s=vox / ms * 1e3, tflops_model=vox * 8.44e6 / ms / 1e9,
               gbs_unfused_model=vox * 5.59e3 / ms / 1e6, finite=bool(torch.isfinite(y).all()), peak_mem_gib=torch.cuda.max_memory_allocated() / 2**30)
    print(json.dumps(res))
    json.dump(res, open(f"tool_out/vae_bench_T{T}.json", "w"), indent=1)

if __name__ == "__main__":
    main()
