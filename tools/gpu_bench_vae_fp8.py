"""Wan VAE decode, bf16 vs WanVAEConfig(fp8_convs=True), on one GPU in one call:
  * the card's name and power limit;
  * whole decodes at 480p x 81 frames (latent 21 x 60 x 104) and 720p x 81 frames (21 x 90 x 160), the two decoders
    alternated, median ms, output voxels/s and TFLOP/s on the 8.44 MFLOP/voxel model (SURVEY.md section 8d);
  * kernel time of each residual-block convolution shape at its real resolution, bf16 (fvb_conv3d_cl) vs FP8
    (fvb_conv3d_cl_fp8), CUDA events over repeated launches;
  * the FP8 decode's distance from the bf16 decode (relative L2, PSNR over the [-1, 1] range).
Random-init decoder at the real widths (base_dim 96). Prints the result as JSON and writes it to tool_out/vae_fp8_bench.json.

    python tools/gpu_bench_vae_fp8.py [--reps 3] [--sizes 480p,720p]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastvideo_b200 import ops, wan_vae  # noqa: E402

MFLOP_PER_VOXEL = 8.44
SIZES = {"480p": (21, 60, 104), "720p": (21, 90, 160)}


def rand_sd(seed=0, base=96, mult=(1, 2, 4, 4), nrb=2, tds=(False, True, True), dev="cuda"):
    """Real-width decoder weights: fan-in scaled convolutions, gamma ~ 1 + 0.2 N(0, 1), small biases."""
    g = torch.Generator(device=dev).manual_seed(seed)
    dims = [base * u for u in [mult[-1]] + list(mult[::-1])]
    sd = {}

    def rn(*shape):
        return torch.randn(*shape, generator=g, device=dev)

    def conv(name, co, ci, k):
        sd[name + ".weight"] = (rn(co, ci, *k) / (ci * k[0] * k[1] * k[2]) ** 0.5).bfloat16()
        sd[name + ".bias"] = (0.02 * rn(co)).bfloat16()

    def res(p, ci, co):
        sd[p + "norm1.gamma"] = 1 + 0.2 * rn(ci, 1, 1, 1)
        sd[p + "norm2.gamma"] = 1 + 0.2 * rn(co, 1, 1, 1)
        conv(p + "conv1", co, ci, (3, 3, 3))
        conv(p + "conv2", co, co, (3, 3, 3))
        if ci != co:
            conv(p + "conv_shortcut", co, ci, (1, 1, 1))

    conv("post_quant_conv", 16, 16, (1, 1, 1))
    conv("decoder.conv_in", dims[0], 16, (3, 3, 3))
    res("decoder.mid_block.resnets.0.", dims[0], dims[0])
    res("decoder.mid_block.resnets.1.", dims[0], dims[0])
    sd["decoder.mid_block.attentions.0.norm.gamma"] = 1 + 0.2 * rn(dims[0], 1, 1)
    for n, co in (("to_qkv", 3 * dims[0]), ("proj", dims[0])):
        sd[f"decoder.mid_block.attentions.0.{n}.weight"] = (rn(co, dims[0], 1, 1) / dims[0] ** 0.5).bfloat16()
        sd[f"decoder.mid_block.attentions.0.{n}.bias"] = torch.zeros(co, device=dev).bfloat16()
    t_up = list(tds)[::-1]
    for i, (ci, co) in enumerate(zip(dims[:-1], dims[1:])):
        if i > 0:
            ci = ci // 2
        cur = ci
        for j in range(nrb + 1):
            res(f"decoder.up_blocks.{i}.resnets.{j}.", cur, co)
            cur = co
        if i != len(mult) - 1:
            p = f"decoder.up_blocks.{i}.upsamplers.0."
            sd[p + "resample.1.weight"] = (rn(co // 2, co, 3, 3) / (9 * co) ** 0.5).bfloat16()
            sd[p + "resample.1.bias"] = torch.zeros(co // 2, device=dev).bfloat16()
            if t_up[i]:
                conv(p + "time_conv", 2 * co, co, (3, 1, 1))
    sd["decoder.norm_out.gamma"] = 1 + 0.2 * rn(dims[-1], 1, 1, 1)
    conv("decoder.conv_out", 3, dims[-1], (3, 3, 3))
    return sd


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired) as e:
        q = f"unavailable ({type(e).__name__})"
    return {"name": name, "power_limit_and_max_sm_clock": q}


def time_ms(fn, iters):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return sorted(a.elapsed_time(b) for a, b in ev)[iters // 2]


def decode_bench(decs, size, reps):
    T, h, w = SIZES[size]
    z = torch.randn(1, 16, T, h, w, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1)).bfloat16()
    outs, times = {}, {k: [] for k in decs}
    for k, d in decs.items():  # warm-up (module loads, buffer allocation)
        outs[k] = d.decode(z)
    torch.cuda.synchronize()
    for _ in range(reps):
        for k, d in decs.items():  # alternated
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            outs[k] = d.decode(z)
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    vox = outs["bf16"].shape[2] * outs["bf16"].shape[3] * outs["bf16"].shape[4]
    res = {"latent": [T, h, w], "out": list(outs["bf16"].shape)}
    for k in decs:
        ms = sorted(times[k])[len(times[k]) // 2]
        res[k] = {"ms": round(ms, 1), "ms_all": [round(t, 1) for t in times[k]], "voxels_per_s": vox / ms * 1e3,
                  "tflops_model": vox * MFLOP_PER_VOXEL * 1e6 / ms / 1e9}
    res["fp8_speedup"] = res["bf16"]["ms"] / res["fp8"]["ms"]
    a, b = outs["fp8"].float(), outs["bf16"].float()
    mse = float(((a - b) ** 2).mean())
    res["fp8_vs_bf16"] = {"rel_l2": float((a - b).norm() / b.norm()), "psnr_db": 10 * math.log10(4.0 / max(mse, 1e-30))}
    del outs
    torch.cuda.empty_cache()
    return res


def conv_bench(iters):
    """Every residual-block conv shape at the 480p resolution it runs at (per latent frame: 1 / 2 / 4 / 4 frames)."""
    shapes = [("mid+up0 384->384", 384, 384, 60, 104, 1), ("up1.0 conv1 192->384", 192, 384, 120, 208, 2),
              ("up1 384->384", 384, 384, 120, 208, 2), ("up2 192->192", 192, 192, 240, 416, 4), ("up3 96->96", 96, 96, 480, 832, 4)]
    out = []
    g = torch.Generator(device="cuda").manual_seed(2)
    for name, ci, co, H, W, T in shapes:
        x = torch.randn(2 + T, H, W, ci, device="cuda", generator=g)
        xb = x.bfloat16()
        bound = float(x.abs().max())
        xq = (x * (448.0 / bound)).clamp(-448, 448).to(torch.float8_e4m3fn)
        w = (torch.randn(co, ci, 3, 3, 3, device="cuda", generator=g) / (27 * ci) ** 0.5).bfloat16()
        b = torch.zeros(co, device="cuda").bfloat16()
        wp, cp, k = ops.pack_conv_weight(w)
        wq, ws, cp8, _ = ops.pack_conv_weight_fp8(w)
        xs = ops.e4m3_x_scale(bound)
        f_b = lambda: ops.conv3d_cl(xb, wp, cp, k, b, T_out=T, t_off=2)
        f_8 = lambda: ops.conv3d_cl_fp8(xq, wq, ws, cp8, k, xs, b, T_out=T, t_off=2)
        for f in (f_b, f_8):
            f()
        torch.cuda.synchronize()
        tb, t8 = [], []
        for _ in range(3):  # alternated
            tb.append(time_ms(f_b, iters))
            t8.append(time_ms(f_8, iters))
        mb, m8 = sorted(tb)[1], sorted(t8)[1]
        flop = 2.0 * T * H * W * co * ci * 27
        out.append({"shape": name, "T": T, "H": H, "W": W, "bf16_ms": round(mb, 3), "fp8_ms": round(m8, 3),
                    "bf16_tflops": flop / mb / 1e9, "fp8_tflops": flop / m8 / 1e9, "speedup": mb / m8})
        del x, xb, xq
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="480p,720p")
    ap.add_argument("--conv-iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = {"card": card()}
    res["convs_480p"] = conv_bench(a.conv_iters)
    print(json.dumps(res["convs_480p"]), flush=True)
    sd = rand_sd()
    decs = {"bf16": wan_vae.WanVAEDecoder(wan_vae.WanVAEConfig(), sd),
            "fp8": wan_vae.WanVAEDecoder(wan_vae.WanVAEConfig(fp8_convs=True), sd)}
    for s in a.sizes.split(","):
        res["decode_" + s] = decode_bench(decs, s, a.reps)
        print(json.dumps({s: res["decode_" + s]}), flush=True)
    res["card_after"] = card()
    os.makedirs("tool_out", exist_ok=True)
    with open(os.path.join("tool_out", "vae_fp8_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
