"""Wan VAE decode on libfvb200: AutoencoderKLWan.decode's feature-cache loop (fastvideo/models/vaes/wanvae.py:1189-1216)
over WanDecoder3d (wanvae.py:857-993), with every convolution an implicit-GEMM tcgen05 kernel on channels-last frames.

Structure mirrored from the reference (parameter names identical, so a reference state_dict loads unchanged):
  post_quant_conv (1x1x1)                                     wanvae.py:1193
  per latent frame:  conv_in -> mid_block(res, attn, res) -> up_blocks -> norm_out/SiLU -> conv_out   wanvae.py:950-993
  WanResidualBlock: shortcut, RMS-norm+SiLU, causal conv (cached), RMS-norm+SiLU, causal conv, + shortcut   wanvae.py:383-462
  WanResample upsample3d / upsample2d incl. the "Rep" first-chunk rule of the time conv             wanvae.py:303-356
  WanAttentionBlock: per-frame single-head attention over H*W                                        wanvae.py:465-507
The causal feature cache is the reference's: each causal conv remembers its last two INPUT frames; a conv call sees
[cached frames | new frames] and frames before the start of the stream are zeros (done by TMA out-of-bounds fill,
never materialised). Numerics follow the reference under bf16 autocast (configs/pipelines/wan.py:59): convolutions
read/write bf16, norms/SiLU/softmax compute in fp32.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass

import torch

from . import ops


@dataclass
class WanVAEConfig:
    """Decoder-side fields of fastvideo/configs/models/vaes/wanvae.py:9-82."""
    base_dim: int = 96
    z_dim: int = 16
    dim_mult: tuple = (1, 2, 4, 4)
    num_res_blocks: int = 2
    temperal_downsample: tuple = (False, True, True)
    out_channels: int = 3
    # Decoder only: conv1 / conv2 of every residual block on e4m3 operands (fvb_conv3d_cl_fp8) with a static activation
    # scale from the producing norm's gamma. Changes the output visibly; bf16 is the default.
    fp8_convs: bool = False


# fused consumer-norm epilogue (fvb_conv3d_cl_norm); FVB_VAE_FUSE_NORM=0/1 overrides (A/B measurements)
FUSE_NORM = os.environ.get("FVB_VAE_FUSE_NORM", "1") == "1"  # saves a read and a write of the activation per norm


class _Conv:
    """One WanCausalConv3d / Conv2d: packed weights + the two-frame input cache.

    The feature cache of a causal convolution (its last two INPUT frames, wanvae.py:160-207) is the head of a persistent
    input buffer [2 + Tn, H, W, Cin]: producers write the new frames straight behind the cached ones (`in_view`), the kernel
    reads the contiguous slice [cached | new], and afterwards the last two frames move to the head -- instead of a
    torch.cat of cache and input plus a clone per call (5 % of the decode in round 1).

    fp8_bound (FP8 residual-block convolution): the static bound of the norm that produces this convolution's input. The
    weights are then e4m3 with one scale per output channel (no bf16 copy kept), the input buffer and cache are e4m3, every
    producer writes e4m3 against that bound (`in_bound`), and the kernel reads it back with x_scale = bound / 448."""
    dtype = torch.bfloat16

    def __init__(self, sd, name, fp8_bound=None):
        w = sd[name + ".weight"]
        self.fp8 = fp8_bound is not None
        self.in_bound = fp8_bound
        if self.fp8:
            self.w, self.w_scale, self.cin_pad, self.k = ops.pack_conv_weight_fp8(w)
            self.x_scale = ops.e4m3_x_scale(fp8_bound)
            self.dtype = torch.float8_e4m3fn
        else:
            self.w, self.cin_pad, self.k = ops.pack_conv_weight(w)
        self.bias = sd[name + ".bias"].to(torch.bfloat16).contiguous()
        self.cin, self.cout = w.shape[1], w.shape[0]
        self.buf = None   # [2 + Tn, H, W, Cin]; frames [2 - n_c, 2) are the cache
        self.n_c = 0
        self.stateless = False  # cache-less decode (AutoencoderKLWan._decode): zero history, nothing remembered

    def reset(self):
        self.n_c = 0

    @property
    def cache(self):
        return None if self.n_c == 0 or self.buf is None else self.buf[2 - self.n_c:2]

    def in_view(self, Tn, H, W, device):
        """Where a producer should write this convolution's next Tn input frames (None: no persistent buffer applies)."""
        if self.k[0] != 3 or self.stateless:
            return None
        b = self.buf
        if b is None or tuple(b.shape[1:3]) != (H, W) or b.shape[0] < 2 + Tn or b.device != torch.device(device):
            nb = torch.empty((2 + Tn, H, W, self.cin), dtype=self.dtype, device=device)
            if b is not None and self.n_c and tuple(b.shape[1:3]) == (H, W):
                nb[2 - self.n_c:2] = b[2 - self.n_c:2]
            else:
                self.n_c = 0
            self.buf = b = nb
        return b[2:2 + Tn]

    def __call__(self, x, resid=None, use_cache=True, interleave=False, norm=None, want_raw=True):
        """x: [Tn, H, W, Cin] new frames. Causal in time when kt == 3. norm = (gamma, silu[, dest_fn[, bound]]) asks for the
        CONSUMER's RMS-norm (+ SiLU) of the output as well: the result is then (raw or None, normed) -- fused into the
        convolution's epilogue when one tile holds a whole channel row (Cout <= 192), else a separate row pass;
        dest_fn(T, H, W, device) may name the buffer the normalised frames go to (the consumer's in_view); a bound that is not
        None makes the normalised frames e4m3 (the consumer is an FP8 convolution)."""
        kt = self.k[0]
        Tn, H, W, _ = x.shape
        if (x.dtype == torch.float8_e4m3fn) != self.fp8:
            raise ops.FvbError(f"{'e4m3' if self.fp8 else 'bf16'} convolution given {x.dtype} input")
        if kt == 1 or not use_cache or self.stateless:
            # stateless: the frames before this call's first one are zeros (TMA out-of-bounds fill) = F.pad(x, 2 * pt)
            buf, n_c = x, 0
        else:
            view = self.in_view(Tn, H, W, x.device)
            if x.data_ptr() != view.data_ptr():
                view.copy_(x)  # the producer did not write in place
            n_c = self.n_c
            buf = self.buf[2 - n_c:2 + Tn]
        fuse = norm is not None and not interleave and 16 < self.cout <= ops.CONV_NORM_MAX_COUT and FUSE_NORM
        dest = norm[2](Tn, H, W, x.device) if norm is not None and len(norm) > 2 and norm[2] is not None else None
        qb = norm[3] if norm is not None and len(norm) > 3 else None
        if fuse and self.fp8:
            out = ops.conv3d_cl_fp8_norm(buf, self.w, self.w_scale, self.cin_pad, self.k, self.x_scale, norm[0], self.bias, resid,
                                         want_raw=want_raw, silu=norm[1], T_out=Tn, t_off=n_c, norm_out=dest, norm_bound=qb)
        elif fuse and qb is not None:
            out = ops.conv3d_cl_norm_e4m3(buf, self.w, self.cin_pad, self.k, norm[0], qb, self.bias, resid, want_raw=want_raw,
                                          silu=norm[1], T_out=Tn, t_off=n_c, norm_out=dest)
        elif fuse:
            out = ops.conv3d_cl_norm(buf, self.w, self.cin_pad, self.k, norm[0], self.bias, resid, want_raw=want_raw,
                                     silu=norm[1], T_out=Tn, t_off=n_c, norm_out=dest)
        else:
            if self.fp8:
                out = ops.conv3d_cl_fp8(buf, self.w, self.w_scale, self.cin_pad, self.k, self.x_scale, self.bias, resid,
                                        T_out=Tn, t_off=n_c)
            else:
                out = ops.conv3d_cl(buf, self.w, self.cin_pad, self.k, self.bias, resid, T_out=Tn, t_off=n_c,
                                    interleave_c=self.cout // 2 if interleave else 0)
            if norm is not None:
                out = (out, _norm(out, norm, out=dest))
        if kt == 3 and use_cache and not self.stateless:  # the stream's last two frames become the head of the buffer
            keep = min(2, n_c + Tn)
            src = self.buf[2 + Tn - keep:2 + Tn]
            self.buf[2 - keep:2] = src.clone() if Tn < 2 else src  # Tn == 1: source and destination overlap
            self.n_c = keep
        return out


def _norm(x, norm, out=None):
    """The consumer's RMS-norm (+ SiLU) as a separate row pass: norm = (gamma, silu[, dest_fn[, bound]]); e4m3 against
    the bound when there is one."""
    bound = norm[3] if len(norm) > 3 else None
    if bound is not None:
        return ops.rmsnorm_silu_cl_e4m3(x, norm[0], bound, silu=norm[1], out=out)
    return ops.rmsnorm_silu_cl(x, norm[0], silu=norm[1], out=out)


class _Linear1x1:
    """1x1(x1) convolution == a linear over channels of channels-last pixels."""

    def __init__(self, sd, name):
        w = sd[name + ".weight"]
        self.w = w.reshape(w.shape[0], w.shape[1]).to(torch.bfloat16).contiguous()
        self.b = sd[name + ".bias"].to(torch.bfloat16).contiguous()
        # pad K to a multiple of 8 for 16-byte rows (z_dim = 16 is already fine)
        assert self.w.shape[1] % 8 == 0

    def __call__(self, x):
        shp = x.shape
        return ops.linear(x.reshape(-1, shp[-1]), self.w, self.b).view(*shp[:-1], self.w.shape[0])


class _ResBlock:
    def __init__(self, sd, p, in_dim, out_dim, fp8=False):
        self.g1 = sd[p + "norm1.gamma"].float().reshape(-1).contiguous()
        self.g2 = sd[p + "norm2.gamma"].float().reshape(-1).contiguous()
        b1, b2 = (ops.rms_norm_e4m3_bound(self.g1), ops.rms_norm_e4m3_bound(self.g2)) if fp8 else (None, None)
        self.conv1, self.conv2 = _Conv(sd, p + "conv1", b1), _Conv(sd, p + "conv2", b2)
        self.shortcut = _Linear1x1(sd, p + "conv_shortcut") if in_dim != out_dim else None

    def convs(self):
        return [self.conv1, self.conv2]

    def first_norm(self):
        return (self.g1, True, self.conv1.in_view, self.conv1.in_bound)

    def __call__(self, x, xn=None, next_norm=None):
        """xn: norm1+SiLU of x if the producer already made it; next_norm: (gamma, silu[, dest_fn]) of the consumer of this
        block's output. Returns (out, normed out or None)."""
        Tn, H, W, _ = x.shape
        h = self.shortcut(x) if self.shortcut is not None else x
        if xn is None:
            xn = _norm(x, self.first_norm(), out=self.conv1.in_view(Tn, H, W, x.device))
        # conv1's output is only ever read through norm2 + SiLU, and only by conv2: written straight into conv2's input buffer
        _, yn = self.conv1(xn, norm=(self.g2, True, self.conv2.in_view, self.conv2.in_bound), want_raw=False)
        if next_norm is None:
            return self.conv2(yn, resid=h), None
        return self.conv2(yn, resid=h, norm=next_norm)


class _Attention:
    def __init__(self, sd, p):
        self.g = sd[p + "norm.gamma"].float().reshape(-1).contiguous()
        self.qkv, self.proj = _Linear1x1(sd, p + "to_qkv"), _Linear1x1(sd, p + "proj")

    def first_norm(self):
        return (self.g, False, None)

    def __call__(self, x, xn=None, next_norm=None):
        T, H, W, C = x.shape
        outs = []
        for t in range(T):  # attention is per frame (wanvae.py:480-497)
            xt = x[t].reshape(H * W, C)
            n = xn[t].reshape(H * W, C) if xn is not None else ops.rmsnorm_silu_cl(xt, self.g, silu=False)
            qkv = self.qkv(n)  # [HW, 3C]
            q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
            s = ops.gemm_f32out(q, k, 1.0 / math.sqrt(C))
            pr = ops.softmax_rows_f32(s)
            o = ops.linear(pr, ops.transpose_bf16(v))  # P @ V
            y = ops.linear(o, self.proj.w, self.proj.b, ops.EPI_RESID_BF16, resid=xt)
            outs.append(y.view(1, H, W, C))
        y = torch.cat(outs, 0) if T > 1 else outs[0]
        return y, (_norm(y, next_norm) if next_norm is not None else None)


def _run_chain(mods, x, final_norm=None, xn=None):
    """Runs a list of blocks, asking every producer for the normalised tensor its consumer starts with (blocks that begin
    with an RMS-norm expose first_norm()), so the norm rides on the producing convolution's epilogue."""
    for i, m in enumerate(mods):
        nxt = mods[i + 1] if i + 1 < len(mods) else None
        next_norm = nxt.first_norm() if hasattr(nxt, "first_norm") else (final_norm if nxt is None else None)
        if hasattr(m, "first_norm"):
            x, xn = m(x, xn, next_norm)
        else:
            x, xn = m(x, next_norm)
    return x, xn


class _Upsample:
    def __init__(self, sd, p, dim, mode):
        self.mode = mode
        self.conv = _Conv(sd, p + "resample.1")  # Conv2d(dim, dim // 2, 3, padding=1)
        self.time_conv = _Conv(sd, p + "time_conv") if mode == "upsample3d" else None
        self.first = True  # the reference's "Rep" sentinel (wanvae.py:327-340)
        self.stateless = False

    def reset(self):
        self.first = True
        if self.time_conv is not None:
            self.time_conv.reset()

    def convs(self):
        return [self.conv] + ([self.time_conv] if self.time_conv is not None else [])

    def __call__(self, x, next_norm=None):
        if self.mode == "upsample3d":
            if self.stateless:
                x = self.time_conv(x, interleave=True)  # no feature cache: every frame is doubled (wanvae.py:341-345)
            elif self.first:
                self.first = False  # first chunk: no temporal upsampling, nothing cached
            else:
                x = self.time_conv(x, interleave=True)  # [2T, H, W, C]
        x = ops.upsample2x_cl(x)
        if next_norm is None:
            return self.conv(x, use_cache=False), None
        return self.conv(x, use_cache=False, norm=next_norm)


class _Downsample:
    """WanResample downsample2d / downsample3d (wanvae.py:291-296, 357-380). The stride-2 3x3 convolution behind
    ZeroPad2d((0, 1, 0, 1)) equals the odd-index samples of the "same"-padded stride-1 convolution, so it runs on the same
    implicit-GEMM kernel (3 of the encoder's ~25 convolutions pay 4x for that; a strided TMA box is the obvious follow-up).
    downsample3d: the first call passes its (single) frame through and remembers it; later calls run the (3, 1, 1) stride-2
    time convolution over [remembered last frame | new frames] -- again every output of the stride-1 form, every second kept."""

    def __init__(self, sd, p, mode):
        self.mode = mode
        self.conv = _Conv(sd, p + "resample.1")
        self.time_conv = _Conv(sd, p + "time_conv") if mode == "downsample3d" else None
        self.prev = None

    def reset(self):
        self.prev = None

    def convs(self):
        return [self.conv] + ([self.time_conv] if self.time_conv is not None else [])

    def __call__(self, x, next_norm=None):
        y = self._down(x)
        return y, (ops.rmsnorm_silu_cl(y, next_norm[0], silu=next_norm[1]) if next_norm is not None else None)

    def _down(self, x):
        y = self.conv(x, use_cache=False)[:, 1::2, 1::2].contiguous()
        if self.mode != "downsample3d":
            return y
        if self.prev is None:
            self.prev = y[-1:].clone()
            return y
        tc = self.time_conv
        buf = torch.cat([self.prev, y], 0)
        self.prev = y[-1:].clone()
        out = ops.conv3d_cl(buf, tc.w, tc.cin_pad, tc.k, tc.bias, None, T_out=y.shape[0] - 1, t_off=2)
        return out[::2].contiguous()


class WanVAEEncoder:
    """AutoencoderKLWan.encode with the feature cache on (wanvae.py:1128-1151) over WanEncoder3d (wanvae.py:586-712): the
    first frame alone, then 4-frame chunks, every causal convolution remembering its last two input frames. Same kernels
    as the decoder (implicit-GEMM convolutions on channels-last frames, fused RMS-norm + SiLU rows, tcgen05 GEMMs for the
    1x1 convolutions and the mid-block attention); parameter names are the reference's."""

    def __init__(self, cfg: WanVAEConfig, state_dict: dict):
        if cfg.fp8_convs:
            raise ops.FvbError("WanVAEConfig.fp8_convs applies to the decoder only; the encoder has no FP8 path")
        sd = dict(state_dict)
        self.cfg = cfg
        dim, mult = cfg.base_dim, list(cfg.dim_mult)
        dims = [dim * u for u in [1] + mult]
        e = "encoder."
        w_in = sd[e + "conv_in.weight"]
        w8 = w_in.new_zeros((w_in.shape[0], 8) + tuple(w_in.shape[2:]))  # RGB padded to 8 channels: 16-byte pixel rows for TMA
        w8[:, :w_in.shape[1]] = w_in
        sd[e + "conv_in.weight"] = w8
        self.in_channels = w_in.shape[1]
        self.conv_in = _Conv(sd, e + "conv_in")
        self.down = []
        n = 0
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            for _ in range(cfg.num_res_blocks):
                self.down.append(_ResBlock(sd, f"{e}down_blocks.{n}.", in_dim, out_dim))
                in_dim = out_dim
                n += 1
            if i != len(mult) - 1:
                self.down.append(_Downsample(sd, f"{e}down_blocks.{n}.", "downsample3d" if cfg.temperal_downsample[i] else "downsample2d"))
                n += 1
        self.mid = [_ResBlock(sd, e + "mid_block.resnets.0.", dims[-1], dims[-1]), _Attention(sd, e + "mid_block.attentions.0."),
                    _ResBlock(sd, e + "mid_block.resnets.1.", dims[-1], dims[-1])]
        self.g_out = sd[e + "norm_out.gamma"].float().reshape(-1).contiguous()
        self.conv_out = _Conv(sd, e + "conv_out")
        self.quant = _Linear1x1(sd, "quant_conv")

    def clear_cache(self):
        for m in [self.conv_in, self.conv_out] + self.down + self.mid:
            if isinstance(m, _Conv):
                m.reset()
            elif isinstance(m, _ResBlock):
                m.conv1.reset(), m.conv2.reset()
            elif isinstance(m, _Downsample):
                m.reset()

    def encode_chunk(self, x_cl: torch.Tensor) -> torch.Tensor:
        mods = self.down + self.mid
        x, xn = self.conv_in(x_cl, norm=mods[0].first_norm())
        _, xn = _run_chain(mods, x, final_norm=(self.g_out, True, self.conv_out.in_view), xn=xn)
        return self.conv_out(xn)

    @torch.no_grad()
    def encode(self, x: torch.Tensor):
        """x: [1, 3, 1 + 4k, H, W] in [-1, 1] -> (mean, logvar), each fp32 [1, z_dim, 1 + k, H/8, W/8]; logvar clamped to
        [-30, 20] as DiagonalGaussianDistribution does (the `.mode()` of the distribution is `mean`)."""
        if not x.is_cuda:
            raise ops.FvbError("WanVAEEncoder.encode needs CUDA tensors (there is no CPU fallback)")
        assert x.shape[0] == 1 and x.shape[1] == self.in_channels
        self.clear_cache()
        T = x.shape[2]
        xc = torch.zeros((T, x.shape[3], x.shape[4], 8), dtype=torch.bfloat16, device=x.device)
        xc[..., :self.in_channels] = x[0].permute(1, 2, 3, 0)
        outs = [self.encode_chunk(xc[:1])]
        for i in range(1, 1 + (T - 1) // 4):  # wanvae.py:1137-1144
            outs.append(self.encode_chunk(xc[1 + 4 * (i - 1):1 + 4 * i]))
        self.clear_cache()
        m = self.quant(torch.cat(outs, 0)).float().permute(3, 0, 1, 2).unsqueeze(0)  # [1, 2 z, T', h, w]
        z = self.cfg.z_dim
        return m[:, :z].contiguous(), m[:, z:].clamp(-30.0, 20.0).contiguous()


class WanVAEDecoder:
    def __init__(self, cfg: WanVAEConfig, state_dict: dict):
        sd = state_dict
        self.cfg = cfg
        dim, mult = cfg.base_dim, list(cfg.dim_mult)
        dims = [dim * u for u in [mult[-1]] + mult[::-1]]
        temperal_upsample = list(cfg.temperal_downsample)[::-1]
        self.post_quant = _Linear1x1(sd, "post_quant_conv")
        d = "decoder."
        self.conv_in = _Conv(sd, d + "conv_in")
        fp8 = cfg.fp8_convs
        self.mid = [_ResBlock(sd, d + "mid_block.resnets.0.", dims[0], dims[0], fp8), _Attention(sd, d + "mid_block.attentions.0."),
                    _ResBlock(sd, d + "mid_block.resnets.1.", dims[0], dims[0], fp8)]
        self.ups = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            if i > 0:
                in_dim = in_dim // 2
            blocks = []
            cur = in_dim
            for j in range(cfg.num_res_blocks + 1):
                blocks.append(_ResBlock(sd, f"{d}up_blocks.{i}.resnets.{j}.", cur, out_dim, fp8))
                cur = out_dim
            if i != len(mult) - 1:
                mode = "upsample3d" if temperal_upsample[i] else "upsample2d"
                blocks.append(_Upsample(sd, f"{d}up_blocks.{i}.upsamplers.0.", out_dim, mode))
            self.ups.append(blocks)
        self.g_out = sd[d + "norm_out.gamma"].float().reshape(-1).contiguous()
        self.conv_out = _Conv(sd, d + "conv_out")

    def _all(self):
        for m in [self.conv_in, self.conv_out] + self.mid + [b for u in self.ups for b in u]:
            yield m

    def clear_cache(self):
        for m in self._all():
            if isinstance(m, _Conv):
                m.reset()
            elif isinstance(m, _ResBlock):
                m.conv1.reset(), m.conv2.reset()
            elif isinstance(m, _Upsample):
                m.reset()

    def decode_chunk(self, z_cl: torch.Tensor) -> torch.Tensor:
        """z_cl: [Tn, h, w, z_dim] (after post_quant_conv). Returns [Tn', 8h, 8w, 3-padded] bf16 channels-last."""
        mods = self.mid + [b for blocks in self.ups for b in blocks]
        x, xn = self.conv_in(z_cl, norm=mods[0].first_norm())
        _, xn = _run_chain(mods, x, final_norm=(self.g_out, True, self.conv_out.in_view), xn=xn)
        return self.conv_out(xn)

    def _set_stateless(self, on: bool) -> None:
        for m in self._all():
            if isinstance(m, _Conv):
                m.stateless = on
            elif isinstance(m, _ResBlock):
                m.conv1.stateless = m.conv2.stateless = on
            elif isinstance(m, _Upsample):
                m.stateless = on
                if m.time_conv is not None:
                    m.time_conv.stateless = on

    @torch.no_grad()
    def decode_tile(self, z: torch.Tensor) -> torch.Tensor:
        """AutoencoderKLWan._decode (wanvae.py:1218-1226): the decoder WITHOUT the feature cache on a whole latent tile --
        causal convolutions see zeros before the tile's first frame, every temporal upsampler doubles every frame.
        z [1, z_dim, T, h, w] -> bf16 [1, 3, 4T, 8h, 8w] clamped to [-1, 1] (the tiled wrappers drop the first three frames)."""
        if not z.is_cuda:
            raise ops.FvbError("WanVAEDecoder.decode_tile needs CUDA tensors (there is no CPU fallback)")
        assert z.shape[0] == 1
        self.clear_cache()
        self._set_stateless(True)
        try:
            zc = z[0].permute(1, 2, 3, 0).contiguous().to(torch.bfloat16)
            out = self.decode_chunk(self.post_quant(zc))  # [4T, H, W, 3-padded]
        finally:
            self._set_stateless(False)
        return ops.clamp_to_nchw(out, self.cfg.out_channels).to(torch.bfloat16).unsqueeze(0)

    @torch.no_grad()
    def decode_tiled(self, z: torch.Tensor, tiling=None, rank: int = 0, world: int = 1, group=None) -> torch.Tensor:
        """AutoencoderKLWan.decode with use_feature_cache=False (wanvae.py:1189-1247 + ParallelTiledVAE.decode,
        models/vaes/common.py:77-92): spatio-temporal tiles through the cache-less decoder, linear seam blends, tiles dealt to
        the ranks of `group` when world > 1. Wan's wrappers double blend_num_frames for the temporal paths and drop the first
        temporal_compression_ratio - 1 frames of every tiled result. Returns [1, 3, 4(T-1)+1, 8h, 8w]."""
        import dataclasses

        from . import vae_tiling as vt
        cfg = tiling or vt.TilingConfig()
        _, _, num_frames, height, width = z.shape
        min_h, min_w, min_t, _, _, _ = vt._latent_tile_dims(cfg)
        n_out = (num_frames - 1) * cfg.temporal_compression_ratio + 1
        drop = cfg.temporal_compression_ratio - 1
        doubled = dataclasses.replace(cfg, blend_num_frames=cfg.blend_num_frames * 2)
        if cfg.use_tiling and cfg.use_parallel_tiling and world > 1:
            return vt.parallel_tiled_decode(z, self.decode_tile, doubled, rank, world, group)[:, :, drop:][:, :, :n_out]
        if cfg.use_tiling and cfg.use_temporal_tiling and num_frames > min_t:
            # inside the temporal loop `self.spatial_tiled_decode` is Wan's override: it drops the first frames of EVERY
            # spatially tiled temporal tile as well (wanvae.py:1235-1239 called from common.py:358-359)
            wan_spatial = lambda t: vt.spatial_tiled_decode(t, self.decode_tile, doubled)[:, :, drop:]
            return vt.tiled_decode(z, self.decode_tile, doubled, spatial_fn=wan_spatial)[:, :, drop:][:, :, :n_out]
        if cfg.use_tiling and (width > min_w or height > min_h):
            return vt.spatial_tiled_decode(z, self.decode_tile, cfg)[:, :, drop:][:, :, :n_out]
        return self.decode_tile(z)[:, :, :n_out]

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z: [1, z_dim, T, h, w] (already de-normalised latents) -> fp32 [1, 3, 1 + 4(T-1), 8h, 8w] in [-1, 1].
        This is AutoencoderKLWan.decode with use_feature_cache=True, the reference's default for Wan
        (fastvideo/configs/models/vaes/wanvae.py:73; wanvae.py:1189-1216): whole frames, one latent frame at a time, no tiling.
        (The tiled variants of ParallelTiledVAE are only reached with the feature cache off; their host logic lives in
        fastvideo_b200/vae_tiling.py.)"""
        if not z.is_cuda:
            raise ops.FvbError("WanVAEDecoder.decode needs CUDA tensors (there is no CPU fallback)")
        assert z.shape[0] == 1
        self.clear_cache()
        zc = z[0].permute(1, 2, 3, 0).contiguous().to(torch.bfloat16)  # [T, h, w, C]
        x = self.post_quant(zc)
        frames = []
        for i in range(x.shape[0]):  # one latent frame at a time (wanvae.py:1197-1205)
            frames.append(self.decode_chunk(x[i:i + 1].contiguous()))
        out = torch.cat(frames, 0)  # [T', H, W, 3]
        self.clear_cache()
        return ops.clamp_to_nchw(out, self.cfg.out_channels).unsqueeze(0)
