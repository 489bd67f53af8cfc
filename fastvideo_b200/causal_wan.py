"""Causal (self-forcing) Wan DiT on libfvb200: KV-cache self-attention over a sliding window of latent frames,
per-latent-frame AdaLN modulation.

Mirrors:
  CausalWanSelfAttention.forward            fastvideo/models/dits/causal_wanvideo.py:73-185  (kv_cache branch; RoPE cache policies
                                            "absolute" and "relativistic", fastvideo/models/dits/_relative_rope.py)
  CausalWanTransformerBlock.forward         fastvideo/models/dits/causal_wanvideo.py:265-342
  CausalWanTransformer3DModel._forward_inference   fastvideo/models/dits/causal_wanvideo.py:546-655
  WanT2VCrossAttention.forward (crossattn_cache)   fastvideo/models/dits/wanvideo.py:188-222
Parameter names are the reference's; the pinned dtype flow is bf16 parameters and bf16 temb (module.to(bfloat16)), in
which the reference's `e = scale_shift_table + temb` is bf16 and every modulation / gate op rounds to bf16 -- the
kernels reproduce those rounding points (FVB_EPI_RESID_GATE_BF16R, fvb_layernorm_modulate round_ln = 3).

Implementation differences that do not change results:
  * the fused QKV GEMM writes K and V straight into the cache rows (per-head column-block offsets of
    fvb_linear_bf16_sp), QK-RMSNorm + RoPE then runs in place on the cache rows: no roped_key / v copies;
  * eviction does not move memory. The reference shifts the non-sink part of the cache left by the evicted token
    count (two clone + copy passes over the whole window per layer, causal_wanvideo.py:141-148); here the non-sink
    region is a ring: eviction advances a head index and new rows overwrite the evicted ones. Softmax attention is
    invariant to key order, and keys are stored already roped with absolute positions, so the result is the same
    set of keys and values. (When the attention window is shorter than the cache, which needs order, the
    reference's shift is used instead.)
  * RoPE is evaluated in float64 like the reference does on this path (it passes float64 tables through).
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import torch

from . import ops
from .distributed import out_proj_sp
from .rope import get_rotary_pos_embed
from .wan_dit import (CrossAttnCache, Modulation, TokenLayout, WanBlock, WanDiT, WanDiTConfig, _HeadNormFramesFn,
                      _any_model_tensor_requires_grad, _any_requires_grad, _linear, _require_trainable, _requires_grad,
                      block_body, block_causal_tiles, block_forward_grad, block_tail, refuse_grad, refuse_model_grad)

GLOBAL_ATTN_COMPAT_MAX_LATENT_FRAMES = 21  # causal_wanvideo.py:32


@dataclass
class CausalConfig:
    """arch_config fields of the causal models (fastvideo/configs/models/dits/wanvideo.py: local_attn_size, sink_size,
    num_frames_per_block, rope_cache_policy)."""
    local_attn_size: int = -1
    sink_size: int = 0
    num_frames_per_block: int = 3
    rope_cache_policy: str = "absolute"


class KVCache:
    """One layer's self-attention cache for batch 1: k, v [cache_tokens, H, d] bf16 plus the reference's two counters
    (global_end_index, local_end_index; causal_denoising.py:380-408). Logical token i (the reference's cache index)
    lives at physical row phys(i); the sink prefix is never moved."""

    def __init__(self, cache_tokens: int, heads: int, head_dim: int, device, sink_tokens: int = 0, storage=None):
        if storage is not None:  # (k, v) views into a caller-owned slab (sequence parallel: peer-mapped symmetric memory)
            self.k, self.v = storage
            assert self.k.shape == (cache_tokens, heads, head_dim) and self.v.shape == self.k.shape
        else:
            self.k = torch.zeros((cache_tokens, heads, head_dim), dtype=torch.bfloat16, device=device)
            self.v = torch.zeros_like(self.k)
        self.size = cache_tokens
        self.sink = sink_tokens
        self.head = 0  # ring offset of logical index `sink` inside the non-sink region
        self.global_end_index = 0
        self.local_end_index = 0

    def reset(self):
        self.head = self.global_end_index = self.local_end_index = 0

    # ---- logical <-> physical
    def segments(self, lo: int, hi: int):
        """Physical [start, stop) runs covering logical [lo, hi), in logical order."""
        segs = []
        if lo < self.sink:
            segs.append((lo, min(hi, self.sink)))
            lo = min(hi, self.sink)
        R = self.size - self.sink
        while lo < hi:
            p = self.sink + (self.head + lo - self.sink) % R
            n = min(hi - lo, self.size - p)
            if segs and segs[-1][1] == p:
                segs[-1] = (segs[-1][0], p + n)  # physically adjacent runs merge (sink prefix followed by ring start)
            else:
                segs.append((p, p + n))
            lo += n
        return segs

    def logical(self, t: torch.Tensor, lo: int, hi: int) -> torch.Tensor:
        return torch.cat([t[a:b] for a, b in self.segments(lo, hi)], 0)

    def window_positions(self, k0: int, k1: int) -> torch.Tensor:
        """int32 [k1 - k0]: position inside the attended window of every PHYSICAL row k0..k1 (the reference's window is
        cache[w0:local_end] in logical order, position = logical index - w0). Used by the relativistic RoPE policy, which
        ropes the un-roped cached keys from position 0 on every call; cached per ring state."""
        key = (k0, k1, self.head)
        if getattr(self, "_pos_key", None) != key:
            p = torch.arange(k0, k1, dtype=torch.int64)
            if self.head == 0:
                pos = p - k0
            else:  # ring: the window is the whole cache (advance() guarantees w0 == 0)
                R = self.size - self.sink
                pos = torch.where(p < self.sink, p, self.sink + (p - self.sink - self.head) % R)
            self._pos, self._pos_key = pos.to(torch.int32).to(self.k.device), key
        return self._pos

    def linearize(self, hi: int) -> None:
        """Re-pack logical [sink, hi) at physical [sink, hi) and reset the ring (the reference's layout)."""
        if self.head == 0:
            return
        for t in (self.k, self.v):
            moved = self.logical(t, self.sink, hi)
            t[self.sink:self.sink + moved.shape[0]] = moved
        self.head = 0

    def advance(self, current_start: int, num_new: int, local_attn_size: int, frame_seqlen: int):
        """The bookkeeping of causal_wanvideo.py:122-176. Returns (physical write segments for the new rows, physical
        [k0, k1) of the keys to attend). Eviction only moves the ring head whenever the attended window is the whole
        cache; otherwise the cache is kept in the reference's (shifted) order."""
        current_end = current_start + num_new
        if local_attn_size == -1:
            max_attention = GLOBAL_ATTN_COMPAT_MAX_LATENT_FRAMES * frame_seqlen
            if current_end > max_attention:
                raise ValueError("Causal Wan local_attn_size=-1 keeps the previous 21-latent-frame KV window; "
                                 f"got current_end={current_end} tokens with frame_seqlen={frame_seqlen}")
        else:
            max_attention = local_attn_size * frame_seqlen
        prev = self.local_end_index
        evicted = 0
        if local_attn_size != -1 and current_end > self.global_end_index and num_new + prev > self.size:
            evicted = num_new + prev - self.size
            if prev - evicted - self.sink < 0:
                raise ops.FvbError("KV cache too small for this block size and sink")
            self.head = (self.head + evicted) % (self.size - self.sink)
        local_end = prev + current_end - self.global_end_index - evicted
        if local_end > self.size or local_end - num_new < 0:
            raise ops.FvbError(f"KV cache overflow: local_end_index {local_end} of {self.size}")
        w0 = max(0, local_end - max_attention)
        if self.head != 0 and not (w0 == 0 and local_end == self.size):
            self.linearize(local_end)  # the window is a strict sub-range: it has to be contiguous and ordered
        self.global_end_index = current_end
        self.local_end_index = local_end
        window = (0, self.size) if self.head != 0 else (w0, local_end)
        return self.segments(local_end - num_new, local_end), window


_SCRATCH: dict = {}
_OFFSETS: dict = {}


def _scratch(key, shape, device) -> torch.Tensor:
    """Persistent workspace (stable address, so the column-offset tables below can be cached). Stream-ordered reuse:
    each layer's q is consumed by its attention launch before the next layer's GEMM overwrites it."""
    k = (key, str(device))
    if k not in _SCRATCH:
        _SCRATCH[k] = torch.empty(shape, dtype=torch.bfloat16, device=device)
    return _SCRATCH[k]


def _qkv_offsets(qs: torch.Tensor, ks: torch.Tensor, vs: torch.Tensor, H: int, d: int) -> torch.Tensor:
    """Element offsets (relative to qs) of the 3H head-column blocks of the fused QKV GEMM: q heads into the scratch
    rows, k / v heads into the cache rows (row stride H*d everywhere)."""
    key = (qs.data_ptr(), ks.data_ptr(), vs.data_ptr(), H, d)
    t = _OFFSETS.get(key)
    if t is None:
        if len(_OFFSETS) > 4096:
            _OFFSETS.clear()
        base = qs.data_ptr()
        t = torch.tensor([j * d for j in range(H)] + [(ks.data_ptr() - base) // 2 + j * d for j in range(H)] +
                         [(vs.data_ptr() - base) // 2 + j * d for j in range(H)], dtype=torch.int64).to(qs.device)
        _OFFSETS[key] = t
    return t


def _ident_offsets(D: int, device) -> torch.Tensor:
    key = ("ident", D, str(device))
    if key not in _OFFSETS:
        _OFFSETS[key] = torch.arange(0, D, 128, dtype=torch.int64, device=device)
    return _OFFSETS[key]


def _max_attention(ccfg: "CausalConfig", fs: int) -> int:
    return (GLOBAL_ATTN_COMPAT_MAX_LATENT_FRAMES if ccfg.local_attn_size == -1 else ccfg.local_attn_size) * fs


def _roped_window(cache: "KVCache", k0: int, k1: int, cos: torch.Tensor, sin: torch.Tensor, d: int) -> torch.Tensor:
    """Relativistic policy: key_window = rope(cache.k[window], table[0:window_len]) (causal_wanvideo.py:174-181) as ONE
    out-of-place row pass into a scratch that every layer reuses (stream-ordered: consumed by this layer's attention)."""
    Hc = cache.k.shape[1]
    Dc = Hc * d
    kr = _scratch(("k_roped", cache.size, Dc), (cache.size, Dc), cache.k.device)
    ops.rmsnorm_rope_scatter(cache.k.view(cache.size, Dc)[k0:k1], None, None, None, kr.data_ptr(), 0, Dc,
                             _ident_offsets(Dc, cache.k.device), cos, sin, rope_row=cache.window_positions(k0, k1), head_dim=d)
    return kr[:k1 - k0].view(k1 - k0, Hc, d)


def causal_block_forward(x: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, temb: torch.Tensor, cos: torch.Tensor,
                         sin: torch.Tensor, cache: KVCache, xcache: CrossAttnCache | None, current_start: int,
                         cfg: WanDiTConfig, ccfg: CausalConfig, frame_seqlen: int | None = None) -> torch.Tensor:
    """x: [S, D] bf16 (one sample; S = F * tokens-per-frame), temb: [F, 6, D] bf16 (timestep_proj of the F latent frames),
    cos/sin: float64 [S, head_dim] for exactly these tokens (absolute frame positions) -- or, with
    rope_cache_policy == "relativistic", the fixed table of the [0, max_attention_frames) window. Returns [S, D] bf16."""
    if ccfg.rope_cache_policy not in ("absolute", "relativistic"):
        raise ops.FvbError(f"unknown rope_cache_policy {ccfg.rope_cache_policy!r}")
    rel = ccfg.rope_cache_policy == "relativistic"
    S, D = x.shape
    H, d = cfg.num_attention_heads, cfg.head_dim
    refuse_grad("the causal block (per-frame bf16 modulation)", blk, x, ctx, temb)
    tpf = S // temb.shape[0]
    fs = tpf if frame_seqlen is None else int(frame_seqlen)
    mod = Modulation.per_frame(blk, temb, tpf)
    # self-attention over the cached window (causal_wanvideo.py:293-319, 73-185)
    n1 = mod.norm1(x, cfg.eps)
    q = _scratch(("q", S, D), (S, D), x.device)
    segs, (k0, k1) = cache.advance(current_start, S, ccfg.local_attn_size, fs)
    kf, vf = cache.k.view(cache.size, D), cache.v.view(cache.size, D)
    # relativistic: the query takes the tail of the window's table (_relative_rope.py:11-26), the cache keeps un-roped keys
    qlo = min(cache.local_end_index, _max_attention(ccfg, fs)) - S if rel else 0
    row = 0
    for p0, p1 in segs:  # one segment unless the ring wraps inside this block
        n = p1 - p0
        qs, ks, vs = q[row:row + n], kf[p0:p1], vf[p0:p1]
        offs = _qkv_offsets(qs, ks, vs, H, d)
        ops.linear_sp(n1[row:row + n], n, D, n1.stride(0), blk.w_qkv, blk.b_qkv, qs, D, out_col_offsets=offs)
        if rel:
            ops.rmsnorm_rope_(qs, blk.norm_q, None, None, cos[qlo + row:qlo + row + n], sin[qlo + row:qlo + row + n], head_dim=d, eps=cfg.eps)
            ops.rmsnorm_rope_(ks, blk.norm_k, head_dim=d, eps=cfg.eps)
        else:
            ops.rmsnorm_rope_(qs, blk.norm_q, ks, blk.norm_k, cos[row:row + n], sin[row:row + n], head_dim=d, eps=cfg.eps)
        row += n
    kw = _roped_window(cache, k0, k1, cos, sin, d) if rel else cache.k[k0:k1]
    a = ops.attention(q.view(1, S, H, d), kw.unsqueeze(0), cache.v[k0:k1].unsqueeze(0), softmax_scale=d ** -0.5)
    y = ops.linear_any(a.reshape(S, D), blk.w_o, blk.b_o, mod.attn_epilogue, resid=x, gate=mod.gate_msa, gate_rows=mod.rows)
    return block_tail(y, blk, ctx, mod, cfg, xcache)


def _require_bf16_model(cfg: WanDiTConfig) -> None:
    if cfg.fp8_linears:
        raise ops.FvbError("the causal rollout runs bf16 linears only: build the model with fp8_linears=False")
    if cfg.attention_8bit:
        raise ops.FvbError("the causal rollout runs bf16 attention only: build the model with attention_8bit=False")


def _pad_text(text: torch.Tensor, text_len: int) -> torch.Tensor:
    """text [B, L, text_dim] padded with zero rows to text_len before the embedder (causal_wanvideo.py:604-609)."""
    if text.shape[1] < text_len:
        text = torch.cat([text, text.new_zeros(text.shape[0], text_len - text.shape[1], text.shape[2])], 1)
    return text


def causal_block_train(x: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, temb: torch.Tensor, lay: TokenLayout,
                       cfg: WanDiTConfig, frame_seqlen: int, checkpoint: bool = False) -> torch.Tensor:
    """The causal block of the training forward: x [S, D] bf16 (one sample, S = F * frame_seqlen), ctx [L, D], temb [F, 6, D]
    bf16; block-causal self-attention over lay.causal, per-frame bf16 modulation. Differentiable (_WanBlockFn) when grad is
    enabled and x, ctx, temb or a tensor of blk.tensors() requires grad; the plain block_body otherwise (the same bits)."""
    if torch.is_grad_enabled() and _any_requires_grad(blk, x, ctx, temb):
        return block_forward_grad(x, blk, ctx, Modulation.per_frame(blk, temb, frame_seqlen), lay, cfg, checkpoint)
    return block_body(x, blk, ctx, Modulation.per_frame(blk, temb, frame_seqlen), lay, cfg)


def _inference_only(path: str):
    """A causal forward (model `self`, or `self.m` for the sequence-parallel one): refused under grad with latents, text or
    a model tensor requiring grad, run under torch.no_grad() otherwise."""
    def wrap(fn):
        @functools.wraps(fn)
        def run(self, latents, text, *args, **kwargs):
            refuse_model_grad(path, getattr(self, "m", self), latents, text)
            with torch.no_grad():
                return fn(self, latents, text, *args, **kwargs)
        return run
    return wrap


class CausalWanDiT(WanDiT):
    """CausalWanTransformer3DModel._forward_inference on libfvb200 (batch 1 per call, like the rollout stage)."""

    def __init__(self, cfg: WanDiTConfig, state_dict: dict, ccfg: CausalConfig, blocks: list | None = None):
        _require_bf16_model(cfg)
        super().__init__(cfg, state_dict, blocks)
        if any(blk.w_kv_img is not None for blk in self.blocks):
            raise ops.FvbError("the causal rollout's cross-attention is text-only: it cannot load image-to-video blocks")
        self.ccfg = ccfg
        self._rope: dict = {}

    @classmethod
    def random(cls, cfg: WanDiTConfig, ccfg: CausalConfig, device="cuda", seed: int = 2029) -> "CausalWanDiT":
        _require_bf16_model(cfg)
        base = WanDiT.random(cfg, device, seed)
        m = cls.__new__(cls)
        m.__dict__.update(base.__dict__)
        m.ccfg, m._rope = ccfg, {}
        return m

    def new_caches(self, frame_seqlen: int, device, cache_frames: int | None = None):
        """Per-layer caches sized like the stage does (causal_denoising.py:380-408): local_attn_size frames, or the
        21-frame compatibility window when local_attn_size == -1."""
        frames = cache_frames or (GLOBAL_ATTN_COMPAT_MAX_LATENT_FRAMES if self.ccfg.local_attn_size == -1
                                  else self.ccfg.local_attn_size)
        H, d = self.cfg.num_attention_heads, self.cfg.head_dim
        kv = [KVCache(frames * frame_seqlen, H, d, device, self.ccfg.sink_size * frame_seqlen) for _ in self.blocks]
        return kv, [CrossAttnCache() for _ in self.blocks]

    def rope_tables(self, frames: int, hw: tuple, start_frame: int, device):
        """float64 tables of frames [start_frame, start_frame + frames) (causal_wanvideo.py:583-598)."""
        key = (frames, tuple(hw), start_frame)
        if key not in self._rope:
            if len(self._rope) >= 16:  # bounded like the reference's LRU (rotary_embedding.py:453-458)
                self._rope.pop(next(iter(self._rope)))
            d = self.cfg.head_dim
            cos, sin = get_rotary_pos_embed((frames, ) + tuple(hw), [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)],
                                            theta=10000.0, start_frame=start_frame, keep_f64=True)
            self._rope[key] = (cos.to(device).contiguous(), sin.to(device).contiguous())
        return self._rope[key]

    def block_rope_tables(self, frames: int, hw: tuple, start_frame: int, device):
        """What the model hands its blocks (causal_wanvideo.py:580-595): the table of this call's frames at their
        absolute positions, or -- relativistic policy -- the fixed table over [0, max_attention_frames)."""
        if self.ccfg.rope_cache_policy == "relativistic":
            frames = GLOBAL_ATTN_COMPAT_MAX_LATENT_FRAMES if self.ccfg.local_attn_size == -1 else self.ccfg.local_attn_size
            start_frame = 0
        return self.rope_tables(frames, hw, start_frame, device)

    def forward(self, latents: torch.Tensor, text: torch.Tensor, timestep: torch.Tensor,
                vsa_sparsity: float | None = None) -> torch.Tensor:
        """WanDiT's bidirectional forward. Inference only for the causal model (forward_train is its training forward): it
        raises FvbError under grad with an input or a tensor of tensors() requiring grad."""
        refuse_model_grad("CausalWanDiT", self, latents, text)
        return super().forward(latents, text, timestep, vsa_sparsity)

    def train_layout(self, seq_shape: tuple, start_frame: int, device) -> TokenLayout:
        """Raster-order layout of the training forward: float64 RoPE tables at absolute frame positions from start_frame
        (with fp32 copies for the RoPE backward) and the block-causal tile tables (wan_dit.block_causal_tiles)."""
        F_, Hh, Ww = seq_shape
        key = ("train", tuple(seq_shape), start_frame, str(device))
        if key not in self._layouts:
            cos, sin = self.rope_tables(F_, (Hh, Ww), start_frame, device)
            tiles = block_causal_tiles(F_, Hh * Ww, self.ccfg.num_frames_per_block, self.ccfg.local_attn_size, device)
            self._layouts[key] = TokenLayout(seq_shape=tuple(seq_shape), cos=cos, sin=sin, causal=tiles,
                                             cos32=cos.float().contiguous(), sin32=sin.float().contiguous())
        return self._layouts[key]

    def forward_train(self, latents: torch.Tensor, text: torch.Tensor, timestep: torch.Tensor, start_frame: int = 0,
                      checkpoint: bool = False) -> torch.Tensor:
        """The training forward of the causal model (CausalWanTransformer3DModel._forward_train, causal_wanvideo.py:420-471):
        latents [B, C, F, H, W] bf16, text [B, L, text_dim], timestep [B, F] (one per latent frame) -> flow prediction, same
        shape as latents. Self-attention is block-causal: token i of frame block b (num_frames_per_block frames) attends the
        keys before the end of its block, and with local_attn_size != -1 only the last local_attn_size frames of them.
        Everything else is forward_inference's arithmetic (per-frame bf16 modulation, float64 RoPE at absolute positions from
        start_frame, text padded to text_len, per-frame head). Differentiable in latents, text and every tensor of tensors()
        when grad is enabled and one of them requires grad (the output has the bits of the call without grad). checkpoint:
        under grad, each block keeps only its input, its modulation and its self-attention output and LSE."""
        cfg = self.cfg
        if _any_model_tensor_requires_grad(self, latents, text):  # refused before anything runs
            if cfg.vsa:
                raise ops.FvbError("the causal model has no sparse self-attention path: build it with vsa=False to train it")
            for blk in self.blocks:
                _require_trainable(blk, cfg)
        if not latents.is_cuda:
            raise ops.FvbError("CausalWanDiT.forward_train needs CUDA tensors (there is no CPU fallback)")
        B = latents.shape[0]
        pt, ph, pw = cfg.patch_size
        F_, Hh, Ww = latents.shape[2] // pt, latents.shape[3] // ph, latents.shape[4] // pw
        if tuple(timestep.shape) != (B, F_):
            raise ops.FvbError(f"forward_train takes one timestep per latent frame: [{B}, {F_}], got {tuple(timestep.shape)}")
        fs = Hh * Ww
        lay = self.train_layout((F_, Hh, Ww), start_frame, latents.device)
        temb, tproj, ctx = self.condition(timestep.flatten(), _pad_text(text, cfg.text_len))  # [B F, D], [B F, 6, D], [B, L, D]
        x = self.patchify(latents.to(torch.bfloat16), lay)
        outs = []
        for b in range(B):
            xb, frames = x[b], slice(b * F_, (b + 1) * F_)
            for blk in self.blocks:
                xb = causal_block_train(xb, blk, ctx[b], tproj[frames], lay, cfg, fs, checkpoint)
            outs.append(self.head_per_frame(xb, temb[frames], fs))
        return self.unpatchify(torch.stack(outs, 0), lay)

    @_inference_only("CausalWanDiT.forward_inference")
    def forward_inference(self, latents: torch.Tensor, text: torch.Tensor, timestep: torch.Tensor, kv_cache: list,
                          crossattn_cache: list | None, current_start: int = 0, start_frame: int = 0) -> torch.Tensor:
        """latents [1, C, F, H, W] bf16 (the frame block being denoised), text [1, L, text_dim] bf16, timestep [1, F]
        (one per latent frame). Returns the flow prediction [1, C, F, H, W]. Raises FvbError under grad with an input or a
        tensor of tensors() requiring grad (there is no backward through the KV-cache rollout; forward_train trains the model)."""
        cfg = self.cfg
        if not latents.is_cuda:
            raise ops.FvbError("CausalWanDiT.forward_inference needs CUDA tensors (there is no CPU fallback)")
        if latents.shape[0] != 1:
            raise ops.FvbError("the causal rollout runs batch 1 (one KV cache per sample)")
        pt, ph, pw = cfg.patch_size
        F_, Hh, Ww = latents.shape[2] // pt, latents.shape[3] // ph, latents.shape[4] // pw
        fs = Hh * Ww
        lay = self.layout((F_, Hh, Ww), latents.device, None)
        cos, sin = self.block_rope_tables(F_, (Hh, Ww), start_frame, latents.device)
        text = _pad_text(text, cfg.text_len)
        temb, tproj, ctx = self.condition(timestep.flatten(), text)  # [F, D], [F, 6, D], [1, L, D]
        x = self.patchify(latents.to(torch.bfloat16), lay)[0]
        for i, blk in enumerate(self.blocks):
            x = causal_block_forward(x, blk, ctx[0], tproj, cos, sin, kv_cache[i],
                                     crossattn_cache[i] if crossattn_cache is not None else None, current_start, cfg,
                                     self.ccfg, frame_seqlen=fs)
        y = self.head_per_frame(x, temb, fs)
        return self.unpatchify(y.unsqueeze(0), lay)

    def head_per_frame(self, x: torch.Tensor, temb: torch.Tensor, frame_seqlen: int) -> torch.Tensor:
        """norm_out + proj_out with one (shift, scale) per latent frame (causal_wanvideo.py:646-650). The causal model
        builds LayerNormScaleShift without compute_dtype (causal_wanvideo.py:398-403), so this is nn.LayerNorm in bf16
        and a bf16 modulation (layernorm.py:253-273) -- not the fp32 variant of WanTransformer3DModel."""
        D = self.cfg.hidden_size
        if temb.dtype != torch.bfloat16 or self.scale_shift_table.dtype != torch.bfloat16:
            raise ops.FvbError("the causal head implements the bf16 modulation flow (bf16 temb and scale_shift_table)")
        e = (self.scale_shift_table.reshape(1, 2, D) + temb.unsqueeze(1)).float()  # [F, 2, D], bf16 values
        if _requires_grad(x, e):
            n = _HeadNormFramesFn.apply(x, e[:, 1], e[:, 0], frame_seqlen, self.cfg.eps)
        else:
            n = ops.layernorm_modulate(x, e[:, 1], e[:, 0], round_ln=True, eps=self.cfg.eps, mod_rows=frame_seqlen, mod_bf16=True)
        return _linear(n, self.w_out, self.b_out)


# ----------------------------------------------------------------------------------------------------------------
# sequence-parallel causal rollout: head-sharded KV cache (SURVEY section 8e / 8f-1; the reference runs replicas)
# ----------------------------------------------------------------------------------------------------------------
class SPCausalWanDiT:
    """CausalWanDiT over `world` ranks. Every rank holds all weights; rank r owns heads [r*H/P, (r+1)*H/P) of every layer's
    KV cache and, of each latent frame of the block being denoised, the contiguous token slice [r*n, (r+1)*n), n = fs / P
    (per-frame slices keep the per-frame AdaLN grouping local: mod_rows = n). Per layer:

      token owners:  LN+modulate -> fused QKV GEMM; V heads go straight from the GEMM epilogue into the OWNER RANK'S cache
                     rows, q / k heads through the RMSNorm+RoPE pass into the owner's q buffer / cache rows (peer-memory
                     stores over NVLink, the same offset tables as the bidirectional push exchange) -> barrier
      head owners:   attention of the block's 3 frames (all tokens, my heads) against my cache window -> rows scattered
                     back to the token owners' buffers by one kernel -> barrier
      token owners:  out-projection (A operand K-segmented by source rank), cross-attention, FFN.

    Only the new block's tokens ever cross the fabric (4 680 of them against a 32 760-token window); the cache itself never
    moves. Cache rows of a frame are laid out [rank][token slice], consistently for every block, so eviction (whole frames)
    and the sink prefix work exactly as in KVCache; attention is invariant to the order of keys inside the window.
    Requires fs % P == 0 and torch symmetric memory (there is no collective fallback on this path: it raises)."""

    def __init__(self, model: CausalWanDiT, rank: int, world: int, group=None):
        import torch.distributed as dist
        _require_bf16_model(model.cfg)
        self.m, self.rank, self.world = model, rank, world
        self.group = group or dist.group.WORLD
        if model.cfg.num_attention_heads % world:
            raise ops.FvbError("num_attention_heads must be divisible by the sequence-parallel size")
        self.Hl = model.cfg.num_attention_heads // world
        self._st = None

    # ---- symmetric slab: [q buffer | back buffer | k, v of every layer], one allocation => one peer delta for every table
    def new_caches(self, frame_seqlen: int, block_tokens: int, device, cache_frames: int | None = None):
        import torch.distributed._symmetric_memory as symm
        m, P, Hl, d = self.m, self.world, self.Hl, self.m.cfg.head_dim
        if frame_seqlen % P:
            raise ops.FvbError(f"tokens per latent frame ({frame_seqlen}) must be divisible by the sequence-parallel size {P}")
        frames = cache_frames or (GLOBAL_ATTN_COMPAT_MAX_LATENT_FRAMES if m.ccfg.local_attn_size == -1 else m.ccfg.local_attn_size)
        size, L = frames * frame_seqlen, len(m.blocks)
        S = block_tokens
        n_q, n_back, n_c = S * Hl * d, S * Hl * d, size * Hl * d  # back: [P(src), S/P, Hl, d] has S * Hl * d elements
        slab = symm.empty((n_q + n_back + 2 * L * n_c,), dtype=torch.bfloat16, device=device)
        slab.zero_()
        hdl = symm.rendezvous(slab, self.group)
        base = [int(p_) for p_ in hdl.buffer_ptrs]
        if any((b - base[self.rank]) % 16 for b in base):
            raise ops.FvbError("peer mappings are not 16-byte congruent")
        q = slab[:n_q].view(S, Hl, d)
        back = slab[n_q:n_q + n_back].view(P, S // P, Hl, d)
        kv, off = [], n_q + n_back
        for _ in range(L):
            k = slab[off:off + n_c].view(size, Hl, d)
            v = slab[off + n_c:off + 2 * n_c].view(size, Hl, d)
            kv.append(KVCache(size, Hl, d, device, m.ccfg.sink_size * frame_seqlen, storage=(k, v)))
            off += 2 * n_c
        H = m.cfg.num_attention_heads
        # per-head element offset from MY slab base to the head's slot in its OWNER's slab (projection-relative)
        head_off = torch.tensor([(base[h // Hl] - base[self.rank]) // 2 + (h % Hl) * d for h in range(H)], dtype=torch.int64,
                                device=device)
        n = frame_seqlen // P
        # return path: block row (f, r', j) -> rank r' back[me][f * n + j]: one segment of n rows per (frame, destination)
        F_ = S // frame_seqlen
        my_back_elem = n_q + self.rank * (S // P) * Hl * d
        seg = torch.tensor([base[r_] + 2 * (my_back_elem + f * n * Hl * d) for f in range(F_) for r_ in range(P)],
                           dtype=torch.int64, device=device)
        torch.cuda.synchronize(device)
        hdl.barrier(channel=0)
        self._st = dict(slab=slab, hdl=hdl, q=q, back=back, head_off=head_off, seg=seg, fs=frame_seqlen, S=S, n=n)
        return kv, [CrossAttnCache() for _ in m.blocks]

    def _block(self, x, blk, ctx, temb, cos, sin, cache: KVCache, xcache, current_start):
        m, st, Hl = self.m, self._st, self.Hl
        cfg, ccfg = m.cfg, m.ccfg
        D, d = cfg.hidden_size, cfg.head_dim
        fs, S, n = st["fs"], st["S"], st["n"]
        refuse_grad("the sequence-parallel causal block", blk, x, ctx, temb)
        mod = Modulation.per_frame(blk, temb, n)
        n1 = mod.norm1(x, cfg.eps)
        segs, (k0, k1) = cache.advance(current_start, S, ccfg.local_attn_size, fs)
        # physical cache row of each frame of the block (write segments split at frame boundaries at most)
        frame_row = []
        for p0, p1 in segs:
            frame_row += list(range(p0, p1, fs))
        qk = ops.linear_any(n1, blk.w_qkv[:2 * D], blk.b_qkv[:2 * D])  # local [S_loc, 2D]: RMSNorm needs whole rows
        slab, rowb = st["slab"], Hl * d
        q_base, k_base, v_base = st["q"].data_ptr(), cache.k.data_ptr(), cache.v.data_ptr()
        v_off = st["head_off"] + (v_base - slab.data_ptr()) // 2
        rel = ccfg.rope_cache_policy == "relativistic"
        for f in range(temb.shape[0]):
            rows = slice(f * n, (f + 1) * n)
            drow = frame_row[f] + self.rank * n     # destination row inside the owner's cache
            qrow = f * fs + self.rank * n           # destination row inside the owner's q buffer (block order)
            ops.linear_sp(n1[rows], n, D, n1.stride(0), blk.w_qkv[2 * D:3 * D], blk.b_qkv[2 * D:3 * D], slab, rowb,
                          out_col_offsets=v_off + drow * rowb)
            if rel:  # keys travel un-roped (cos/sin are my query rows' tables: the tail of the window)
                ops.rmsnorm_rope_scatter(qk[rows, :D], blk.norm_q, None, None, q_base + 2 * qrow * rowb, 0, rowb, st["head_off"],
                                         cos[rows], sin[rows], head_dim=d, eps=cfg.eps)
                ops.rmsnorm_rope_scatter(qk[rows, D:], blk.norm_k, None, None, k_base + 2 * drow * rowb, 0, rowb, st["head_off"],
                                         head_dim=d, eps=cfg.eps)
            else:
                ops.rmsnorm_rope_scatter(qk[rows, :D], blk.norm_q, qk[rows, D:], blk.norm_k, q_base + 2 * qrow * rowb,
                                         k_base + 2 * drow * rowb, rowb, st["head_off"], cos[rows], sin[rows], head_dim=d, eps=cfg.eps)
        st["hdl"].barrier(channel=0)  # every rank's q / k / v rows of this block have landed in my slab
        kw = _roped_window(cache, k0, k1, st["win_cos"], st["win_sin"], d) if rel else cache.k[k0:k1]
        o = ops.attention(st["q"].unsqueeze(0), kw.unsqueeze(0), cache.v[k0:k1].unsqueeze(0), softmax_scale=d ** -0.5)
        ops.scatter_rows_to_segments(o[0].view(S, rowb), st["seg"], n)
        st["hdl"].barrier(channel=1)  # my tokens' heads have arrived from every rank (and everyone is done reading q)
        return block_tail(out_proj_sp(st["back"], blk, x, mod), blk, ctx, mod, cfg, xcache)

    @_inference_only("SPCausalWanDiT.forward_inference")
    def forward_inference(self, latents, text, timestep, kv_cache, crossattn_cache, current_start: int = 0, start_frame: int = 0):
        """Same contract as CausalWanDiT.forward_inference; every rank passes the same inputs and gets the full prediction."""
        import torch.distributed as dist
        m, cfg, st, P = self.m, self.m.cfg, self._st, self.world
        if m.ccfg.rope_cache_policy not in ("absolute", "relativistic"):
            raise ops.FvbError(f"unknown rope_cache_policy {m.ccfg.rope_cache_policy!r}")
        pt, ph, pw = cfg.patch_size
        F_, Hh, Ww = latents.shape[2] // pt, latents.shape[3] // ph, latents.shape[4] // pw
        fs, n = Hh * Ww, st["n"]
        assert fs == st["fs"] and F_ * fs == st["S"]
        lay = m.layout((F_, Hh, Ww), latents.device, None)
        cos, sin = m.block_rope_tables(F_, (Hh, Ww), start_frame, latents.device)
        text = _pad_text(text, cfg.text_len)
        temb, tproj, ctx = m.condition(timestep.flatten(), text)
        # my rows of the block: for every frame, tokens [rank * n, (rank + 1) * n)
        idx = (torch.arange(F_, device=latents.device)[:, None] * fs + self.rank * n +
               torch.arange(n, device=latents.device)[None, :]).reshape(-1)
        patches = m.patches(latents.to(torch.bfloat16))[0]
        x = ops.linear(patches[idx].contiguous(), m.w_patch, m.b_patch)
        qlo = 0
        if m.ccfg.rope_cache_policy == "relativistic":
            # every layer's cache moves in lock-step: the window length after this call's advance() follows from layer 0's
            # counters (the bookkeeping of KVCache.advance / causal_wanvideo.py:122-176, evaluated without side effects)
            c0 = kv_cache[0]
            end = current_start + F_ * fs
            prev = c0.local_end_index
            evicted = max(0, F_ * fs + prev - c0.size) if (m.ccfg.local_attn_size != -1 and end > c0.global_end_index) else 0
            local_end = prev + end - c0.global_end_index - evicted
            qlo = min(local_end, _max_attention(m.ccfg, fs)) - F_ * fs
            st["win_cos"], st["win_sin"] = cos, sin
        cl, sl = cos[qlo + idx].contiguous(), sin[qlo + idx].contiguous()
        for i, blk in enumerate(m.blocks):
            x = self._block(x, blk, ctx[0], tproj, cl, sl, kv_cache[i], crossattn_cache[i] if crossattn_cache is not None else None,
                            current_start)
        y_loc = m.head_per_frame(x, temb, n)  # [F * n, C * pt * ph * pw]
        y_all = torch.empty((P, *y_loc.shape), dtype=y_loc.dtype, device=y_loc.device)
        dist.all_gather_into_tensor(y_all.view(-1), y_loc.contiguous().view(-1), group=self.group)
        # [P, F, n, c] -> block order (f, r, j)
        y = y_all.view(P, F_, n, -1).permute(1, 0, 2, 3).reshape(F_ * fs, -1)
        return m.unpatchify(y.unsqueeze(0), lay)
