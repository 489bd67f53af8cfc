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

import math
from dataclasses import dataclass

import torch

from . import ops
from .rope import get_rotary_pos_embed
from .wan_dit import WanBlock, WanDiT, WanDiTConfig

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


class CrossAttnCache:
    """crossattn_cache entry (wanvideo.py:202-211): text K/V computed on the first call of a rollout."""

    def __init__(self):
        self.kv = None


def causal_block_forward(x: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, temb: torch.Tensor, cos: torch.Tensor,
                         sin: torch.Tensor, cache: KVCache, xcache: CrossAttnCache | None, current_start: int,
                         cfg: WanDiTConfig, ccfg: CausalConfig, frame_seqlen: int | None = None) -> torch.Tensor:
    """x: [S, D] bf16 (one sample; S = F * tokens-per-frame), temb: [F, 6, D] bf16 (timestep_proj of the F latent frames),
    cos/sin: float64 [S, head_dim] for exactly these tokens (absolute frame positions) -- or, with
    rope_cache_policy == "relativistic", the fixed table of the [0, max_attention_frames) window. Returns [S, D] bf16."""
    if ccfg.rope_cache_policy not in ("absolute", "relativistic"):
        raise ops.FvbError(f"unknown rope_cache_policy {ccfg.rope_cache_policy!r}")
    rel = ccfg.rope_cache_policy == "relativistic"
    if temb.dtype != torch.bfloat16 or blk.scale_shift_table.dtype != torch.bfloat16:
        raise ops.FvbError("the causal block implements the bf16 modulation flow (bf16 temb and scale_shift_table)")
    S, D = x.shape
    H, d = cfg.num_attention_heads, cfg.head_dim
    nf = temb.shape[0]
    tpf = S // nf
    fs = tpf if frame_seqlen is None else int(frame_seqlen)
    # e = scale_shift_table + temb in bf16 (causal_wanvideo.py:288); the kernels take fp32 copies of those bf16 values
    e = (blk.scale_shift_table + temb.unsqueeze(0)).reshape(nf, 6, D).float()
    shift_msa, scale_msa, gate_msa, c_shift, c_scale, c_gate = (e[:, i] for i in range(6))  # [F, D] views, stride 6D

    # 1. self-attention over the cached window (causal_wanvideo.py:293-319, 73-185)
    n1 = ops.layernorm_modulate(x, scale_msa, shift_msa, round_ln=True, eps=cfg.eps, mod_rows=tpf, mod_bf16=True)
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
    # to_out + per-frame gated residual (bf16 product), then LayerNorm(affine) of the bf16 residual (layernorm.py:159-213)
    x = ops.linear(a.reshape(S, D), blk.w_o, blk.b_o, ops.EPI_RESID_GATE_BF16R, resid=x, gate=gate_msa, gate_rows=tpf)
    n2 = ops.layernorm_modulate(x, None, None, blk.norm2_w, blk.norm2_b, round_ln=True, eps=cfg.eps)

    # 2. cross-attention, text K/V cached across the rollout (wanvideo.py:188-222)
    q2 = ops.linear(n2, blk.w_q2, blk.b_q2)
    ops.rmsnorm_rope_(q2, blk.norm_q2, head_dim=d, eps=cfg.eps)
    if xcache is not None and xcache.kv is not None:
        kv2 = xcache.kv
    else:
        kv2 = ops.linear(ctx, blk.w_kv2, blk.b_kv2)
        ops.rmsnorm_rope_(kv2[:, :D], blk.norm_k2, head_dim=d, eps=cfg.eps)
        if xcache is not None:
            xcache.kv = kv2
    a2 = ops.attention(q2.unflatten(1, (H, d)).unsqueeze(0), kv2[:, :D].unflatten(1, (H, d)).unsqueeze(0),
                       kv2[:, D:].unflatten(1, (H, d)).unsqueeze(0), softmax_scale=d ** -0.5).reshape(S, D)
    x = ops.linear(a2, blk.w_o2, blk.b_o2, ops.EPI_RESID_BF16, resid=x)
    n3 = ops.layernorm_modulate(x, c_scale, c_shift, round_ln=True, eps=cfg.eps, mod_rows=tpf, mod_bf16=True)

    # 3. feed-forward + per-frame gated residual (causal_wanvideo.py:338-340)
    f = ops.linear(n3, blk.w_1, blk.b_1, ops.EPI_BIAS_GELU_TANH)
    return ops.linear(f, blk.w_2, blk.b_2, ops.EPI_RESID_GATE_BF16R, resid=x, gate=c_gate, gate_rows=tpf)


class CausalWanDiT(WanDiT):
    """CausalWanTransformer3DModel._forward_inference on libfvb200 (batch 1 per call, like the rollout stage)."""

    def __init__(self, cfg: WanDiTConfig, state_dict: dict, ccfg: CausalConfig, blocks: list | None = None):
        super().__init__(cfg, state_dict, blocks)
        self.ccfg = ccfg
        self._rope: dict = {}

    @classmethod
    def random(cls, cfg: WanDiTConfig, ccfg: CausalConfig, device="cuda", seed: int = 2029) -> "CausalWanDiT":
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

    @torch.no_grad()
    def forward_inference(self, latents: torch.Tensor, text: torch.Tensor, timestep: torch.Tensor, kv_cache: list,
                          crossattn_cache: list | None, current_start: int = 0, start_frame: int = 0) -> torch.Tensor:
        """latents [1, C, F, H, W] bf16 (the frame block being denoised), text [1, L, text_dim] bf16, timestep [1, F]
        (one per latent frame). Returns the flow prediction [1, C, F, H, W]."""
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
        # text padded with zero rows to text_len before the embedder (causal_wanvideo.py:604-609)
        if text.shape[1] < cfg.text_len:
            text = torch.cat([text, text.new_zeros(1, cfg.text_len - text.shape[1], text.shape[2])], 1)
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
        n = ops.layernorm_modulate(x, e[:, 1], e[:, 0], round_ln=True, eps=self.cfg.eps, mod_rows=frame_seqlen, mod_bf16=True)
        return ops.linear(n, self.w_out, self.b_out)


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
        m, st, P, Hl = self.m, self._st, self.world, self.Hl
        cfg, ccfg = m.cfg, m.ccfg
        D, H, d = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim
        fs, S, n = st["fs"], st["S"], st["n"]
        S_loc, nf = x.shape[0], temb.shape[0]
        e = (blk.scale_shift_table + temb.unsqueeze(0)).reshape(nf, 6, D).float()
        shift_msa, scale_msa, gate_msa, c_shift, c_scale, c_gate = (e[:, i] for i in range(6))
        n1 = ops.layernorm_modulate(x, scale_msa, shift_msa, round_ln=True, eps=cfg.eps, mod_rows=n, mod_bf16=True)
        segs, (k0, k1) = cache.advance(current_start, S, ccfg.local_attn_size, fs)
        # physical cache row of each frame of the block (write segments split at frame boundaries at most)
        frame_row = []
        for p0, p1 in segs:
            frame_row += list(range(p0, p1, fs))
        qk = ops.linear(n1, blk.w_qkv[:2 * D], blk.b_qkv[:2 * D])  # local [S_loc, 2D]: RMSNorm needs whole rows
        slab, rowb = st["slab"], Hl * d
        q_base, k_base, v_base = st["q"].data_ptr(), cache.k.data_ptr(), cache.v.data_ptr()
        v_off = st["head_off"] + (v_base - slab.data_ptr()) // 2
        rel = ccfg.rope_cache_policy == "relativistic"
        for f in range(nf):
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
        y = torch.empty((S_loc, D), dtype=torch.bfloat16, device=x.device)
        ops.linear_sp(st["back"], S_loc, D, rowb, blk.w_o, blk.b_o, y, D, ops.EPI_RESID_GATE_BF16R, x_seg_len=rowb,
                      x_seg_stride=S_loc * rowb, resid=x, gate=gate_msa, gate_rows=n)
        x = y
        n2 = ops.layernorm_modulate(x, None, None, blk.norm2_w, blk.norm2_b, round_ln=True, eps=cfg.eps)
        q2 = ops.linear(n2, blk.w_q2, blk.b_q2)
        ops.rmsnorm_rope_(q2, blk.norm_q2, head_dim=d, eps=cfg.eps)
        if xcache is not None and xcache.kv is not None:
            kv2 = xcache.kv
        else:
            kv2 = ops.linear(ctx, blk.w_kv2, blk.b_kv2)
            ops.rmsnorm_rope_(kv2[:, :D], blk.norm_k2, head_dim=d, eps=cfg.eps)
            if xcache is not None:
                xcache.kv = kv2
        a2 = ops.attention(q2.unflatten(1, (H, d)).unsqueeze(0), kv2[:, :D].unflatten(1, (H, d)).unsqueeze(0),
                           kv2[:, D:].unflatten(1, (H, d)).unsqueeze(0), softmax_scale=d ** -0.5).reshape(S_loc, D)
        x = ops.linear(a2, blk.w_o2, blk.b_o2, ops.EPI_RESID_BF16, resid=x)
        n3 = ops.layernorm_modulate(x, c_scale, c_shift, round_ln=True, eps=cfg.eps, mod_rows=n, mod_bf16=True)
        f_ = ops.linear(n3, blk.w_1, blk.b_1, ops.EPI_BIAS_GELU_TANH)
        return ops.linear(f_, blk.w_2, blk.b_2, ops.EPI_RESID_GATE_BF16R, resid=x, gate=c_gate, gate_rows=n)

    @torch.no_grad()
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
        if text.shape[1] < cfg.text_len:
            text = torch.cat([text, text.new_zeros(1, cfg.text_len - text.shape[1], text.shape[2])], 1)
        temb, tproj, ctx = m.condition(timestep.flatten(), text)
        # my rows of the block: for every frame, tokens [rank * n, (rank + 1) * n)
        idx = (torch.arange(F_, device=latents.device)[:, None] * fs + self.rank * n +
               torch.arange(n, device=latents.device)[None, :]).reshape(-1)
        B, C, T, Hl_, Wl_ = latents.shape
        patches = latents.to(torch.bfloat16).view(B, C, T // pt, pt, Hl_ // ph, ph, Wl_ // pw, pw) \
            .permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(F_ * fs, C * pt * ph * pw)
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
