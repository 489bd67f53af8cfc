"""Wan DiT denoising-step forward on libfvb200 (single rank; the sequence-parallel variant lives in
fastvideo_b200/distributed.py and reuses the per-block routines here).

Mirrors, op for op and rounding point for rounding point:
  WanTransformerBlock.forward / WanTransformerBlock_VSA.forward  fastvideo/models/dits/wanvideo.py:361-434, 520-582
  WanT2VCrossAttention.forward                                   fastvideo/models/dits/wanvideo.py:188-222
  WanTransformer3DModel.forward                                  fastvideo/models/dits/wanvideo.py:656-766
  WanTimeTextImageEmbedding.forward                              fastvideo/models/dits/wanvideo.py:100-135
Parameter names are the reference's (so a reference state_dict loads unchanged); q/k/v(/gate) projections are
concatenated at load time so one GEMM produces them.

B200-first differences that do not change results:
  * every linear is one tcgen05 GEMM with its bias / GELU / gated-residual epilogue fused;
  * QK-RMSNorm + RoPE is one in-place pass over the fused QKV buffer; attention reads q/k/v straight out of
    that buffer through strided TMA descriptors (no torch.cat, no transposes);
  * with VSA the whole network runs in compact tile-major token order (one permutation at patchify, one at
    unpatchify) instead of a tile scatter + untile gather around every attention layer, and no zero padding
    rows are carried (the attention kernel masks by variable block size).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import torch

from . import ops, vsa
from .rope import get_rotary_pos_embed

VSA_TILE = (4, 4, 4)  # fastvideo/attention/backends/video_sparse_attn.py:29


@dataclass
class WanDiTConfig:
    """Subset of fastvideo/configs/models/dits/wanvideo.py:64-93 that the forward needs."""
    hidden_size: int = 5120
    num_attention_heads: int = 40
    ffn_dim: int = 13824
    num_layers: int = 40
    in_channels: int = 16
    out_channels: int = 16
    patch_size: tuple = (1, 2, 2)
    text_dim: int = 4096
    text_len: int = 512
    freq_dim: int = 256
    eps: float = 1e-6
    vsa: bool = False  # WanTransformerBlock_VSA (to_gate_compress present)
    # Opt-in FP8: the six token-stream GEMMs of every block (FP8_LINEARS) run on e4m3 weights (per output channel) and
    # e4m3 activations (per token) through ops.linear_fp8; those weights are quantised once at load and no bf16 copy is
    # kept. The text-side K/V projections, the embedders, patch embedding and proj_out stay bf16.
    fp8_linears: bool = False
    # Opt-in 8-bit self-attention (INT8 Q K^T, FP8 P V; ops.quantize_attention_8bit + ops.attention_8bit), dense and the VSA
    # sparse branch. Cross-attention and the VSA compression branch stay bf16. Independent of fp8_linears.
    attention_8bit: bool = False
    # Opt-in INT8 weights: every block linear (INT8_LINEARS) keeps int8 weights with one fp32 scale per output channel
    # (ops.Int8Weight, quantised once at load; no bf16 copy is kept) and runs on bf16 activations through
    # fvb_linear_w8_sp. The embedders, patch embedding and proj_out stay bf16. Combines with vsa and attention_8bit, and
    # runs on the sequence-parallel and causal paths; exclusive with fp8_linears.
    int8_weights: bool = False
    # Opt-in W8A8, on top of int8_weights: the activations of every INT8_LINEARS GEMM are quantised to int8 as well, one
    # fp32 scale per token (fvb_quantize_int8_rows), and the GEMM runs s8 x s8 -> s32 (fvb_linear_w8a8_sp). Same paths as
    # int8_weights; the weights are the same Int8Weight objects, marked for int8 activations.
    int8_activations: bool = False

    def __post_init__(self):
        if self.int8_weights and self.fp8_linears:
            raise ops.FvbError("int8_weights and fp8_linears are exclusive: pick one weight format")
        if self.int8_activations and not self.int8_weights:
            raise ops.FvbError("int8_activations needs int8_weights=True (the W8A8 GEMM takes int8 weights)")

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


WAN_14B = dict(hidden_size=5120, num_attention_heads=40, ffn_dim=13824, num_layers=40)
WAN_1_3B = dict(hidden_size=1536, num_attention_heads=12, ffn_dim=8960, num_layers=30)


def random_state_dict(cfg: WanDiTConfig, device="cuda", seed: int = 2029, dtype=torch.bfloat16,
                      layers: int | None = None) -> dict:
    """Synthetic weights with the reference's names: xavier-uniform for >=2-D, zeros for biases, ones for norm
    weights, scale_shift_table ~ randn/sqrt(D) (recipe of fastvideo/tests/distributed/test_sp_wan.py:113-126,
    wanvideo.py:359)."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    D, F = cfg.hidden_size, cfg.ffn_dim
    sd = {}

    def lin(name, out_f, in_f, fan_in=None, fan_out=None):
        a = math.sqrt(6.0 / ((fan_in or in_f) + (fan_out or out_f)))
        w = torch.empty((out_f, in_f), device=device, dtype=torch.float32)
        w.uniform_(-a, a, generator=g)
        sd[name + ".weight"] = w.to(dtype)
        sd[name + ".bias"] = torch.zeros(out_f, device=device, dtype=dtype)

    pt, ph, pw = cfg.patch_size
    kin = cfg.in_channels * pt * ph * pw
    lin("patch_embedding.proj", D, kin, fan_in=kin, fan_out=D * pt * ph * pw)
    sd["patch_embedding.proj.weight"] = sd["patch_embedding.proj.weight"].view(D, cfg.in_channels, pt, ph, pw)
    lin("condition_embedder.time_embedder.mlp.fc_in", D, cfg.freq_dim)
    lin("condition_embedder.time_embedder.mlp.fc_out", D, D)
    lin("condition_embedder.time_modulation.linear", 6 * D, D)
    lin("condition_embedder.text_embedder.fc_in", D, cfg.text_dim)
    lin("condition_embedder.text_embedder.fc_out", D, D)
    for i in range(cfg.num_layers if layers is None else layers):
        p = f"blocks.{i}."
        for n in ("to_q", "to_k", "to_v", "to_out") + (("to_gate_compress",) if cfg.vsa else ()):
            lin(p + n, D, D)
        for n in ("attn2.to_q", "attn2.to_k", "attn2.to_v", "attn2.to_out"):
            lin(p + n, D, D)
        lin(p + "ffn.fc_in", F, D)
        lin(p + "ffn.fc_out", D, F)
        for n in ("norm_q", "norm_k", "attn2.norm_q", "attn2.norm_k"):
            sd[p + n + ".weight"] = torch.ones(D, device=device, dtype=dtype)
        sd[p + "self_attn_residual_norm.norm.weight"] = torch.ones(D, device=device, dtype=dtype)
        sd[p + "self_attn_residual_norm.norm.bias"] = torch.zeros(D, device=device, dtype=dtype)
        sd[p + "scale_shift_table"] = (torch.randn((1, 6, D), device=device, generator=g) / D ** 0.5).to(dtype)
    sd["scale_shift_table"] = (torch.randn((1, 2, D), device=device, generator=g) / D ** 0.5).to(dtype)
    lin("proj_out", cfg.out_channels * pt * ph * pw, D)
    return sd


# WanBlock weights that multiply the token stream; with WanDiTConfig.fp8_linears they are ops.Fp8Weight
FP8_LINEARS = ("w_qkv", "w_o", "w_q2", "w_o2", "w_1", "w_2")
# every WanBlock linear weight; with WanDiTConfig.int8_weights they are ops.Int8Weight (w_kv_img only on I2V blocks)
INT8_LINEARS = FP8_LINEARS + ("w_kv2", "w_kv_img")


class WanBlock:
    """Weights of one transformer block in the layout the kernels want."""

    def __init__(self, sd: dict, prefix: str, cfg: WanDiTConfig):
        g = lambda n: sd[prefix + n]
        bf = lambda t: t.to(torch.bfloat16).contiguous()
        # RMSNorm weights keep an fp32 dtype: with an fp32 parameter `x.to(orig_dtype) * self.weight` (layernorm.py:73-79) is
        # an fp32 product that is rounded only once, after RoPE -- the row kernels reproduce that (SURVEY a4)
        nw = lambda t: t.contiguous() if t.dtype == torch.float32 else bf(t)
        names = ["to_q", "to_k", "to_v"] + (["to_gate_compress"] if cfg.vsa else [])
        self.w_qkv = bf(torch.cat([g(n + ".weight") for n in names], 0))
        self.b_qkv = bf(torch.cat([g(n + ".bias") for n in names], 0))
        self.norm_q = nw(g("norm_q.weight"))
        self.norm_k = nw(g("norm_k.weight"))
        self.w_o, self.b_o = bf(g("to_out.weight")), bf(g("to_out.bias"))
        self.norm2_w = g("self_attn_residual_norm.norm.weight").float().contiguous()
        self.norm2_b = g("self_attn_residual_norm.norm.bias").float().contiguous()
        self.w_q2, self.b_q2 = bf(g("attn2.to_q.weight")), bf(g("attn2.to_q.bias"))
        self.w_kv2 = bf(torch.cat([g("attn2.to_k.weight"), g("attn2.to_v.weight")], 0))
        self.b_kv2 = bf(torch.cat([g("attn2.to_k.bias"), g("attn2.to_v.bias")], 0))
        self.norm_q2 = nw(g("attn2.norm_q.weight"))
        self.norm_k2 = nw(g("attn2.norm_k.weight"))
        # WanI2VCrossAttention (wanvideo.py:225-280): image-token K/V projections next to the text ones
        self.w_kv_img = self.b_kv_img = self.norm_k_img = None
        if prefix + "attn2.add_k_proj.weight" in sd:
            self.w_kv_img = bf(torch.cat([g("attn2.add_k_proj.weight"), g("attn2.add_v_proj.weight")], 0))
            self.b_kv_img = bf(torch.cat([g("attn2.add_k_proj.bias"), g("attn2.add_v_proj.bias")], 0))
            self.norm_k_img = bf(g("attn2.norm_added_k.weight"))
        self.w_o2, self.b_o2 = bf(g("attn2.to_out.weight")), bf(g("attn2.to_out.bias"))
        self.w_1, self.b_1 = bf(g("ffn.fc_in.weight")), bf(g("ffn.fc_in.bias"))
        self.w_2, self.b_2 = bf(g("ffn.fc_out.weight")), bf(g("ffn.fc_out.bias"))
        self.scale_shift_table = g("scale_shift_table")  # dtype as loaded: the modulation sum happens in torch
        self.trainable = not (cfg.fp8_linears or cfg.int8_weights)
        if cfg.fp8_linears:
            for n in FP8_LINEARS:  # replacing the attribute drops the block's bf16 copy
                setattr(self, n, ops.Fp8Weight.quantize(getattr(self, n)))
        if cfg.int8_weights:
            for n in INT8_LINEARS:
                if getattr(self, n) is not None:
                    setattr(self, n, ops.Int8Weight.quantize(getattr(self, n), cfg.int8_activations))


    def tensors(self) -> dict:
        """The block's trainable tensors in its own fused layout, by attribute name (every one a leaf an optimizer can
        step; w_kv_img / b_kv_img / norm_k_img only on I2V blocks). `to_reference_names` maps this dict, or one of their
        .grad, back to the reference parameter names."""
        names = ["w_qkv", "b_qkv", "norm_q", "norm_k", "w_o", "b_o", "norm2_w", "norm2_b", "w_q2", "b_q2", "w_kv2", "b_kv2",
                 "norm_q2", "norm_k2", "w_o2", "b_o2", "w_1", "b_1", "w_2", "b_2", "scale_shift_table"]
        if self.w_kv_img is not None:
            names += ["w_kv_img", "b_kv_img", "norm_k_img"]
        return {n: getattr(self, n) for n in names}

    @staticmethod
    def to_reference_names(t: dict, prefix: str = "", like: dict | None = None) -> dict:
        """{fused name: tensor} (WanBlock.tensors(), or the same keys holding gradients) -> {reference name: tensor}: the
        fused QKV(+gate) / text KV / image KV rows are split back into their projections (views, no copies). An entry may be
        None (the .grad of a tensor that is not trained): its reference names map to None, and `like` (the block's own
        tensors()) gives the shapes the split needs."""
        out = {}
        s = t if like is None else like
        D = s["w_o"].shape[0]
        rows = lambda src, a, b: None if t[src] is None else t[src][a:b]
        qkv = ["to_q", "to_k", "to_v", "to_gate_compress"][:s["w_qkv"].shape[0] // D]
        for i, n in enumerate(qkv):
            out[n + ".weight"] = rows("w_qkv", i * D, (i + 1) * D)
            out[n + ".bias"] = rows("b_qkv", i * D, (i + 1) * D)
        for src, dst in (("w_kv2", "attn2.to_{}.weight"), ("b_kv2", "attn2.to_{}.bias")):
            out[dst.format("k")], out[dst.format("v")] = rows(src, 0, D), rows(src, D, None)
        if "w_kv_img" in t:
            for src, dst in (("w_kv_img", "attn2.add_{}_proj.weight"), ("b_kv_img", "attn2.add_{}_proj.bias")):
                out[dst.format("k")], out[dst.format("v")] = rows(src, 0, D), rows(src, D, None)
            out["attn2.norm_added_k.weight"] = t["norm_k_img"]
        plain = {"norm_q": "norm_q.weight", "norm_k": "norm_k.weight", "w_o": "to_out.weight", "b_o": "to_out.bias",
                 "norm2_w": "self_attn_residual_norm.norm.weight", "norm2_b": "self_attn_residual_norm.norm.bias",
                 "w_q2": "attn2.to_q.weight", "b_q2": "attn2.to_q.bias", "norm_q2": "attn2.norm_q.weight",
                 "norm_k2": "attn2.norm_k.weight", "w_o2": "attn2.to_out.weight", "b_o2": "attn2.to_out.bias",
                 "w_1": "ffn.fc_in.weight", "b_1": "ffn.fc_in.bias", "w_2": "ffn.fc_out.weight", "b_2": "ffn.fc_out.bias",
                 "scale_shift_table": "scale_shift_table"}
        for src, dst in plain.items():
            out[dst] = t[src]
        return {prefix + k: v for k, v in out.items()}


@dataclass
class TokenLayout:
    """How the S tokens of this forward are ordered, and what attention needs to know about it."""
    seq_shape: tuple                    # (T, H, W) after patchify
    cos: torch.Tensor                   # fp32 [S, head_dim] RoPE tables in RASTER order
    sin: torch.Tensor
    perm: torch.Tensor | None = None    # int64 [S]: position -> raster index (None = raster order)
    inv_perm: torch.Tensor | None = None
    rope_row: torch.Tensor | None = None  # int32 [S] = perm
    vbs: torch.Tensor | None = None     # int32 [n_tiles] variable block sizes
    block_off: torch.Tensor | None = None  # int32 [n_tiles + 1]
    row_block: torch.Tensor | None = None  # int32 [S] token position -> tile
    topk: int = 0
    causal: "BlockCausalTiles | None" = None  # block-causal self-attention (causal model training)
    cos32: torch.Tensor | None = None   # fp32 copies of float64 cos / sin for the RoPE backward (None: cos / sin are fp32)
    sin32: torch.Tensor | None = None


@dataclass
class BlockCausalTiles:
    """Block-causal self-attention as a block list over variable-length tiles (ops.attention_blocklist /
    ops.attention_sparse_bwd). Token i of frame block b = i // (n fs) attends key j iff j < end_b = min((b + 1) n fs, S) and,
    with a local window of W = local_attn_size fs tokens, j >= end_b - W. q tiles (at most 64 rows, token order) are cut at
    every end_b, kv tiles also at every window start inside the sequence, so each (q tile, kv tile) pair is wholly inside or
    wholly outside the mask."""
    q_off: torch.Tensor     # int32 [nqb + 1]
    kv_off: torch.Tensor    # int32 [nkb + 1]
    tile_map: torch.Tensor  # bool [1, 1, nqb, nkb]
    q2k_idx: torch.Tensor   # int32 [1, 1, nqb, nkb] / q2k_num [1, 1, nqb]: ops.map_to_index(tile_map)
    q2k_num: torch.Tensor
    k2q_idx: torch.Tensor   # int32 [1, 1, nkb, nqb] / k2q_num [1, 1, nkb]: the transposed map's lists
    k2q_num: torch.Tensor

    @property
    def nkb(self) -> int:
        return self.kv_off.numel() - 1


def block_causal_tile_map(frames: int, frame_seqlen: int, frames_per_block: int, local_attn_size: int = -1):
    """Host tile tables of the block-causal mask (BlockCausalTiles): (q_off int32 [nqb + 1], kv_off int32 [nkb + 1], tile_map
    bool [nqb, nkb]). frames need not be a multiple of frames_per_block (the last block is shorter)."""
    S, L = frames * frame_seqlen, frames_per_block * frame_seqlen
    if S <= 0 or L <= 0 or (local_attn_size != -1 and local_attn_size <= 0):
        raise ops.FvbError("block-causal tiles need frames, frame_seqlen, frames_per_block > 0 and local_attn_size -1 or > 0")
    ends = [min(e, S) for e in range(L, S + L, L)]
    W = local_attn_size * frame_seqlen if local_attn_size != -1 else None
    lo = [max(0, e - W) if W is not None else 0 for e in ends]

    def tiles(cuts):
        cuts = sorted(set(cuts) | {0, S})
        off = [a + i for a, b in zip(cuts, cuts[1:]) for i in range(0, b - a, 64)]
        return torch.tensor(off + [S], dtype=torch.int32)

    q_off, kv_off = tiles(ends), tiles(ends + lo)
    block = torch.bucketize(q_off[:-1].long(), torch.tensor(ends), right=True)  # frame block of each q tile
    end_q, lo_q = torch.tensor(ends)[block], torch.tensor(lo)[block]
    tile_map = (kv_off[None, 1:].long() <= end_q[:, None]) & (kv_off[None, :-1].long() >= lo_q[:, None])
    return q_off, kv_off, tile_map


_BLOCK_CAUSAL: dict = {}


def block_causal_tiles(frames: int, frame_seqlen: int, frames_per_block: int, local_attn_size: int, device) -> BlockCausalTiles:
    """BlockCausalTiles on `device`, built once per (frames, frame_seqlen, frames_per_block, local_attn_size, device)."""
    key = (frames, frame_seqlen, frames_per_block, local_attn_size, str(device))
    if key not in _BLOCK_CAUSAL:
        q_off, kv_off, tile_map = block_causal_tile_map(frames, frame_seqlen, frames_per_block, local_attn_size)
        m = tile_map.to(device)[None, None]
        q2k_idx, q2k_num = ops.map_to_index(m.contiguous())
        k2q_idx, k2q_num = ops.map_to_index(m.transpose(-1, -2).contiguous())
        _BLOCK_CAUSAL[key] = BlockCausalTiles(q_off.to(device), kv_off.to(device), m, q2k_idx, q2k_num, k2q_idx, k2q_num)
    return _BLOCK_CAUSAL[key]


def make_layout(seq_shape, cfg: WanDiTConfig, device, vsa_sparsity: float | None = None) -> TokenLayout:
    d = cfg.head_dim
    rope_dim_list = [d - 4 * (d // 6), 2 * (d // 6), 2 * (d // 6)]  # wanvideo.py:680
    cos, sin = get_rotary_pos_embed(seq_shape, rope_dim_list, theta=10000.0)
    lay = TokenLayout(seq_shape=tuple(seq_shape), cos=cos.to(device).contiguous(), sin=sin.to(device).contiguous())
    if vsa_sparsity is not None:
        t = ops.vsa_tile_index(seq_shape, VSA_TILE, device=device)
        lay.perm = t["tile_partition"]
        lay.inv_perm = t["reverse_partition"]
        lay.rope_row = t["tile_partition"].to(torch.int32)
        lay.vbs = t["variable_block_sizes"]
        lay.block_off = t["block_offsets"]
        nblk = lay.vbs.numel()
        lay.row_block = torch.repeat_interleave(torch.arange(nblk, device=device, dtype=torch.int32), lay.vbs.long())
        # compute_topk: fastvideo/attention/backends/video_sparse_attn.py:161-163
        lay.topk = max(1, min(math.ceil((1 - vsa_sparsity) * nblk), nblk))
    return lay


@dataclass
class Modulation:
    """AdaLN modulation of one block and the rounding flow it implies: fp32 (WanTransformerBlock, wanvideo.py:388-390; one
    row for all tokens) or bf16 (CausalWanTransformerBlock, causal_wanvideo.py:288; one row per latent frame of `rows`
    tokens, every modulation / gate product rounded to bf16)."""
    shift_msa: torch.Tensor
    scale_msa: torch.Tensor
    gate_msa: torch.Tensor
    c_shift: torch.Tensor
    c_scale: torch.Tensor
    c_gate: torch.Tensor
    rows: int = 0  # tokens per modulation row; 0: one row for all tokens
    bf16: bool = False

    @classmethod
    def fp32(cls, blk: WanBlock, temb6: torch.Tensor) -> "Modulation":  # temb6: [1, 6, D]
        e = blk.scale_shift_table + temb6.float()
        return cls(*[t.reshape(temb6.shape[-1]).contiguous() for t in e.chunk(6, dim=1)])

    @classmethod
    def per_frame(cls, blk: WanBlock, temb: torch.Tensor, rows: int) -> "Modulation":  # temb: [F, 6, D] bf16
        if temb.dtype != torch.bfloat16 or blk.scale_shift_table.dtype != torch.bfloat16:
            raise ops.FvbError("the causal block implements the bf16 modulation flow (bf16 temb and scale_shift_table)")
        # the kernels take fp32 copies of the bf16 sums; the [F, D] views keep their 6D row stride
        e = (blk.scale_shift_table + temb.unsqueeze(0)).reshape(temb.shape).float()
        return cls(*(e[:, i] for i in range(6)), rows=rows, bf16=True)

    def norm1(self, x: torch.Tensor, eps: float) -> torch.Tensor:
        return ops.layernorm_modulate(x, self.scale_msa, self.shift_msa, round_ln=self.bf16, eps=eps, mod_rows=self.rows,
                                      mod_bf16=self.bf16)

    @property
    def attn_epilogue(self) -> int:  # out-projection + gated residual: fp32 output, or bf16 product and output
        return ops.EPI_RESID_GATE_BF16R if self.bf16 else ops.EPI_RESID_GATE_F32

    @property
    def ffn_epilogue(self) -> int:
        return ops.EPI_RESID_GATE_BF16R if self.bf16 else ops.EPI_RESID_GATE_BF16


@dataclass
class CrossAttnCache:
    """crossattn_cache entry (wanvideo.py:202-211): text K/V computed on the first call of a rollout."""
    kv: torch.Tensor | None = None


I2V_IMAGE_TOKENS = 257  # wanvideo.py:259-260: the first 257 context rows are the CLIP image tokens


def _keep(keep: dict | None, **tensors) -> None:
    """With `keep` (the block under grad, _WanBlockFn), record tensors the backward needs."""
    if keep is not None:
        keep.update(tensors)


def _linear_kept(keep: dict | None, name: str, x, w, bias, epilogue: int, **kw) -> torch.Tensor:
    """linear_any; with `keep`, the bf16 y the epilogue consumes is kept under `name` as well (fvb_linear_bf16_aux)."""
    if keep is None:
        return ops.linear_any(x, w, bias, epilogue, **kw)
    out, keep[name] = ops.linear_aux(x, w, bias, epilogue, **kw)
    return out


def _attention_kept(keep: dict | None, name: str, q, k, v, softmax_scale: float) -> torch.Tensor:
    """ops.attention; with `keep`, its log-sum-exp is kept under `name`."""
    if keep is None:
        return ops.attention(q, k, v, softmax_scale=softmax_scale)
    out, keep[name] = ops.attention(q, k, v, softmax_scale=softmax_scale, return_lse=True)
    return out


def cross_attention(n2: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, cfg: WanDiTConfig,
                    xcache: CrossAttnCache | None = None, keep: dict | None = None) -> torch.Tensor:
    """WanT2VCrossAttention.forward (wanvideo.py:188-222), or WanI2VCrossAttention.forward (:225-280) when the block
    carries add_k_proj / add_v_proj: text attention + image-token attention, summed in bf16. Returns [S, D] (pre to_out).
    With `xcache`, the text K/V are computed on the first call and reused afterwards. `keep`: see _keep."""
    S, D = n2.shape
    H, d = cfg.num_attention_heads, cfg.head_dim
    hd = lambda t: t.unflatten(1, (H, d)).unsqueeze(0)
    q2 = ops.linear_any(n2, blk.w_q2, blk.b_q2)
    _keep(keep, q2_pre=q2.clone() if keep is not None else None)
    ops.rmsnorm_rope_(q2, blk.norm_q2, head_dim=d, eps=cfg.eps)
    img = None
    if blk.w_kv_img is not None:
        ctx_img, ctx = ctx[:I2V_IMAGE_TOKENS], ctx[I2V_IMAGE_TOKENS:]
        kvi = ops.linear_any(ctx_img.contiguous(), blk.w_kv_img, blk.b_kv_img)
        _keep(keep, ki_pre=kvi[:, :D].clone() if keep is not None else None)
        ops.rmsnorm_rope_(kvi[:, :D], blk.norm_k_img, head_dim=d, eps=cfg.eps)
        img = _attention_kept(keep, "lse_i", hd(q2), hd(kvi[:, :D]), hd(kvi[:, D:]), d ** -0.5).reshape(S, D)
        _keep(keep, kvi=kvi, img=img)
        if ctx.shape[0] == 0:
            if keep is not None:
                raise ops.FvbError("the I2V block backward needs text tokens after the 257 image tokens")
            return img  # zeros_like(q) + img_x
    if xcache is not None and xcache.kv is not None:
        kv2 = xcache.kv
    else:
        kv2 = ops.linear_any(ctx.contiguous(), blk.w_kv2, blk.b_kv2)  # [L, 2D]
        _keep(keep, k2_pre=kv2[:, :D].clone() if keep is not None else None)
        ops.rmsnorm_rope_(kv2[:, :D], blk.norm_k2, head_dim=d, eps=cfg.eps)
        if xcache is not None:
            xcache.kv = kv2
    a2 = _attention_kept(keep, "lse2", hd(q2), hd(kv2[:, :D]), hd(kv2[:, D:]), d ** -0.5).reshape(S, D)
    _keep(keep, q2=q2, kv2=kv2, a2t=a2)
    return a2 if img is None else a2 + img  # `x = x + img_x` on bf16 tensors


def block_tail(y: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, mod: Modulation, cfg: WanDiTConfig,
               xcache: CrossAttnCache | None = None, keep: dict | None = None) -> torch.Tensor:
    """The block after the self-attention out-projection y (fp32 or bf16, per mod.attn_epilogue): LayerNorm(affine),
    cross-attention, feed-forward (wanvideo.py:415-432, causal_wanvideo.py:321-340). Returns [S, D] bf16. `keep`: see
    _keep (fp32 modulation flow only)."""
    if mod.bf16:  # LayerNorm of the bf16 residual (layernorm.py:159-213)
        n2, x = ops.layernorm_modulate(y, None, None, blk.norm2_w, blk.norm2_b, round_ln=True, eps=cfg.eps), y
    else:  # LayerNorm of the fp32 residual, which also becomes the bf16 residual stream
        n2, x = ops.layernorm_modulate(y, None, None, blk.norm2_w, blk.norm2_b, eps=cfg.eps, want_hidden=True)
    a2 = cross_attention(n2, blk, ctx, cfg, xcache, keep)
    x = ops.linear_any(a2, blk.w_o2, blk.b_o2, ops.EPI_RESID_BF16, resid=x)
    n3 = ops.layernorm_modulate(x, mod.c_scale, mod.c_shift, round_ln=True, eps=cfg.eps, mod_rows=mod.rows, mod_bf16=mod.bf16)
    f = _linear_kept(keep, "h", n3, blk.w_1, blk.b_1, ops.EPI_BIAS_GELU_TANH)
    _keep(keep, n2=n2, a2=a2, x2=x, n3=n3, f=f)
    return _linear_kept(keep, "o3", f, blk.w_2, blk.b_2, mod.ffn_epilogue, resid=x, gate=mod.c_gate, gate_rows=mod.rows)


def block_forward(x: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, temb6: torch.Tensor, lay: TokenLayout,
                  cfg: WanDiTConfig, checkpoint: bool = False) -> torch.Tensor:
    """x: [S, D] bf16 (one sample), ctx: [L, D] bf16 text states, temb6: [1, 6, D] (timestep_proj). Returns [S, D].
    Differentiable (in x, ctx, temb6 and every tensor of blk.tensors()) when grad is enabled and one of them requires grad:
    the block then runs _WanBlockFn, whose forward is this same body (block_body) and returns the same bits.
    checkpoint: under grad, keep only the block input, the modulation and the self-attention results
    (checkpoint_bytes_per_block); the backward re-runs the block around the saved self-attention first."""
    if torch.is_grad_enabled() and _any_requires_grad(blk, x, ctx, temb6):
        _require_trainable(blk, cfg)
        # torch ops: autograd carries the six vectors back to scale_shift_table and temb6
        return block_forward_grad(x, blk, ctx, Modulation.fp32(blk, temb6), lay, cfg, checkpoint)
    return block_body(x, blk, ctx, Modulation.fp32(blk, temb6), lay, cfg)


def block_body(x: torch.Tensor, blk: WanBlock, ctx: torch.Tensor, mod: Modulation, lay: TokenLayout, cfg: WanDiTConfig,
               keep: dict | None = None, attn: dict | None = None, replay: bool = False) -> torch.Tensor:
    """The single-rank block: self-attention (wanvideo.py:393-415; block-causal over lay.causal's tile lists when it is set),
    then block_tail. `keep`: see _keep. `attn` (the checkpointed block, _WanBlockFn) records the self-attention results:
    dense and block-causal "a" and "lse"; VSA the tensors
    _VideoSparseAttnFn saves besides q / k / v / gate, under their _VideoSparseAttnFn.SAVED names. With `replay` those
    results are used instead of launching the self-attention (for VSA the output is recombined from the saved branches
    and the recomputed gate by the same fvb_vsa_combine call, so the same bits)."""
    S, D = x.shape
    H, d = cfg.num_attention_heads, cfg.head_dim
    n1 = mod.norm1(x, cfg.eps)
    qkv = ops.linear_any(n1, blk.w_qkv, blk.b_qkv)  # [S, 3D or 4D]
    _keep(keep, n1=n1, qkv=qkv, qk_pre=qkv[:, :2 * D].clone() if keep is not None else None)
    ops.rmsnorm_rope_(qkv[:, :D], blk.norm_q, qkv[:, D:2 * D], blk.norm_k, lay.cos, lay.sin, lay.rope_row, head_dim=d,
                      eps=cfg.eps)
    q = qkv[:, :D].unflatten(1, (H, d)).unsqueeze(0)
    k = qkv[:, D:2 * D].unflatten(1, (H, d)).unsqueeze(0)
    v = qkv[:, 2 * D:3 * D].unflatten(1, (H, d)).unsqueeze(0)
    if cfg.vsa:
        gate = qkv[:, 3 * D:4 * D].unflatten(1, (H, d)).unsqueeze(0)
        if replay:
            a = ops.vsa_combine(attn["out_s"], attn["out_c"], gate, row_block=lay.row_block)
            _keep(keep, vsa=(q, k, v, gate, *(attn[n] for n in vsa._VideoSparseAttnFn.SAVED[4:])))
        elif keep is None and attn is None:
            a = vsa.video_sparse_attn_bshd(q, k, v, lay.vbs, lay.topk, gate=gate, block_off=lay.block_off,
                                           row_block=lay.row_block, attn_8bit=cfg.attention_8bit)
        else:  # the same kernels in the same order (bit-identical), keeping what the VSA backward needs
            vctx = _SavedCtx()
            a = vsa._VideoSparseAttnFn.forward(vctx, q, k, v, gate, lay.vbs, lay.topk, None, lay.block_off, lay.row_block)
            _keep(keep, vsa=vctx.saved_tensors)
            if attn is not None:
                attn.update(zip(vsa._VideoSparseAttnFn.SAVED[4:], vctx.saved_tensors[4:]))
    elif cfg.attention_8bit:
        a = ops.attention_8bit(ops.quantize_attention_8bit(q, k, v), d ** -0.5)
    elif replay:
        a = attn["a"]
        _keep(keep, lse=attn["lse"])
    elif lay.causal is not None:  # block-causal (causal model training): the tile lists of lay.causal
        c = lay.causal
        a, lse = ops.attention_blocklist(q, k, v, c.q2k_idx, c.q2k_num, softmax_scale=d ** -0.5, return_lse=True,
                                         q_off=c.q_off, kv_off=c.kv_off, nkb=c.nkb)
        a = a.reshape(S, D)
        _keep(keep, lse=lse)
        if attn is not None:
            attn.update(a=a, lse=lse)
    elif attn is not None:
        a, attn["lse"] = ops.attention(q, k, v, softmax_scale=d ** -0.5, return_lse=True)
        attn["a"] = a = a.reshape(S, D)
    else:
        a = _attention_kept(keep, "lse", q, k, v, d ** -0.5)
    _keep(keep, a=a.reshape(S, D))
    y = _linear_kept(keep, "o1", a.reshape(S, D), blk.w_o, blk.b_o, mod.attn_epilogue, resid=x, gate=mod.gate_msa,
                     gate_rows=mod.rows)
    _keep(keep, y=y)
    return block_tail(y, blk, ctx, mod, cfg, keep=keep)


# ------------------------------------------------------------------------------------------------ block backward
def _any_requires_grad(blk: WanBlock, *inputs) -> bool:
    # quantised weights (ops.Fp8Weight / ops.Int8Weight) are not tensors and never require grad
    return any(getattr(t, "requires_grad", False) for t in (*inputs, *blk.tensors().values()))


def refuse_grad(path: str, blk: WanBlock, *inputs) -> None:
    """Raise FvbError when a block path without a backward would run under grad with something requiring grad (it would
    otherwise return an output without a grad_fn)."""
    if torch.is_grad_enabled() and _any_requires_grad(blk, *inputs):
        raise ops.FvbError(f"{path} has no backward: run it under torch.no_grad(), or train the single-rank block "
                           "(wan_dit.block_forward)")


_BLOCK_TENSORS = ("w_qkv", "b_qkv", "norm_q", "norm_k", "w_o", "b_o", "norm2_w", "norm2_b", "w_q2", "b_q2", "w_kv2", "b_kv2",
                  "norm_q2", "norm_k2", "w_o2", "b_o2", "w_1", "b_1", "w_2", "b_2", "w_kv_img", "b_kv_img", "norm_k_img")
_FN_LEAD = 13  # _WanBlockFn inputs before the block tensors: x, ctx, six modulation vectors, blk, lay, cfg, checkpoint, rows


def _require_trainable(blk: WanBlock, cfg: WanDiTConfig) -> None:
    """Raise FvbError for a block configuration the backward does not cover."""
    if not blk.trainable or cfg.attention_8bit:
        raise ops.FvbError("the Wan block backward covers bf16 linears and bf16 attention: fp8_linears, int8_weights / "
                           "int8_activations and attention_8bit run without grad only")
    for n in ("norm_q", "norm_k", "norm_q2", "norm_k2", "norm_k_img"):
        t = getattr(blk, n)
        if t is not None and t.dtype != torch.bfloat16:
            raise ops.FvbError(f"the Wan block backward needs bf16 RMSNorm weights ({n} is {t.dtype})")
    if cfg.vsa and vsa.SPARSE_KERNEL != "ws":
        raise ops.FvbError("the VSA backward needs the block-list sparse kernel (FVB_VSA_KERNEL=ws)")


def block_forward_grad(x, blk: WanBlock, ctx, mod: Modulation, lay: TokenLayout, cfg: WanDiTConfig, checkpoint: bool) -> torch.Tensor:
    """The block under grad (_WanBlockFn) for a modulation computed with torch ops (Modulation.fp32, or Modulation.per_frame:
    the bf16 flow, one row per mod.rows tokens)."""
    if mod.bf16 != (mod.rows > 0):
        raise ops.FvbError("the block backward covers the fp32 modulation flow and the per-frame bf16 one")
    return _WanBlockFn.apply(x, ctx, mod.shift_msa, mod.scale_msa, mod.gate_msa, mod.c_shift, mod.c_scale, mod.c_gate, blk, lay,
                             cfg, checkpoint, mod.rows, *(getattr(blk, n) for n in _BLOCK_TENSORS))


def checkpoint_bytes_per_block(S: int, D: int, H: int, n_tiles: int = 0, frames: int = 1) -> int:
    """Bytes a checkpointed block (block_forward(..., checkpoint=True)) keeps from its forward to its backward, for S
    tokens of width D in H heads: the bf16 input, the fp32 modulation vectors (six rows of D, or of F D for the causal model's
    per-frame modulation over `frames` latent frames), and the self-attention results. Dense or block-causal (n_tiles 0):
    the bf16 output and the fp32 LSE. VSA (n_tiles tiles): the sparse branch's bf16 output and fp32 LSE, the block
    means (q, k transposed with rows padded to 8 tiles; v) and the compression output, the block-score softmax (rows
    padded to 8), the int32 index lists and counts and the bool block map. The layout tables and the text states are
    shared by every block and not counted."""
    n, n8 = n_tiles, (n_tiles + 7) // 8 * 8
    common = 2 * S * D + 6 * 4 * D * frames + 2 * S * D + 4 * S * H
    if not n_tiles:
        return common
    d = D // H
    return common + H * (2 * 2 * d * n8 + 2 * 2 * n * d + 2 * n * n8 + 4 * n * n + 4 * n + n * n)


class _SavedCtx:
    """Stands in for an autograd ctx when _VideoSparseAttnFn runs inside _WanBlockFn (its tensors are then saved by
    _WanBlockFn's own ctx)."""

    def save_for_backward(self, *t):
        self.saved_tensors = t


class _WanBlockFn(torch.autograd.Function):
    """block_forward with autograd. The forward is block_body with a `keep` dict: the same kernel calls (same bits), plus
    storage for the backward -- the pre-norm q / k / q2 / k2 (cloned before the in-place norms), the attention LSEs, and the
    pre-epilogue bf16 y of the fc_in / to_out / fc_out GEMMs (fvb_linear_bf16_aux). The backward is torch autograd's for the
    reference block (DESIGN.md "Wan block backward"); weight / bias / context gradients that no input needs are skipped.
    With `checkpoint` the forward keeps only x, ctx, the modulation vectors and the self-attention results (block_body's
    `attn`); the backward first re-runs block_body with a `keep` dict around those results (no self-attention launch) and
    then proceeds as without checkpoint. The forward kernels are deterministic, so the re-run keeps the same bits and the
    gradients are those of the forward without checkpoint."""

    @staticmethod
    def forward(fctx, x, ctx, shift_msa, scale_msa, gate_msa, c_shift, c_scale, c_gate, blk, lay, cfg, checkpoint, rows, *params):
        keep, attn = (None, {}) if checkpoint else ({}, None)
        mod = Modulation(shift_msa, scale_msa, gate_msa, c_shift, c_scale, c_gate, rows=rows, bf16=rows > 0)
        out = block_body(x.detach(), blk, ctx.detach(), mod, lay, cfg, keep, attn)
        fctx.blk, fctx.lay, fctx.cfg, fctx.checkpoint, fctx.rows = blk, lay, cfg, checkpoint, rows
        if checkpoint:
            fctx.names = tuple(attn)
            fctx.save_for_backward(x, ctx, scale_msa, gate_msa, c_scale, c_gate, shift_msa, c_shift, *attn.values())
            return out
        vsa_saved = keep.pop("vsa", ())
        fctx.names = tuple(keep)
        fctx.save_for_backward(x, ctx, scale_msa, gate_msa, c_scale, c_gate, *keep.values(), *vsa_saved)
        return out

    @staticmethod
    def backward(fctx, dout):
        x, ctx, scale_msa, gate_msa, c_scale, c_gate = fctx.saved_tensors[:6]
        blk, lay, cfg, R = fctx.blk, fctx.lay, fctx.cfg, fctx.rows
        if fctx.checkpoint:
            shift_msa, c_shift, *saved = fctx.saved_tensors[6:]
            kp = {}
            block_body(x, blk, ctx, Modulation(shift_msa, scale_msa, gate_msa, c_shift, c_scale, c_gate, rows=R, bf16=R > 0), lay,
                       cfg, kp, dict(zip(fctx.names, saved)), replay=True)
            vsa_saved = kp.pop("vsa", ())
        else:
            names = fctx.names
            kp = dict(zip(names, fctx.saved_tensors[6:6 + len(names)]))
            vsa_saved = fctx.saved_tensors[6 + len(names):]
        need = lambda n: fctx.needs_input_grad[_FN_LEAD + _BLOCK_TENSORS.index(n)]
        S, D = x.shape
        H, d = cfg.num_attention_heads, cfg.head_dim
        hd = lambda t: t.unflatten(1, (H, d)).unsqueeze(0)
        eps = cfg.eps
        want_dctx = fctx.needs_input_grad[1]
        g = {}
        dout = dout.to(torch.bfloat16).contiguous()
        # per-frame bf16 modulation flow (R > 0): the grouped kernels, one modulation / gate row per R tokens
        resid_gate_bwd = ((lambda do, y_, gt, need_db: ops.resid_gate_grouped_bwd(do, y_, gt, R, need_db)) if R
                          else ops.resid_gate_bwd)
        # feed-forward: out = bf16(x2 + o3 * c_gate), o3 = fc_out(f), f = gelu(h), h = fc_in(n3)
        d_o3, d_cgate, g["b_2"] = resid_gate_bwd(dout, kp["o3"], c_gate, need_db=need("b_2"))
        if need("w_2"):
            g["w_2"] = ops.linear_bwd(kp["f"], blk.w_2, d_o3, need_dx=False)[1]
        dh = ops.linear_dgrad_gelu(d_o3, blk.w_2, kp["h"])
        dn3, g["w_1"], g["b_1"] = ops.linear_bwd(kp["n3"], blk.w_1, dh, need_dw=need("w_1"), need_db=need("b_1"))
        if R:
            dx2, d_cscale, d_cshift = ops.layernorm_modulate_grouped_bwd(kp["x2"], dn3, c_scale, R, gin=dout, eps=eps)
        else:
            dx2, d_cscale, d_cshift = ops.layernorm_modulate_bwd(kp["x2"], dn3, scale=c_scale, round_ln=True, gin=dout, eps=eps)
        # cross-attention: x2 = bf16(xb + to_out2(a2)), a2 = a2t (+ img)
        da2, g["w_o2"], g["b_o2"] = ops.linear_bwd(kp["a2"], blk.w_o2, dx2, need_dw=need("w_o2"), need_db=need("b_o2"))
        q2, kv2 = kp["q2"], kp["kv2"]
        dq2, dk2, dv2 = ops.attention_bwd(hd(q2), hd(kv2[:, :D]), hd(kv2[:, D:]), hd(kp["a2t"]), kp["lse2"], hd(da2),
                                          softmax_scale=d ** -0.5)
        dq2 = dq2.view(S, D)
        ctx_txt = ctx[I2V_IMAGE_TOKENS:] if blk.w_kv_img is not None else ctx
        dctx_txt = dctx_img = None
        if want_dctx or need("w_kv2") or need("b_kv2") or need("norm_k2"):
            dkv2 = torch.empty_like(kv2)
            dk2_pre, g["norm_k2"] = ops.rmsnorm_bwd(kp["k2_pre"], blk.norm_k2, dk2.view(-1, D), eps=eps,
                                                    want_dw=need("norm_k2"))
            dkv2[:, :D].copy_(dk2_pre)
            dkv2[:, D:].copy_(dv2.view(-1, D))
            dctx_txt, g["w_kv2"], g["b_kv2"] = ops.linear_bwd(ctx_txt.contiguous(), blk.w_kv2, dkv2, need_dx=want_dctx,
                                                               need_dw=need("w_kv2"), need_db=need("b_kv2"))
        if blk.w_kv_img is not None:
            kvi = kp["kvi"]
            dq2i, dki, dvi = ops.attention_bwd(hd(q2), hd(kvi[:, :D]), hd(kvi[:, D:]), hd(kp["img"]), kp["lse_i"], hd(da2),
                                               softmax_scale=d ** -0.5)
            dq2 = dq2 + dq2i.view(S, D)
            if want_dctx or need("w_kv_img") or need("b_kv_img") or need("norm_k_img"):
                dkvi = torch.empty_like(kvi)
                dki_pre, g["norm_k_img"] = ops.rmsnorm_bwd(kp["ki_pre"], blk.norm_k_img, dki.view(-1, D), eps=eps,
                                                           want_dw=need("norm_k_img"))
                dkvi[:, :D].copy_(dki_pre)
                dkvi[:, D:].copy_(dvi.view(-1, D))
                dctx_img, g["w_kv_img"], g["b_kv_img"] = ops.linear_bwd(
                    ctx[:I2V_IMAGE_TOKENS].contiguous(), blk.w_kv_img, dkvi, need_dx=want_dctx, need_dw=need("w_kv_img"),
                    need_db=need("b_kv_img"))
        dctx = None
        if want_dctx:
            dctx = dctx_txt if dctx_img is None else torch.cat([dctx_img, dctx_txt], 0)
        dq2_pre, g["norm_q2"] = ops.rmsnorm_bwd(kp["q2_pre"], blk.norm_q2, dq2, eps=eps, want_dw=need("norm_q2"))
        dn2, g["w_q2"], g["b_q2"] = ops.linear_bwd(kp["n2"], blk.w_q2, dq2_pre, need_dw=need("w_q2"), need_db=need("b_q2"))
        # norm2 of the residual y (fp32, or bf16 in the per-frame flow; n2 = bf16(LN(y) w + b)); xb = bf16(y) carries dx2 into
        # dy as well
        dy, g["norm2_w"], g["norm2_b"] = ops.layernorm_modulate_bwd(kp["y"], dn2, weight=blk.norm2_w, gin=dx2, eps=eps)
        # self-attention out-projection: y = x + o1 * gate_msa
        d_o1, d_gate_msa, g["b_o"] = resid_gate_bwd(dy, kp["o1"], gate_msa, need_db=need("b_o"))
        da, g["w_o"], _ = ops.linear_bwd(kp["a"], blk.w_o, d_o1, need_dw=need("w_o"))
        qkv = kp["qkv"]
        dqkv = torch.empty_like(qkv)
        if cfg.vsa:
            vctx = _SavedCtx()
            vctx.saved_tensors = vsa_saved
            vctx.needs_input_grad = (True, True, True, True)
            dq, dk, dv, dgate = vsa._VideoSparseAttnFn.backward(vctx, hd(da))[:4]
            dqkv[:, 3 * D:].copy_(dgate.view(S, D))
        elif lay.causal is not None:
            c = lay.causal
            q, k, v = hd(qkv[:, :D]), hd(qkv[:, D:2 * D]), hd(qkv[:, 2 * D:3 * D])
            dq, dk, dv = ops.attention_sparse_bwd(q, k, v, hd(kp["a"]), kp["lse"], hd(da), c.q2k_idx, c.q2k_num, c.k2q_idx,
                                                  c.k2q_num, q_off=c.q_off, kv_off=c.kv_off, softmax_scale=d ** -0.5)
        else:
            q, k, v = hd(qkv[:, :D]), hd(qkv[:, D:2 * D]), hd(qkv[:, 2 * D:3 * D])
            dq, dk, dv = ops.attention_bwd(q, k, v, hd(kp["a"]), kp["lse"], hd(da), softmax_scale=d ** -0.5)
        dqkv[:, 2 * D:3 * D].copy_(dv.reshape(S, D))
        qk_pre = kp["qk_pre"]
        g["norm_q"], g["norm_k"] = ops.rmsnorm_rope_bwd(qk_pre[:, :D], blk.norm_q, dq.reshape(S, D), dqkv[:, :D],
                                                        qk_pre[:, D:], blk.norm_k, dk.reshape(S, D), dqkv[:, D:2 * D],
                                                        lay.cos if lay.cos32 is None else lay.cos32,
                                                        lay.sin if lay.sin32 is None else lay.sin32, lay.rope_row, head_dim=d, eps=eps,
                                                        want_dw=need("norm_q") or need("norm_k"))
        dn1, g["w_qkv"], g["b_qkv"] = ops.linear_bwd(kp["n1"], blk.w_qkv, dqkv, need_dw=need("w_qkv"), need_db=need("b_qkv"))
        if R:
            dx, d_scale_msa, d_shift_msa = ops.layernorm_modulate_grouped_bwd(x, dn1, scale_msa, R, gin=dy, eps=eps)
        else:
            dx, d_scale_msa, d_shift_msa = ops.layernorm_modulate_bwd(x, dn1, scale=scale_msa, gin=dy, eps=eps)
        return (dx, dctx, d_shift_msa, d_scale_msa, d_gate_msa, d_cshift, d_cscale, d_cgate, None, None, None, None, None,
                *(g.get(n) if need(n) else None for n in _BLOCK_TENSORS))


def _requires_grad(*tensors) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _any_model_tensor_requires_grad(model, *inputs) -> bool:
    """Grad enabled and an input or a tensor of model.tensors() requires grad (quantised weights are not tensors)."""
    return torch.is_grad_enabled() and _requires_grad(*inputs, *(t for t in model.tensors().values()
                                                                 if isinstance(t, torch.Tensor)))


def refuse_model_grad(path: str, model, *inputs) -> None:
    """Raise FvbError when a model forward without a backward would run with grad enabled and an input or a tensor of
    model.tensors() requiring grad."""
    if _any_model_tensor_requires_grad(model, *inputs):
        raise ops.FvbError(f"{path} has no backward: run it under torch.no_grad(), or train the single-rank model "
                           "(WanDiT.forward)")


def _linear(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """ops.linear over the last axis of x; through ops.LinearFn when grad is enabled and x, w or b requires grad."""
    if not _requires_grad(x, w, b):
        return ops.linear(x, w, b)
    return ops.LinearFn.apply(x.reshape(-1, x.shape[-1]), w, b).view(*x.shape[:-1], w.shape[0])


class _GeluMlpFn(torch.autograd.Function):
    """y = fc_out(gelu_tanh(fc_in(x))) over rows of x [M, K] (the text embedder, wanvideo.py:100-135 / mlp.py:47-51): fc_in
    with its GELU epilogue on fvb_linear_bf16_aux (which also keeps the pre-GELU h), fc_out on fvb_linear_bf16, the no-grad
    calls' bits. The backward is the block feed-forward's: fc_out's weight / bias gradients on linear_bwd, dh = bf16(bf16(dy
    w_out) gelu'(h)) in one GEMM epilogue (fvb_linear_dgrad_gelu_bf16, which needs fc_out's weight, hence one Function for
    both linears), then linear_bwd of fc_in."""

    @staticmethod
    def forward(ctx, x, w_in, b_in, w_out, b_out):
        f, h = ops.linear_aux(x, w_in, b_in, ops.EPI_BIAS_GELU_TANH)
        ctx.save_for_backward(x, w_in, w_out, f, h)
        return ops.linear(f, w_out, b_out)

    @staticmethod
    def backward(ctx, dy):
        x, w_in, w_out, f, h = ctx.saved_tensors
        need_x, need_w_in, need_b_in, need_w_out, need_b_out = ctx.needs_input_grad
        dy = dy.to(torch.bfloat16).contiguous()
        _, dw_out, db_out = ops.linear_bwd(f, w_out, dy, need_dx=False, need_dw=need_w_out, need_db=need_b_out)
        dx = dw_in = db_in = None
        if need_x or need_w_in or need_b_in:
            dh = ops.linear_dgrad_gelu(dy, w_out, h)
            dx, dw_in, db_in = ops.linear_bwd(x, w_in, dh, need_dx=need_x, need_dw=need_w_in, need_db=need_b_in)
        return dx, dw_in, db_in, dw_out, db_out


class _HeadNormFn(torch.autograd.Function):
    """norm_out: n = bf16(bf16(LN(x)) (1 + scale) + shift) (ops.layernorm_modulate with round_ln, the no-grad call's bits);
    backward on fvb_layernorm_modulate_bwd (dx bf16, d_scale / d_shift fp32)."""

    @staticmethod
    def forward(ctx, x, scale, shift, eps):
        ctx.save_for_backward(x, scale)
        ctx.eps = eps
        return ops.layernorm_modulate(x, scale, shift, round_ln=True, eps=eps)

    @staticmethod
    def backward(ctx, dn):
        x, scale = ctx.saved_tensors
        dx, d_scale, d_shift = ops.layernorm_modulate_bwd(x, dn.to(torch.bfloat16).contiguous(), scale=scale, round_ln=True,
                                                          eps=ctx.eps)
        return dx, d_scale, d_shift, None


class _HeadNormFramesFn(torch.autograd.Function):
    """The causal head's norm_out with one (scale, shift) row per `rows` tokens in the bf16 modulation flow
    (ops.layernorm_modulate with round_ln, mod_rows and mod_bf16, the no-grad call's bits); backward on
    fvb_layernorm_modulate_grouped_bwd (dx bf16, d_scale / d_shift fp32 [F, D])."""

    @staticmethod
    def forward(ctx, x, scale, shift, rows, eps):
        ctx.save_for_backward(x, scale)
        ctx.rows, ctx.eps = rows, eps
        return ops.layernorm_modulate(x, scale, shift, round_ln=True, eps=eps, mod_rows=rows, mod_bf16=True)

    @staticmethod
    def backward(ctx, dn):
        x, scale = ctx.saved_tensors
        dx, d_scale, d_shift = ops.layernorm_modulate_grouped_bwd(x, dn.to(torch.bfloat16).contiguous(), scale, ctx.rows,
                                                                  eps=ctx.eps)
        return dx, d_scale, d_shift, None, None


# WanDiT's own trainable tensors (attribute name -> reference parameter name); the blocks' follow under blocks.{i}.
_MODEL_TENSORS = {
    "w_patch": "patch_embedding.proj.weight", "b_patch": "patch_embedding.proj.bias",
    "w_t1": "condition_embedder.time_embedder.mlp.fc_in.weight", "b_t1": "condition_embedder.time_embedder.mlp.fc_in.bias",
    "w_t2": "condition_embedder.time_embedder.mlp.fc_out.weight", "b_t2": "condition_embedder.time_embedder.mlp.fc_out.bias",
    "w_tm": "condition_embedder.time_modulation.linear.weight", "b_tm": "condition_embedder.time_modulation.linear.bias",
    "w_x1": "condition_embedder.text_embedder.fc_in.weight", "b_x1": "condition_embedder.text_embedder.fc_in.bias",
    "w_x2": "condition_embedder.text_embedder.fc_out.weight", "b_x2": "condition_embedder.text_embedder.fc_out.bias",
    "scale_shift_table": "scale_shift_table", "w_out": "proj_out.weight", "b_out": "proj_out.bias"}


class WanDiT:
    """WanTransformer3DModel on libfvb200: the denoising forward, and its backward when grad is enabled and latents, text or
    a tensor of tensors() requires grad (forward(..., checkpoint=True) for block activation checkpointing). The
    sequence-parallel (distributed.SPWanDiT) and causal (causal_wan.CausalWanDiT) models reuse its pieces for inference."""

    def __init__(self, cfg: WanDiTConfig, state_dict: dict, blocks: list | None = None):
        self.cfg = cfg
        sd = state_dict
        bf = lambda t: t.to(torch.bfloat16).contiguous()
        D = cfg.hidden_size
        if blocks is None:
            n_layers = 0
            while f"blocks.{n_layers}.to_q.weight" in sd:
                n_layers += 1
            blocks = [WanBlock(sd, f"blocks.{i}.", cfg) for i in range(n_layers)]
        self.blocks = blocks
        self.w_patch = bf(sd["patch_embedding.proj.weight"].reshape(D, -1))
        self.b_patch = bf(sd["patch_embedding.proj.bias"])
        ce = "condition_embedder."
        self.w_t1, self.b_t1 = bf(sd[ce + "time_embedder.mlp.fc_in.weight"]), bf(sd[ce + "time_embedder.mlp.fc_in.bias"])
        self.w_t2, self.b_t2 = bf(sd[ce + "time_embedder.mlp.fc_out.weight"]), bf(sd[ce + "time_embedder.mlp.fc_out.bias"])
        self.w_tm, self.b_tm = bf(sd[ce + "time_modulation.linear.weight"]), bf(sd[ce + "time_modulation.linear.bias"])
        self.w_x1, self.b_x1 = bf(sd[ce + "text_embedder.fc_in.weight"]), bf(sd[ce + "text_embedder.fc_in.bias"])
        self.w_x2, self.b_x2 = bf(sd[ce + "text_embedder.fc_out.weight"]), bf(sd[ce + "text_embedder.fc_out.bias"])
        self.scale_shift_table = sd["scale_shift_table"]
        self.w_out, self.b_out = bf(sd["proj_out.weight"]), bf(sd["proj_out.bias"])
        self._layouts: dict = {}

    @classmethod
    def random(cls, cfg: WanDiTConfig, device="cuda", seed: int = 2029) -> "WanDiT":
        """Synthetic random-init model of the given architecture, built layer by layer so that peak memory stays
        at one copy of the weights (30 GB for a 14B expert in bf16; with fp8_linears or int8_weights the block weights take
        half)."""
        blocks = []
        for i in range(cfg.num_layers):
            one = WanDiTConfig(**{**cfg.__dict__, "num_layers": 1})
            sd = random_state_dict(one, device, seed + 1 + i, layers=1)
            blocks.append(WanBlock(sd, "blocks.0.", cfg))
            del sd
        return cls(cfg, random_state_dict(cfg, device, seed, layers=0), blocks=blocks)

    def tensors(self) -> dict:
        """Every trainable tensor, by attribute name: the model's own (patch embedding, condition embedder, head) and each
        block's WanBlock.tensors() under "blocks.{i}.". Each is a leaf an optimizer can step; set requires_grad on the ones
        to train. to_reference_names maps this dict, or the same keys holding gradients, to the reference names."""
        out = {n: getattr(self, n) for n in _MODEL_TENSORS}
        for i, blk in enumerate(self.blocks):
            out.update({f"blocks.{i}.{n}": t for n, t in blk.tensors().items()})
        return out

    def to_reference_names(self, t: dict) -> dict:
        """{name: tensor} as tensors() returns it, or the same keys holding gradients -> {reference parameter name: tensor},
        every one a view of the given tensor in the reference's shape (w_patch [D, C * pt * ph * pw] becomes
        patch_embedding.proj.weight [D, C, pt, ph, pw]). None entries (the .grad of a tensor that is not trained) map to
        None. WanDiT(cfg, model.to_reference_names(model.tensors())) rebuilds the model."""
        out = {ref: t[n] for n, ref in _MODEL_TENSORS.items()}
        w = t["w_patch"]
        if w is not None:
            out["patch_embedding.proj.weight"] = w.view(w.shape[0], self.cfg.in_channels, *self.cfg.patch_size)
        blocks: dict = {}
        for k, v in t.items():
            if k.startswith("blocks."):
                i, n = k[len("blocks."):].split(".", 1)
                blocks.setdefault(int(i), {})[n] = v
        for i in sorted(blocks):
            out.update(WanBlock.to_reference_names(blocks[i], f"blocks.{i}.", like=self.blocks[i].tensors()))
        return out

    # ---- pieces of WanTransformer3DModel.forward ----
    def layout(self, seq_shape, device, vsa_sparsity=None) -> TokenLayout:
        key = (tuple(seq_shape), vsa_sparsity if self.cfg.vsa else None)
        if key not in self._layouts:
            self._layouts[key] = make_layout(seq_shape, self.cfg, device, key[1])
        return self._layouts[key]

    def condition(self, timestep: torch.Tensor, text: torch.Tensor):
        """WanTimeTextImageEmbedding.forward (wanvideo.py:100-135): temb [B, D], timestep_proj [B, 6, D], ctx [B, L, D]."""
        cfg = self.cfg
        half = cfg.freq_dim // 2
        # timestep_embedding, fastvideo/layers/visual_embedding.py:137-158 (fp32, cos | sin)
        if getattr(self, "_t_freqs", None) is None or self._t_freqs.device != timestep.device:
            # computed on the host exactly as the reference does, uploaded once (a pageable H2D copy cannot be captured)
            self._t_freqs = torch.exp(-math.log(10000) * torch.arange(0, half, dtype=torch.float32) / half).to(timestep.device)
        freqs = self._t_freqs
        args = timestep[:, None].float() * freqs[None]
        t_freq = torch.cat([torch.cos(args), torch.sin(args)], dim=-1).to(torch.bfloat16)
        h = _linear(t_freq, self.w_t1, self.b_t1)
        temb = _linear(torch.nn.functional.silu(h), self.w_t2, self.b_t2)          # [B, D]
        tproj = _linear(torch.nn.functional.silu(temb), self.w_tm, self.b_tm)       # [B, 6D]
        if _requires_grad(text, self.w_x1, self.b_x1, self.w_x2, self.b_x2):
            ctx = _GeluMlpFn.apply(text.reshape(-1, text.shape[-1]), self.w_x1, self.b_x1, self.w_x2,
                                   self.b_x2).view(*text.shape[:-1], -1)
        else:
            ctx = ops.linear(ops.linear(text, self.w_x1, self.b_x1, ops.EPI_BIAS_GELU_TANH), self.w_x2, self.b_x2)
        return temb, tproj.unflatten(1, (6, -1)), ctx

    def patches(self, latents: torch.Tensor) -> torch.Tensor:
        """[B, C, T, H, W] -> [B, S, C*pt*ph*pw]: the (c, pt, ph, pw) patches of every token, in raster order."""
        B, C, T, Hh, Ww = latents.shape
        pt, ph, pw = self.cfg.patch_size
        x = latents.view(B, C, T // pt, pt, Hh // ph, ph, Ww // pw, pw).permute(0, 2, 4, 6, 1, 3, 5, 7)
        return x.reshape(B, -1, C * pt * ph * pw)

    def patchify(self, latents: torch.Tensor, lay: TokenLayout) -> torch.Tensor:
        """[B, C, T, H, W] -> [B, S, D]: Conv3d(kernel = stride = patch) as a GEMM over (c, pt, ph, pw) patches
        (fastvideo/layers/visual_embedding.py:47-55; wanvideo.py:689-690), tokens emitted in layout order."""
        x = self.patches(latents)
        if lay.perm is not None:
            x = x[:, lay.perm]
        return _linear(x.contiguous(), self.w_patch, self.b_patch)

    def head(self, x: torch.Tensor, temb: torch.Tensor, lay: TokenLayout, batch_index: int = 0) -> torch.Tensor:
        """norm_out + proj_out for one sample (wanvideo.py:746-759). x: [S, D] -> [S, C*pt*ph*pw]."""
        D = self.cfg.hidden_size
        e = self.scale_shift_table + temb[batch_index:batch_index + 1].unsqueeze(1)  # [1, 2, D], parameter dtype
        shift = e[:, 0].reshape(D).float().contiguous()
        # (1.0 + scale) is evaluated in e's dtype (bf16) before it meets the fp32 LN output (layernorm.py:262-268):
        # scale' = bf16(1 + scale) - 1 is exact in fp32 and makes the kernel's fp32 (1 + scale') equal to it
        scale = ((1.0 + e[:, 1]).float() - 1.0).reshape(D).contiguous()
        if _requires_grad(x, scale, shift):
            n = _HeadNormFn.apply(x, scale, shift, self.cfg.eps)
        else:
            n = ops.layernorm_modulate(x, scale, shift, round_ln=True, eps=self.cfg.eps)
        return _linear(n, self.w_out, self.b_out)

    def unpatchify(self, y: torch.Tensor, lay: TokenLayout) -> torch.Tensor:
        """[B, S, C*pt*ph*pw] (layout order) -> [B, C, T, H, W] (wanvideo.py:761-764)."""
        B = y.shape[0]
        if lay.inv_perm is not None:
            y = y[:, lay.inv_perm]
        T, Hh, Ww = lay.seq_shape
        pt, ph, pw = self.cfg.patch_size
        y = y.reshape(B, T, Hh, Ww, pt, ph, pw, -1).permute(0, 7, 1, 4, 2, 5, 3, 6)
        return y.flatten(6, 7).flatten(4, 5).flatten(2, 3)

    def forward(self, latents: torch.Tensor, text: torch.Tensor, timestep: torch.Tensor,
                vsa_sparsity: float | None = None, checkpoint: bool = False) -> torch.Tensor:
        """latents [B, C, T, H, W] bf16, text [B, L, text_dim] bf16, timestep [B] -> noise prediction, same shape.
        Differentiable in latents, text and every tensor of tensors() when grad is enabled and one of them requires grad
        (the output is the same bits as without grad); otherwise the plain inference calls. checkpoint: under grad, each
        block keeps only its input, its modulation and its self-attention results (block_forward)."""
        cfg = self.cfg
        if not latents.is_cuda:
            raise ops.FvbError("WanDiT.forward needs CUDA tensors (there is no CPU fallback)")
        if _any_model_tensor_requires_grad(self, latents, text):
            for blk in self.blocks:  # refused before anything runs, even when only the model's own tensors require grad
                _require_trainable(blk, cfg)
        B = latents.shape[0]
        pt, ph, pw = cfg.patch_size
        seq_shape = (latents.shape[2] // pt, latents.shape[3] // ph, latents.shape[4] // pw)
        lay = self.layout(seq_shape, latents.device, vsa_sparsity if cfg.vsa else None)
        temb, tproj, ctx = self.condition(timestep, text)
        x = self.patchify(latents.to(torch.bfloat16), lay)
        outs = []
        for b in range(B):
            xb = x[b]
            for blk in self.blocks:
                xb = block_forward(xb, blk, ctx[b], tproj[b:b + 1], lay, cfg, checkpoint)
            outs.append(self.head(xb, temb, lay, b))
        return self.unpatchify(torch.stack(outs, 0), lay)
