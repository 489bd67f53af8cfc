"""Host-side mirror of the reference's attention plug-in interfaces, on top of libfvb200.

The reference selects attention through `AttentionBackend` subclasses (fastvideo/attention/backends/abstract.py:31-194):
static get_name / get_impl_cls / get_metadata_cls / get_builder_cls, an `AttentionImpl` with
preprocess_qkv -> forward -> postprocess_output on [B, S, H_local, d] tensors, and per-step metadata built by an
`AttentionMetadataBuilder` and delivered through the forward context (fastvideo/attention/layer.py:62-79, 134-158;
fastvideo/pipelines/stages/denoising.py:466-482). The classes below have the same names, methods, argument
meaning and error behaviour; INTEGRATION.md shows the few lines that register them inside a FastVideo checkout
(subclassing the real ABCs there). They are usable stand-alone as well (tests/, bench.py).

Kernel-package level entry points (fastvideo-kernel/python/fastvideo_kernel/__init__.py:1-62) are mirrored too:
video_sparse_attn (fastvideo_b200/vsa.py), block_sparse_attn_from_indices and sliding_tile_attention (here).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any

import torch

from . import ops, vsa

VSA_TILE_SIZE = (4, 4, 4)  # fastvideo/attention/backends/video_sparse_attn.py:29


# ----------------------------------------------------------------------------------------------------- dense (SDPA)
@dataclass
class B200AttentionMetadata:
    """SDPAMetadata (fastvideo/attention/backends/sdpa.py:40-67): current_timestep and an optional boolean mask.
    Arbitrary dense masks are not a Wan hot-path input; block structure is expressed with block lists instead."""
    current_timestep: int = 0
    attn_mask: torch.Tensor | None = None


class B200AttentionMetadataBuilder:
    def prepare(self) -> None:
        pass

    def build(self, current_timestep: int = 0, attn_mask: torch.Tensor | None = None, **kwargs) -> B200AttentionMetadata:
        return B200AttentionMetadata(current_timestep, attn_mask)


class B200AttentionImpl:
    """SDPAImpl (sdpa.py:106-147): forward(q, k, v, attn_metadata) on [B, S, H, d] -> [B, S, H, d]."""

    def __init__(self, num_heads: int, head_size: int, causal: bool = False, softmax_scale: float | None = None,
                 num_kv_heads: int | None = None, prefix: str = "", **extra_impl_args) -> None:
        if causal:
            raise NotImplementedError("causal attention is not part of the Wan bidirectional hot path")
        if head_size != 128:
            raise ValueError(f"libfvb200 attention supports head_size 128, got {head_size}")
        self.softmax_scale = softmax_scale if softmax_scale is not None else head_size ** -0.5

    def preprocess_qkv(self, qkv: torch.Tensor, attn_metadata) -> torch.Tensor:
        return qkv

    def postprocess_output(self, output: torch.Tensor, attn_metadata) -> torch.Tensor:
        return output

    def forward(self, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, attn_metadata=None) -> torch.Tensor:
        if attn_metadata is not None and getattr(attn_metadata, "attn_mask", None) is not None:
            raise NotImplementedError("dense boolean masks: use block lists (block_sparse_attn_from_indices / STA)")
        if torch.is_grad_enabled() and (query.requires_grad or key.requires_grad or value.requires_grad):
            return _DenseAttnFn.apply(query, key, value, self.softmax_scale)
        return ops.attention(query, key, value, softmax_scale=self.softmax_scale)


class B200Attention8bitImpl(B200AttentionImpl):
    """B200AttentionImpl on the 8-bit attention (INT8 Q K^T, FP8 P V): q, k, v are quantised per call
    (ops.quantize_attention_8bit), then ops.attention_8bit."""

    def forward(self, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, attn_metadata=None) -> torch.Tensor:
        if attn_metadata is not None and getattr(attn_metadata, "attn_mask", None) is not None:
            raise NotImplementedError("dense boolean masks: use block lists (block_sparse_attn_from_indices / STA)")
        return ops.attention_8bit(ops.quantize_attention_8bit(query, key, value), self.softmax_scale)


class B200AttentionBackend:
    accept_output_buffer: bool = True

    @staticmethod
    def get_supported_head_sizes() -> list[int]:
        return [128]

    @staticmethod
    def get_name() -> str:
        return "FVB200_ATTN"  # distinct name; plugin.install() adds the enum member (platforms/interface.py:13-27)

    @staticmethod
    def get_impl_cls():
        return B200AttentionImpl

    @staticmethod
    def get_metadata_cls():
        return B200AttentionMetadata

    @staticmethod
    def get_builder_cls():
        return B200AttentionMetadataBuilder


# ----------------------------------------------------------------------------------------------------- VSA backend
@dataclass
class VideoSparseAttentionMetadata:
    """Same fields as the reference's dataclass (video_sparse_attn.py:139-158) + the compact-layout tables."""
    current_timestep: int
    dit_seq_shape: list[int]
    VSA_sparsity: float
    num_tiles: list[int]
    total_seq_length: int
    tile_partition_indices: torch.Tensor
    reverse_tile_partition_indices: torch.Tensor
    variable_block_sizes: torch.Tensor
    non_pad_index: torch.Tensor
    untile_combined_index: torch.Tensor
    block_offsets: torch.Tensor = None      # int32 [n_tiles + 1]: first row of each tile in compact tile-major order
    row_block: torch.Tensor = None          # int32 [S]: compact row -> tile
    tile_buf: torch.Tensor | None = None
    cache_tile_buf: bool = True


_TABLE_CACHE: dict = {}


class VideoSparseAttentionMetadataBuilder:
    """build(current_timestep, raw_latent_shape, patch_size, VSA_sparsity, device) -- video_sparse_attn.py:192-235.
    The tables come from one CUDA kernel (fvb_vsa_tile_index) instead of a Python triple loop, cached per shape."""

    def __init__(self) -> None:
        pass

    def prepare(self) -> None:
        pass

    def build(self, current_timestep: int, raw_latent_shape: tuple[int, int, int], patch_size: tuple[int, int, int],
              VSA_sparsity: float, device: torch.device, cache_tile_buf: bool = True, **kwargs: dict[str, Any]):
        dit_seq_shape = tuple(raw_latent_shape[i] // patch_size[i] for i in range(3))
        num_tiles = tuple(math.ceil(dit_seq_shape[i] / VSA_TILE_SIZE[i]) for i in range(3))
        key = (dit_seq_shape, str(device))
        if key not in _TABLE_CACHE:
            t = ops.vsa_tile_index(dit_seq_shape, VSA_TILE_SIZE, device=device)
            t["row_block"] = torch.repeat_interleave(
                torch.arange(t["variable_block_sizes"].numel(), device=device, dtype=torch.int32),
                t["variable_block_sizes"].long())
            _TABLE_CACHE[key] = t
        t = _TABLE_CACHE[key]
        return VideoSparseAttentionMetadata(
            current_timestep=current_timestep, dit_seq_shape=list(dit_seq_shape), VSA_sparsity=VSA_sparsity,
            num_tiles=list(num_tiles), total_seq_length=math.prod(dit_seq_shape),
            tile_partition_indices=t["tile_partition"], reverse_tile_partition_indices=t["reverse_partition"],
            variable_block_sizes=t["variable_block_sizes"], non_pad_index=t["non_pad"],
            untile_combined_index=t["untile_combined"], block_offsets=t["block_offsets"], row_block=t["row_block"],
            cache_tile_buf=cache_tile_buf)


def compute_topk(sparsity: float, num_blocks: int) -> int:
    """video_sparse_attn.py:161-163."""
    return max(1, min(math.ceil((1 - sparsity) * num_blocks), num_blocks))


class _PermuteRowsFn(torch.autograd.Function):
    """ops.gather_rows of [B, S, W] rows by a permutation table; the backward gathers the gradient with the inverse table."""

    @staticmethod
    def forward(ctx, x, idx, inv):
        ctx.save_for_backward(inv)
        return ops.gather_rows(x, idx)

    @staticmethod
    def backward(ctx, g):
        inv, = ctx.saved_tensors
        return ops.gather_rows(g.to(torch.bfloat16).contiguous(), inv), None, None


class VideoSparseAttentionImpl:
    """VideoSparseAttentionImpl (video_sparse_attn.py:238-342). preprocess_qkv tiles the stacked [4B, S, H, d] tensor,
    forward runs VSA, postprocess_output untiles. Here "tiling" is a pure permutation into COMPACT tile-major order
    (no zero-padded rows: the kernels mask by variable block size), done by one gather kernel.
    Differentiable: with grad enabled and an input that requires grad, tile / untile are autograd permutations (the
    backward gathers with the inverse table) and forward runs vsa._VideoSparseAttnFn in the compact layout, whose output
    is the no-grad call's, bit for bit."""

    def __init__(self, num_heads: int, head_size: int, causal: bool = False, softmax_scale: float | None = None,
                 num_kv_heads: int | None = None, prefix: str = "", **extra_impl_args) -> None:
        if head_size != 128:
            raise ValueError(f"libfvb200 VSA supports head_size 128, got {head_size}")
        self.prefix = prefix

    @staticmethod
    def _permute(x: torch.Tensor, idx: torch.Tensor, inv: torch.Tensor) -> torch.Tensor:
        B, S, H, d = x.shape
        x3 = x.reshape(B, S, H * d)
        if torch.is_grad_enabled() and x.requires_grad:
            return _PermuteRowsFn.apply(x3, idx, inv).view(B, S, H, d)
        return ops.gather_rows(x3, idx).view(B, S, H, d)

    def tile(self, x: torch.Tensor, md: VideoSparseAttentionMetadata) -> torch.Tensor:
        return self._permute(x, md.tile_partition_indices, md.reverse_tile_partition_indices)

    def untile(self, x: torch.Tensor, md: VideoSparseAttentionMetadata) -> torch.Tensor:
        return self._permute(x, md.reverse_tile_partition_indices, md.tile_partition_indices)

    def preprocess_qkv(self, qkv: torch.Tensor, attn_metadata: VideoSparseAttentionMetadata) -> torch.Tensor:
        return self.tile(qkv, attn_metadata)

    def postprocess_output(self, output: torch.Tensor, attn_metadata: VideoSparseAttentionMetadata) -> torch.Tensor:
        return self.untile(output, attn_metadata)

    def forward(self, query: torch.Tensor, key: torch.Tensor, value: torch.Tensor, gate_compress: torch.Tensor,
                attn_metadata: VideoSparseAttentionMetadata) -> torch.Tensor:
        md = attn_metadata
        topk = compute_topk(md.VSA_sparsity, md.variable_block_sizes.numel())
        inputs = (query, key, value) if gate_compress is None else (query, key, value, gate_compress)
        if torch.is_grad_enabled() and any(t.requires_grad for t in inputs):
            return vsa._VideoSparseAttnFn.apply(query, key, value, gate_compress, md.variable_block_sizes, topk, None,
                                                md.block_offsets, md.row_block)
        return vsa.video_sparse_attn_bshd(query, key, value, md.variable_block_sizes, topk, gate=gate_compress,
                                          block_off=md.block_offsets, row_block=md.row_block)


class VideoSparseAttentionBackend:
    accept_output_buffer: bool = True

    @staticmethod
    def get_supported_head_sizes() -> list[int]:
        return [128]

    @staticmethod
    def get_name() -> str:
        return "VIDEO_SPARSE_ATTN"  # must equal the enum member (attention/layer.py:78; wanvideo.py:628-629)

    @staticmethod
    def get_impl_cls():
        return VideoSparseAttentionImpl

    @staticmethod
    def get_metadata_cls():
        return VideoSparseAttentionMetadata

    @staticmethod
    def get_builder_cls():
        return VideoSparseAttentionMetadataBuilder


# ----------------------------------------------------------------------------------------------------- kernel-package API
def _lists_to_map(q2k_idx: torch.Tensor, q2k_num: torch.Tensor, nkv: int) -> torch.Tensor:
    valid = torch.arange(q2k_idx.shape[-1], device=q2k_idx.device)[None, None, None, :] < q2k_num[..., None]
    bmap = torch.zeros((*q2k_idx.shape[:3], nkv + 1), dtype=torch.bool, device=q2k_idx.device)
    bmap.scatter_(3, torch.where(valid, q2k_idx, nkv).long(), True)
    return bmap[..., :nkv]


def _usable_strides(t: torch.Tensor) -> bool:
    """True when the attention kernels can read t ([B, S, H, 128]) in place: unit channel stride, (b, s, h) strides that are
    non-zero multiples of 8 (TMA), a 16-byte aligned base."""
    return t.stride(3) == 1 and all(s != 0 and s % 8 == 0 for s in t.stride()[:3]) and t.data_ptr() % 16 == 0


class _DenseAttnFn(torch.autograd.Function):
    """Dense attention on [B, S, H, 128] views: forward on fvb_attention_fwd (the output is the no-grad call's, bit for bit),
    backward on fvb_attention_bwd -- what the reference's FlashAttention / SDPA backends give autograd."""

    @staticmethod
    def forward(ctx, q, k, v, softmax_scale):
        out, lse = ops.attention(q, k, v, softmax_scale=softmax_scale, return_lse=True)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.softmax_scale = softmax_scale
        return out

    @staticmethod
    def backward(ctx, grad_o):
        q, k, v, out, lse = ctx.saved_tensors
        go = grad_o.to(torch.bfloat16)
        if not _usable_strides(go):
            go = go.contiguous()
        dq, dk, dv = ops.attention_bwd(q, k, v, out, lse, go, softmax_scale=ctx.softmax_scale)
        return dq, dk, dv, None


class _BlockSparseAttnFn(torch.autograd.Function):
    """Forward on fvb_attention_blocklist_fwd, backward on fvb_attention_blocklist_bwd -- the autograd pair the reference
    registers for its custom op (block_sparse_attn.py:217-243)."""

    @staticmethod
    def forward(ctx, q, k, v, q2k_idx, q2k_num, vbs):
        out = torch.empty_like(q)
        o, lse = ops.attention_blocklist(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), q2k_idx, q2k_num,
                                         out=out.transpose(1, 2), return_lse=True, kv_len=vbs, nkb=k.shape[2] // 64)
        ctx.save_for_backward(q, k, v, out, lse, q2k_idx, q2k_num, vbs)
        ctx.mark_non_differentiable(lse)
        return out, lse

    @staticmethod
    def backward(ctx, grad_o, grad_lse):
        q, k, v, out, lse, q2k_idx, q2k_num, vbs = ctx.saved_tensors
        nkv = k.shape[2] // 64
        # inverse lists (kv block -> the q blocks that selected it, ascending): the transposed block map through the same
        # ordered-compaction kernel as the forward lists (the reference: triton_kernels/index.py:147-250 invert_indices)
        k2q_idx, k2q_num = ops.map_to_index(_lists_to_map(q2k_idx, q2k_num, nkv).transpose(-1, -2).contiguous())
        go = grad_o.to(torch.bfloat16).contiguous()
        dq, dk, dv = ops.attention_blocklist_bwd(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), out.transpose(1, 2), lse,
                                                 go.transpose(1, 2), q2k_idx, q2k_num, k2q_idx, k2q_num, kv_len=vbs)
        return dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2), None, None, None


def block_sparse_attn_from_indices(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q2k_idx: torch.Tensor,
                                   q2k_num: torch.Tensor, variable_block_sizes: torch.Tensor):
    """block_sparse_attn_from_indices(q, k, v, q2k_idx, q2k_num, vbs) -> (o, lse) on [B, H, S_pad, 128] tensors, with
    autograd (fastvideo-kernel/python/fastvideo_kernel/block_sparse_attn.py:347-393; sm100a contract
    fastvideo-kernel/csrc/attention/block_sparse_sm100a.cu:53-114). q2k_idx int32 [B, H, nq, nkv] (first q2k_num
    entries valid), LSE = max(qk*scale*log2e) + log2(sum), rows with count 0 -> zeros."""
    if q.dtype != torch.bfloat16 or q2k_idx.dtype != torch.int32 or q2k_num.dtype != torch.int32:
        raise ValueError("expected bf16 q/k/v and int32 indices")
    B, H, S, d = q.shape
    if d != 128 or S % 64 != 0 or k.shape[2] % 64 != 0:
        raise ValueError("head_dim must be 128 and sequence lengths multiples of 64")
    return _BlockSparseAttnFn.apply(q, k, v, q2k_idx.contiguous(), q2k_num.contiguous(), variable_block_sizes.to(torch.int32))


def sliding_tile_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, window_size: list, text_length: int = 0,
                           has_text: bool = False, seq_shape: str = "30x48x80", tile_size=(6, 8, 8)) -> torch.Tensor:
    """sliding_tile_attention(q, k, v, window_size per head, text_length, has_text, seq_shape)
    (fastvideo-kernel/python/fastvideo_kernel/ops.py:21-62) on [B, H, S, 128] tensors in tile-major token order.
    window_size[h] = (t, h, w) in tiles; seq_shape "TxHxW" is the token canvas; tiles of tile_size tokens
    (6x8x8 = 384 for the reference kernel; any tile volume that is a multiple of 64 works here)."""
    if has_text or text_length:
        raise NotImplementedError("text tokens in STA are not used by the Wan pipelines")
    T, Hh, Ww = (int(s) for s in seq_shape.split("x"))
    ct, ch, cw = T // tile_size[0], Hh // tile_size[1], Ww // tile_size[2]
    vol = math.prod(tile_size)
    if vol % 64 != 0 or q.shape[2] != ct * ch * cw * vol:
        raise ValueError("tile volume must be a multiple of 64 and the sequence must cover the canvas")
    B, H, S, d = q.shape
    sub = vol // 64
    tmap = ops.sta_map((ct, ch, cw), [tuple(w) for w in window_size], device=q.device)       # [H, n_tiles, n_tiles]
    bmap = tmap.repeat_interleave(sub, 1).repeat_interleave(sub, 2)                           # 64-token block map
    sched, cnt = ops.pair_schedule(bmap.unsqueeze(0))
    out = torch.empty_like(q)
    ops.attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), out=out.transpose(1, 2), sched=sched,
                  sched_cnt=cnt, nqb=S // 64, nkb=S // 64)
    return out
