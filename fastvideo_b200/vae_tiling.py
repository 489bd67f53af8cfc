"""Tiled VAE decode: the host-side tile loop and seam blending of ParallelTiledVAE
(fastvideo/models/vaes/common.py:77-92 decode dispatch, :94-113 blend_v/h/t, :162-264 parallel_tiled_decode,
:266-277 _merge_spatial_tiles, :279-313 spatial_tiled_decode, :349-374 tiled_decode), written against a `decode_fn`
callback for the per-tile decoder ([B, C, T, h, w] -> [B, 3, 4(T-1)+1, 8h, 8w]).

Where the reference uses it: `ParallelTiledVAE.decode` is what a VAE's decode falls through to when its feature cache is
off; for Wan the cache is ON by default (fastvideo/configs/models/vaes/wanvae.py:73), so the default Wan decode is the
un-tiled per-latent-frame loop that fastvideo_b200/wan_vae.py implements, and at the shapes in BASELINE.json the
un-tiled decode fits in the 80 GB of an H100. This module is the multi-GPU / memory-bounded variant of row a21 (tiles dealt to ranks, one
all_gather, blended seams). Its caller is fastvideo_b200.wan_vae.WanVAEDecoder.decode_tiled, which supplies the cache-less
per-tile decoder (AutoencoderKLWan._decode: 4T frames per tile) and Wan's wrappers around these methods (wanvae.py:1228-1247:
`blend_num_frames *= 2` on the temporal paths, first three frames of every tiled result dropped).

The tile arithmetic and the blend order follow the reference; the blends are vectorised (one pass per seam instead of one
per seam row) with the same rounding points. tests/test_vae_tiling_cpu.py pins the result bit-exactly, in fp32 and bf16,
against outputs of the reference's own ParallelTiledVAE methods (oracle/gen_golden.py `tiling`).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable

import torch


@dataclass
class TilingConfig:
    """fastvideo/configs/models/vaes/base.py:29-46 plus the two compression ratios of the Wan VAE."""
    tile_sample_min_height: int = 256
    tile_sample_min_width: int = 256
    tile_sample_min_num_frames: int = 16
    tile_sample_stride_height: int = 192
    tile_sample_stride_width: int = 192
    tile_sample_stride_num_frames: int = 12
    blend_num_frames: int | None = None  # default: min - stride (base.py:46)
    use_tiling: bool = True
    use_temporal_tiling: bool = True
    use_parallel_tiling: bool = True
    spatial_compression_ratio: int = 8
    temporal_compression_ratio: int = 4

    def __post_init__(self):
        if self.blend_num_frames is None:
            self.blend_num_frames = self.tile_sample_min_num_frames - self.tile_sample_stride_num_frames


# ---- seam blends (common.py:94-113) ----
def _blend(a: torch.Tensor, b: torch.Tensor, blend_extent: int, dim: int) -> torch.Tensor:
    """b[..., i, ...] <- a[..., -E + i, ...] * (1 - i/E) + b[..., i, ...] * (i/E) for i < E along `dim`, in place on b.
    The reference loops over i with python-float weights; one vectorised pass gives the same bits: the weights are formed
    in float64 and rounded to fp32 (what a python scalar becomes inside the op), each product is rounded to the tensors'
    dtype and so is the sum -- three launches per seam instead of three per row of the seam."""
    E = min(a.shape[dim], b.shape[dim], blend_extent)
    if E <= 0:
        return b
    w = torch.arange(E, dtype=torch.float64, device=b.device) / E
    shape = [1] * b.dim()
    shape[dim] = E
    wb = w.to(torch.float32).view(shape)
    wa = (1.0 - w).to(torch.float32).view(shape)
    ta = (a.narrow(dim, a.shape[dim] - E, E).float() * wa).to(b.dtype)
    head = b.narrow(dim, 0, E)
    tb = (head.float() * wb).to(b.dtype)
    head.copy_(ta + tb)
    return b


def blend_v(a: torch.Tensor, b: torch.Tensor, blend_extent: int) -> torch.Tensor:
    return _blend(a, b, blend_extent, -2)


def blend_h(a: torch.Tensor, b: torch.Tensor, blend_extent: int) -> torch.Tensor:
    return _blend(a, b, blend_extent, -1)


def blend_t(a: torch.Tensor, b: torch.Tensor, blend_extent: int) -> torch.Tensor:
    return _blend(a, b, blend_extent, -3)


def merge_spatial_tiles(tiles, blend_height: int, blend_width: int, stride_height: int, stride_width: int) -> torch.Tensor:
    """common.py:266-277: blend each tile with the one above and the one to its left, crop to the stride, concatenate."""
    result_rows = []
    for i, row in enumerate(tiles):
        result_row = []
        for j, tile in enumerate(row):
            if i > 0:
                tile = blend_v(tiles[i - 1][j], tile, blend_height)
            if j > 0:
                tile = blend_h(row[j - 1], tile, blend_width)
            result_row.append(tile[:, :, :, :stride_height, :stride_width])
        result_rows.append(torch.cat(result_row, dim=-1))
    return torch.cat(result_rows, dim=-2)


def _latent_tile_dims(cfg: TilingConfig):
    s, t = cfg.spatial_compression_ratio, cfg.temporal_compression_ratio
    return (cfg.tile_sample_min_height // s, cfg.tile_sample_min_width // s, cfg.tile_sample_min_num_frames // t,
            cfg.tile_sample_stride_height // s, cfg.tile_sample_stride_width // s, cfg.tile_sample_stride_num_frames // t)


def spatial_tiled_decode(z: torch.Tensor, decode_fn: Callable, cfg: TilingConfig) -> torch.Tensor:
    """common.py:279-313."""
    _, _, _, height, width = z.shape
    min_h, min_w, _, stride_h, stride_w, _ = _latent_tile_dims(cfg)
    blend_height = cfg.tile_sample_min_height - cfg.tile_sample_stride_height
    blend_width = cfg.tile_sample_min_width - cfg.tile_sample_stride_width
    rows = []
    for i in range(0, height, stride_h):
        row = []
        for j in range(0, width, stride_w):
            row.append(decode_fn(z[:, :, :, i:i + min_h, j:j + min_w]))
        rows.append(row)
    return merge_spatial_tiles(rows, blend_height, blend_width, cfg.tile_sample_stride_height, cfg.tile_sample_stride_width)


def tiled_decode(z: torch.Tensor, decode_fn: Callable, cfg: TilingConfig, spatial_fn: Callable | None = None) -> torch.Tensor:
    """common.py:349-374: temporal tiles of min+1 latent frames (the first decoded frame of every later tile is dropped),
    each decoded whole or spatially tiled, blended over blend_num_frames, cropped to the temporal stride. `spatial_fn`
    stands for `self.spatial_tiled_decode`, which a subclass may override: AutoencoderKLWan's version also drops the first
    temporal_compression_ratio - 1 frames of every spatially tiled temporal tile (wanvae.py:1235-1239)."""
    min_h, min_w, min_t, _, _, stride_t = _latent_tile_dims(cfg)
    num_frames = z.shape[2]
    row = []
    for i in range(0, num_frames, stride_t):
        tile = z[:, :, i:i + min_t + 1, :, :]
        if cfg.use_tiling and (tile.shape[-1] > min_w or tile.shape[-2] > min_h):
            decoded = spatial_fn(tile) if spatial_fn is not None else spatial_tiled_decode(tile, decode_fn, cfg)
        else:
            decoded = decode_fn(tile)
        if i > 0:
            decoded = decoded[:, :, 1:, :, :]
        row.append(decoded)
    result_row = []
    for i, tile in enumerate(row):
        if i > 0:
            tile = blend_t(row[i - 1], tile, cfg.blend_num_frames)
            result_row.append(tile[:, :, :cfg.tile_sample_stride_num_frames, :, :])
        else:
            result_row.append(tile[:, :, :cfg.tile_sample_stride_num_frames + 1, :, :])
    return torch.cat(result_row, dim=2)


def parallel_tile_plan(shape, cfg: TilingConfig, world: int):
    """Tile grid and the contiguous range of tile indices per rank (common.py:170-192). Returns (num_t, num_h, num_w,
    [(start, end) per rank]); global index = (t * num_h + h) * num_w + w."""
    _, _, T, H, W = shape
    _, _, _, stride_h, stride_w, stride_t = _latent_tile_dims(cfg)
    num_t = (T + stride_t - 1) // stride_t
    num_h = (H + stride_h - 1) // stride_h
    num_w = (W + stride_w - 1) // stride_w
    total = num_t * num_h * num_w
    per_rank = (total + world - 1) // world
    return num_t, num_h, num_w, [(min(r * per_rank, total), min((r + 1) * per_rank, total)) for r in range(world)]


def parallel_tiled_decode(z: torch.Tensor, decode_fn: Callable, cfg: TilingConfig, rank: int = 0, world: int = 1,
                          group=None) -> torch.Tensor:
    """common.py:162-264: spatio-temporal tiles dealt to the ranks in contiguous index ranges, decoded locally, gathered
    (one padded all_gather of the flattened tiles + their shapes), then merged exactly like the serial path. Every rank
    returns the full video. With world == 1 no collective is issued."""
    import torch.distributed as dist
    min_h, min_w, min_t, stride_h, stride_w, stride_t = _latent_tile_dims(cfg)
    blend_height = cfg.tile_sample_min_height - cfg.tile_sample_stride_height
    blend_width = cfg.tile_sample_min_width - cfg.tile_sample_stride_width
    num_t, num_h, num_w, ranges = parallel_tile_plan(z.shape, cfg, world)
    spatial = num_h * num_w

    def coords(g):
        return g // spatial, (g % spatial) // num_w, (g % spatial) % num_w

    local, shapes = [], []
    for g in range(*ranges[rank]):
        t_idx, h_idx, w_idx = coords(g)
        t0, h0, w0 = t_idx * stride_t, h_idx * stride_h, w_idx * stride_w
        tile = decode_fn(z[:, :, t0:t0 + min_t + 1, h0:h0 + min_h, w0:w0 + min_w])
        if t0 > 0:
            tile = tile[:, :, 1:, :, :]
        shapes.append(tuple(tile.shape))
        local.append(tile.reshape(-1))
    data = [[[None for _ in range(num_w)] for _ in range(num_h)] for _ in range(num_t)]
    # The reference stages the tiles in a torch.zeros(...) buffer of the DEFAULT dtype (common.py:216-217), i.e. float32:
    # on this path the seams are blended in fp32 and the result is fp32 whatever the decoder's dtype. Mirrored here.
    if world == 1:
        for g, (flat, shp) in enumerate(zip(local, shapes)):
            t_idx, h_idx, w_idx = coords(g)
            data[t_idx][h_idx][w_idx] = flat.float().reshape(shp)
    else:
        flat = torch.cat(local, dim=0).contiguous() if local else z.new_zeros(0)
        size = torch.tensor([flat.numel()], device=flat.device, dtype=torch.int64)
        sizes = [torch.zeros_like(size) for _ in range(world)]
        dist.all_gather(sizes, size, group=group)
        max_size = max(int(s.item()) for s in sizes)
        padded = torch.zeros(max_size, device=flat.device, dtype=torch.float32)
        padded[:flat.numel()] = flat
        gathered = torch.zeros(world * max_size, device=flat.device, dtype=torch.float32)
        dist.all_gather_into_tensor(gathered, padded, group=group)
        all_shapes = [None] * world
        dist.all_gather_object(all_shapes, shapes, group=group)
        g = 0
        for r in range(world):
            off = 0
            for shp in all_shapes[r]:
                n = 1
                for v in shp:
                    n *= v
                t_idx, h_idx, w_idx = coords(g)
                data[t_idx][h_idx][w_idx] = gathered[r * max_size + off:r * max_size + off + n].reshape(shp)
                off += n
                g += 1
    slices, last = [], None
    for i, tem in enumerate(data):
        cur = merge_spatial_tiles(tem, blend_height, blend_width, cfg.tile_sample_stride_height, cfg.tile_sample_stride_width)
        if i > 0:
            cur = blend_t(last, cur, cfg.blend_num_frames)
            slices.append(cur[:, :, :cfg.tile_sample_stride_num_frames, :, :])
        else:
            slices.append(cur[:, :, :cfg.tile_sample_stride_num_frames + 1, :, :])
        last = cur
    return torch.cat(slices, dim=2)


def decode(z: torch.Tensor, decode_fn: Callable, cfg: TilingConfig, rank: int = 0, world: int = 1, group=None) -> torch.Tensor:
    """ParallelTiledVAE.decode (common.py:77-92): choose parallel / temporal / spatial tiling or the plain decode, and trim
    to (T - 1) * temporal_ratio + 1 frames."""
    _, _, num_frames, height, width = z.shape
    min_h, min_w, min_t, _, _, _ = _latent_tile_dims(cfg)
    num_sample_frames = (num_frames - 1) * cfg.temporal_compression_ratio + 1
    if cfg.use_tiling and cfg.use_parallel_tiling and world > 1:
        return parallel_tiled_decode(z, decode_fn, cfg, rank, world, group)[:, :, :num_sample_frames]
    if cfg.use_tiling and cfg.use_temporal_tiling and num_frames > min_t:
        return tiled_decode(z, decode_fn, cfg)[:, :, :num_sample_frames]
    if cfg.use_tiling and (width > min_w or height > min_h):
        return spatial_tiled_decode(z, decode_fn, cfg)[:, :, :num_sample_frames]
    return decode_fn(z)[:, :, :num_sample_frames]
