"""Spatial tile driver — the tile loop of /root/reference/inference_upscale_a_video.py:200-304 (SURVEY.md §8f rank 2) as a
plan + executor, so that large frames can be dealt to GPUs tile by tile.

`plan_tiles` reproduces the reference geometry exactly (tiles of `tile_size` plus `overlap` LR pixels of context on every
side, the last row / column merged into its neighbour when the remainder is <= overlap, hard paste of the central region,
no blending); it is pinned by `tests/golden/tiles.json`, which is produced by EXECUTING the reference's own loop
(`oracle/make_golden_tiles.py`).  `upscale_tiled` runs the pipeline per tile; `iter_upscale_tiled` samples every tile
first, then decodes and pastes 3 frames at a time, so that the output never exists for the whole clip at once.  With
torch.distributed initialised, tiles are dealt round-robin to ranks (each tile is an independent pipeline run: no per-step
collective at all) and the pasted outputs are combined with one all_reduce, at the end or per chunk.  The reference
consumes ONE generator sequentially over the tiles (inference...:197,268); to keep that stream every rank draws the noise
of every tile in loop order and uses its own.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Iterator, List, Optional, Tuple

import torch

from . import sharding
from .pipeline_upscale_a_video import randn_tensor


@dataclass(frozen=True)
class Tile:
    in_box: Tuple[int, int, int, int]    # (y0, y1, x0, x1) on the LR frame, including the overlap context
    out_box: Tuple[int, int, int, int]   # (y0, y1, x0, x1) on the 4x output frame
    src_box: Tuple[int, int, int, int]   # (y0, y1, x0, x1) inside the tile's 4x output


def needs_tiling(h: int, w: int) -> bool:
    """inference_upscale_a_video.py:201-202"""
    return h * w >= 384 * 384


def plan_tiles(h: int, w: int, tile_size: int = 256, overlap: int = 64, scale: int = 4) -> List[Tile]:
    tiles_x, tiles_y = math.ceil(w / tile_size), math.ceil(h / tile_size)
    # a trailing tile whose fresh area would not exceed the overlap is merged into its neighbour (inference...:220-227)
    merge_w = (tiles_x - 1) * tile_size + overlap >= w
    merge_h = (tiles_y - 1) * tile_size + overlap >= h
    if merge_w:
        tiles_x -= 1
    if merge_h:
        tiles_y -= 1
    out_h, out_w = h * scale, w * scale
    plan = []
    for y in range(tiles_y):
        for x in range(tiles_x):
            x0, y0 = x * tile_size, y * tile_size
            x1, y1 = min(x0 + tile_size, w), min(y0 + tile_size, h)
            px0, px1 = max(x0 - overlap, 0), min(x1 + overlap, w)
            py0, py1 = max(y0 - overlap, 0), min(y1 + overlap, h)
            last_x, last_y = (x == tiles_x - 1 and merge_w), (y == tiles_y - 1 and merge_h)
            ox0, oy0 = x0 * scale, y0 * scale
            ox1 = out_w if last_x else x1 * scale
            oy1 = out_h if last_y else y1 * scale
            sx0, sy0 = (x0 - px0) * scale, (y0 - py0) * scale
            plan.append(Tile((py0, py1, px0, px1), (oy0, oy1, ox0, ox1), (sy0, sy0 + oy1 - oy0, sx0, sx0 + ox1 - ox0)))
    return plan


_SOLO_GROUPS = {}


def _solo_group(rank: int, world: int):
    """single-rank process groups, created once per world size (new_group is a collective and a communicator that is
    never destroyed would leak one NCCL communicator per rank per clip)"""
    if world not in _SOLO_GROUPS:
        import torch.distributed as dist
        _SOLO_GROUPS[world] = [dist.new_group([r]) for r in range(world)]  # every rank creates every group
    return _SOLO_GROUPS[world][rank]


def _rank_tiles(pipeline, image, flows_bi, generator, plan, process_group, pipe_kwargs):
    """Yields `(tile, LR clip of the tile, its flows, noise, initial latents)` for this rank's tiles in plan order, while
    `pipeline.process_group` is this rank's single-rank group.  Every rank draws every tile's noise from the one
    generator, so each tile gets the draw the reference's serial loop would give it."""
    b, _, t, _, _ = image.shape
    rank, world = sharding.world_info(process_group)
    dtype = None
    for key in ("prompt_embeds", "negative_prompt_embeds"):
        if pipe_kwargs.get(key) is not None:
            dtype = pipe_kwargs[key].dtype
    if dtype is None:
        dtype = getattr(pipeline.text_encoder, "dtype", torch.float16)
    c_lat = pipeline.vae.config.latent_channels
    # tiles are independent pipeline runs: inside a tile the pipeline must not shard windows over the same ranks
    saved_group = pipeline.process_group
    try:
        pipeline.process_group = _solo_group(rank, world) if world > 1 else saved_group
        for i, tl in enumerate(plan):
            py0, py1, px0, px1 = tl.in_box
            tile = image[:, :, :, py0:py1, px0:px1]
            # the generator stream of the reference: per tile, first the LR noise, then the initial latents
            noise = randn_tensor(tile.shape, generator=generator, device=image.device, dtype=dtype)
            latents = randn_tensor((b, c_lat, t, py1 - py0, px1 - px0), generator=generator, device=image.device, dtype=dtype)
            if i % world != rank:
                continue
            flows = None
            if flows_bi is not None:
                flows = [f[:, :, :, py0:py1, px0:px1] for f in flows_bi]
            yield tl, tile, flows, noise, latents
    finally:
        pipeline.process_group = saved_group


def _paste(out, tl, res):
    oy0, oy1, ox0, ox1 = tl.out_box
    sy0, sy1, sx0, sx1 = tl.src_box
    out[:, :, :, oy0:oy1, ox0:ox1] = res[:, :, :, sy0:sy1, sx0:sx1]


@torch.no_grad()
def upscale_tiled(pipeline, image: torch.Tensor, flows_bi: Optional[list] = None, generator=None, tile_size: int = 256,
                  overlap: int = 64, process_group=None, **pipe_kwargs) -> torch.Tensor:
    """image: (1, 3, T, H, W) LR clip in [-1, 1] on the GPU.  Returns the (1, 3, T, 4H, 4W) output like the reference's
    tile branch.  `pipe_kwargs` go to `VideoUpscalePipeline.__call__` (prompt / prompt_embeds, steps, guidance, ...)."""
    b, c, t, h, w = image.shape
    plan = plan_tiles(h, w, tile_size, overlap)
    out = image.new_zeros((b, c, t, 4 * h, 4 * w), dtype=torch.float32)
    for tl, tile, flows, noise, latents in _rank_tiles(pipeline, image, flows_bi, generator, plan, process_group,
                                                       pipe_kwargs):
        _paste(out, tl, pipeline(image=tile, flows_bi=flows, noise=noise, latents=latents, **pipe_kwargs).images)
    if sharding.world_info(process_group)[1] > 1:
        import torch.distributed as dist
        dist.all_reduce(out, group=process_group)  # paste regions are disjoint: sum == union
    return out


@torch.no_grad()
def iter_upscale_tiled(pipeline, image: torch.Tensor, flows_bi: Optional[list] = None, generator=None,
                       tile_size: int = 256, overlap: int = 64, process_group=None,
                       **pipe_kwargs) -> Iterator[Tuple[int, int, torch.Tensor]]:
    """`upscale_tiled` a few frames at a time: yields `(s, e, chunk)` in the order of `sharding.decode_chunks(T)`, `chunk`
    the fp32 (1, 3, e - s, 4H, 4W) output of frames [s, e), equal to `upscale_tiled(...)[:, :, s:e]`.  Every tile of
    this rank is sampled first (`pipeline.sample_latents`) and only its latents are kept; then each chunk decodes every
    tile's frames [s, e) (`pipeline.decode_latents_vsr`) and pastes them, with one all_reduce per chunk across ranks."""
    b, c, t, h, w = image.shape
    plan = plan_tiles(h, w, tile_size, overlap)
    sampled = []
    for tl, tile, flows, noise, latents in _rank_tiles(pipeline, image, flows_bi, generator, plan, process_group,
                                                       pipe_kwargs):
        r = pipeline.sample_latents(image=tile, flows_bi=flows, noise=noise, latents=latents, **pipe_kwargs)
        sampled.append((tl, r.latents, r.w_lr))
        del r  # the record's LR copy is taken again from `image` per chunk
    world = sharding.world_info(process_group)[1]
    for s, e in sharding.decode_chunks(t):
        out = image.new_zeros((b, c, e - s, 4 * h, 4 * w), dtype=torch.float32)
        for tl, latents, w_lr in sampled:
            py0, py1, px0, px1 = tl.in_box
            lr = image[:, :, s:e, py0:py1, px0:px1].to(torch.float32)
            _paste(out, tl, pipeline.decode_latents_vsr(latents[:, :, s:e], lr, w_lr))
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(out, group=process_group)  # paste regions are disjoint: sum == union
        yield s, e, out
