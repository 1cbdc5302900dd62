"""Multi-GPU work partitioning for the sampling loop (SURVEY.md §8e).

The reference is single-GPU and serial (pipeline_upscale_a_video.py:621-635, 693-697).  Within one DDIM step the
8-frame UNet windows are independent, and so are the 3-frame VAE decode chunks; everything else (window blend, CFG,
step_v0, flow propagation — a recurrence over the WHOLE clip — and step_vt) is cheap 4-channel elementwise work.
So: one process per GPU with replicated weights, window w of the step goes to rank `w % world`, ONE all_gather of
the windows' noise predictions per step (the "propagation boundary"), after which every rank redundantly runs
the elementwise tail in the reference's exact window order (the 0.5/0.5 blend is order dependent).  Decode chunks
are dealt the same way and gathered `world` at a time.  No collective exists when world == 1.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import torch
import torch.distributed as dist

SHORT_SEQ, OVERLAP_SEQ, DECODE_SEQ = 8, 2, 3  # pipeline_upscale_a_video.py:601-602, 685


def unet_windows(T: int) -> List[Tuple[int, int]]:
    """window list of pipeline_upscale_a_video.py:621-625 in loop order, incl. the re-anchored last window
    (which can duplicate its predecessor, e.g. T=14 -> (0,8),(6,14),(6,14))."""
    if T <= SHORT_SEQ:
        return [(0, T)]
    out = []
    for s in range(0, T, SHORT_SEQ - OVERLAP_SEQ):
        e = min(T, s + SHORT_SEQ)
        if e - s < SHORT_SEQ:
            s = e - SHORT_SEQ
        out.append((s, e))
    return out


def decode_chunks(T: int) -> List[Tuple[int, int]]:
    """pipeline_upscale_a_video.py:685-697"""
    if T <= DECODE_SEQ:
        return [(0, T)]
    return [(s, min(T, s + DECODE_SEQ)) for s in range(0, T, DECODE_SEQ)]


def assign(units: Sequence, world: int) -> Dict[int, List[int]]:
    """unique unit index -> owner rank, round robin; returns rank -> list of unique-unit indices"""
    uniq: List = []
    for u in units:
        if u not in uniq:
            uniq.append(u)
    owners: Dict[int, List[int]] = {r: [] for r in range(world)}
    for i, _ in enumerate(uniq):
        owners[i % world].append(i)
    return owners


def unique(units: Sequence) -> List:
    uniq: List = []
    for u in units:
        if u not in uniq:
            uniq.append(u)
    return uniq


# relative cost of a UNet call on ONE classifier-free-guidance half of a window, against the call on both halves (which
# shares the text-independent prefix, ~3.6 % of the work: unet_video.py `cfg_shared_input`)
HALF_UNIT_COST = 0.52


def window_units(n_windows: int, world: int, can_split: bool) -> List[Tuple[int, int]]:
    """work units of one DDIM step, in dealing order: (window index, half) with half = -1 for "both CFG halves in one
    UNet call".  GroupNorm statistics, attention and convolutions never mix batch items, so a window's two halves are
    independent UNet calls; dealing HALVES turns e.g. 11 windows on 8 ranks from 2 rounds into 3 half-rounds = 1.56.
    Halves are used only when that lowers the makespan (never for world == 1, never when windows divide evenly)."""
    if n_windows == 0:
        return []
    rounds_full = -(-n_windows // world)
    rounds_half = -(-2 * n_windows // world)
    if can_split and world > 1 and rounds_half * HALF_UNIT_COST < rounds_full:
        return [(w, h) for w in range(n_windows) for h in (0, 1)]
    return [(w, -1) for w in range(n_windows)]


_COMM_EVENTS = None  # list of (start, end) CUDA events while bench.py measures the collective's share of a step


def comm_events_reset(on: bool):
    global _COMM_EVENTS
    _COMM_EVENTS = [] if on else None


def comm_events_ms() -> float:
    if not _COMM_EVENTS:
        return 0.0
    torch.cuda.synchronize()
    return float(sum(s.elapsed_time(e) for s, e in _COMM_EVENTS))


def world_info(group=None) -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def all_gather_units(local: Dict[int, torch.Tensor], n_units: int, unit_shape, dtype, device, group=None
                     ) -> List[torch.Tensor]:
    """Every rank contributes the unique units it computed (`local`: unit index -> tensor of `unit_shape`); returns
    all `n_units` tensors on every rank.  One all_gather of a (units_per_rank, *unit_shape) buffer."""
    rank, world = world_info(group)
    if world == 1:
        return [local[i] for i in range(n_units)]
    per_rank = (n_units + world - 1) // world
    send = torch.zeros((per_rank, *unit_shape), dtype=dtype, device=device)
    mine = [i for i in range(n_units) if i % world == rank]
    for slot, i in enumerate(mine):
        send[slot].copy_(local[i])
    recv = torch.empty((world, per_rank, *unit_shape), dtype=dtype, device=device)
    ev = None
    if _COMM_EVENTS is not None and device.type == "cuda":
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
        ev[0].record()
    dist.all_gather_into_tensor(recv.view(world * per_rank, *unit_shape), send, group=group)
    if ev is not None:
        ev[1].record()
        _COMM_EVENTS.append(ev)
    out = []
    for i in range(n_units):
        out.append(recv[i % world, i // world])
    return out
