"""Scenes longer than one clip: K clips chained through their boundary frame, or through m shared frames
(DESIGN.md section 11).

Each clip of `T` frames is conditioned on one frame at index `a` (`T-1` with `use_last_frame`, else `0`). Clip 0 takes
the dataset's real frame; clip k > 0 takes the frame of clip k-1 that lands on its index `a` (`handoff_index`), after
the round trip a user would make through the writers and the dataset: clamp to [-1, 1] and quantise to uint8 exactly
as `frame_io._to_uint8_hwc` does, then map back with `/127.5 - 1` (nuscenes_datasets_video.py:551-552). With
`use_last_frame` the scene therefore grows into the past, otherwise into the future.

Consecutive clips share m frames: m = 1 (the boundary frame) when `overlap` is None, else `overlap`, 1 <= m <= T-1.
With `use_last_frame` clip k's frames T-m .. T-1 are clip k-1's frames 0 .. m-1; without it, clip k's frames 0 .. m-1
are clip k-1's frames T-m .. T-1. A shared frame has one chronological number in both clips and is kept once, from
the clip that generated it first, so a scene has K(T-m)+m frames in chronological order. With an explicit `overlap`
clip k keeps clip k-1's latents of the shared frames as a known region (`known_region`) and generates only the rest.

Pure host code: the device work of a scene is K ordinary clips (`DiffusionEngine3D.sample_scene`)."""
from __future__ import annotations

import numpy as np
import torch

from .frame_io import _to_uint8_hwc


def check_overlap(overlap, num_frames: int) -> None:
    """None (the boundary frame only, regenerated) or 1 <= overlap <= T-1 shared frames; raises ValueError otherwise."""
    if overlap is None:
        return
    if isinstance(overlap, bool) or not isinstance(overlap, (int, np.integer)) or not 1 <= overlap <= num_frames - 1:
        raise ValueError(f"overlap must be an integer in 1 .. {num_frames - 1} (clips of {num_frames} frames), got {overlap!r}")


def _shared(overlap) -> int:
    return 1 if overlap is None else int(overlap)


def cond_index(num_frames: int, use_last_frame: bool) -> int:
    """Index of the conditioning frame inside a clip (nuscenes_datasets_video.py:559-566)."""
    return num_frames - 1 if use_last_frame else 0


def handoff_index(num_frames: int, use_last_frame: bool, overlap=None) -> int:
    """Index of the frame of clip k-1 that conditions clip k: the shared frame that lands on clip k's conditioning
    index, m-1 with `use_last_frame` and T-m without (the end opposite the conditioning frame for m = 1)."""
    m = _shared(overlap)
    return m - 1 if use_last_frame else num_frames - m


def shared_frames(num_frames: int, use_last_frame: bool, overlap=None) -> tuple[range, range]:
    """(indices in clip k, indices in clip k-1) of the frames the two clips share, pairwise the same scene frame."""
    T, m = num_frames, _shared(overlap)
    head, tail = range(0, m), range(T - m, T)
    return (tail, head) if use_last_frame else (head, tail)


def scene_length(clips: int, num_frames: int, overlap=None) -> int:
    m = _shared(overlap)
    return clips * (num_frames - m) + m


def quantize_frame(img_chw: torch.Tensor) -> torch.Tensor:
    """Decoded frame [3, H, W] -> the frame a dataset would read back from the writers' JPEG source: uint8 as the
    writers quantise it, then `/127.5 - 1` in float32. Returns a CPU float32 [3, H, W] tensor."""
    u8 = _to_uint8_hwc(img_chw)
    return torch.from_numpy(u8.astype(np.float32) / 127.5 - 1.0).permute(2, 0, 1).contiguous()


def condition_from_frame(frame_chw: torch.Tensor, num_frames: int, use_last_frame: bool) -> torch.Tensor:
    """`final_cond_zero` of one clip [T, 3, H, W]: zeros except `frame_chw` at the conditioning index."""
    cond = torch.zeros(num_frames, *frame_chw.shape, dtype=frame_chw.dtype, device=frame_chw.device)
    cond[cond_index(num_frames, use_last_frame)] = frame_chw
    return cond


def known_region(prev_latent: torch.Tensor, use_last_frame: bool, overlap) -> tuple[torch.Tensor, torch.Tensor]:
    """Clip k's (known [T, 4, h, w], mask [T, h, w]) from clip k-1's final latent [T, 4, h, w]: the shared frames are
    clip k-1's latents with mask 0 (kept), every other frame is zero with mask 1 (generated). Float32, on the device
    of `prev_latent`."""
    T = prev_latent.shape[0]
    check_overlap(overlap, T)
    cur, prev = shared_frames(T, use_last_frame, overlap)
    known = torch.zeros(prev_latent.shape, dtype=torch.float32, device=prev_latent.device)
    mask = torch.ones((T, *prev_latent.shape[2:]), dtype=torch.float32, device=prev_latent.device)
    known[cur.start:cur.stop] = prev_latent[prev.start:prev.stop]
    mask[cur.start:cur.stop] = 0.0
    return known, mask


def scene_slices(clips: int, num_frames: int, use_last_frame: bool, overlap=None) -> list[tuple[int, int, int]]:
    """(clip, first frame, end frame) ranges that make up the scene in chronological order. Clip k > 0 leaves out the
    frames it shares with clip k-1, which clip k-1 already holds."""
    T, m = num_frames, _shared(overlap)
    if use_last_frame:                          # clip k ends where clip k-1 begins: the latest clip comes first
        return [(k, 0, T - m) for k in range(clips - 1, 0, -1)] + [(0, 0, T)]
    return [(0, 0, T)] + [(k, m, T) for k in range(1, clips)]


def scene_order(per_clip, use_last_frame: bool, overlap=None):
    """Concatenates per-clip sequences (tensors [T, ...] or lists of length T, e.g. `filenames`) into the scene's
    chronological order with the shared frames kept once."""
    T = len(per_clip[0])
    parts = [per_clip[k][lo:hi] for k, lo, hi in scene_slices(len(per_clip), T, use_last_frame, overlap)]
    if isinstance(per_clip[0], torch.Tensor):
        return torch.cat(parts)
    return [x for p in parts for x in p]


def scene_frame_number(clip: int, frame: int, clips: int, num_frames: int, use_last_frame: bool, overlap=None) -> int:
    """Chronological position of frame `frame` of clip `clip` in the scene (the copies of a shared frame share it)."""
    start = (clips - 1 - clip) if use_last_frame else clip
    return start * (num_frames - _shared(overlap)) + frame
