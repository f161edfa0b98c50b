"""Scenes longer than one clip: K clips chained through their boundary frame (DESIGN.md section 11).

Each clip of `T` frames is conditioned on one frame at index `a` (`T-1` with `use_last_frame`, else `0`). Clip 0 takes
the dataset's real frame; clip k > 0 takes the frame of clip k-1 at the opposite end, index `T-1-a`, after the round
trip a user would make through the writers and the dataset: clamp to [-1, 1] and quantise to uint8 exactly as
`frame_io._to_uint8_hwc` does, then map back with `/127.5 - 1` (nuscenes_datasets_video.py:551-552). With
`use_last_frame` the scene therefore grows into the past, otherwise into the future. The boundary frame is kept once,
from the clip that generated it first, so a scene has K(T-1)+1 frames in chronological order.

Pure host code: the device work of a scene is K ordinary `log_images` clips (`DiffusionEngine3D.sample_scene`)."""
from __future__ import annotations

import numpy as np
import torch

from .frame_io import _to_uint8_hwc


def cond_index(num_frames: int, use_last_frame: bool) -> int:
    """Index of the conditioning frame inside a clip (nuscenes_datasets_video.py:559-566)."""
    return num_frames - 1 if use_last_frame else 0


def handoff_index(num_frames: int, use_last_frame: bool) -> int:
    """Index of the frame of clip k-1 that conditions clip k: the end opposite the conditioning frame."""
    return num_frames - 1 - cond_index(num_frames, use_last_frame)


def scene_length(clips: int, num_frames: int) -> int:
    return clips * (num_frames - 1) + 1


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


def scene_slices(clips: int, num_frames: int, use_last_frame: bool) -> list[tuple[int, int, int]]:
    """(clip, first frame, end frame) ranges that make up the scene in chronological order. Clip k > 0 leaves out its
    conditioning frame, which clip k-1 already holds."""
    T = num_frames
    if use_last_frame:                          # clip k ends where clip k-1 begins: the latest clip comes first
        return [(k, 0, T - 1) for k in range(clips - 1, 0, -1)] + [(0, 0, T)]
    return [(0, 0, T)] + [(k, 1, T) for k in range(1, clips)]


def scene_order(per_clip, use_last_frame: bool):
    """Concatenates per-clip sequences (tensors [T, ...] or lists of length T, e.g. `filenames`) into the scene's
    chronological order with the boundary frames kept once."""
    T = len(per_clip[0])
    parts = [per_clip[k][lo:hi] for k, lo, hi in scene_slices(len(per_clip), T, use_last_frame)]
    if isinstance(per_clip[0], torch.Tensor):
        return torch.cat(parts)
    return [x for p in parts for x in p]


def scene_frame_number(clip: int, frame: int, clips: int, num_frames: int, use_last_frame: bool) -> int:
    """Chronological position of frame `frame` of clip `clip` in the scene (the two copies of a boundary frame share
    it)."""
    start = (clips - 1 - clip) if use_last_frame else clip
    return start * (num_frames - 1) + frame
