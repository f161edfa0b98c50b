"""Paste the recorded pixels back outside an edit (DESIGN.md section 13).

An edit keeps the recorded latent outside its mask, but the decoder reconstructs every pixel, so the kept regions of a
decoded edit are a lossy reconstruction of the recording. `composite_frames` takes the decode where cells were
regenerated, the recorded pixels where they were not, and a linear ramp of `feather` pixels outside the regenerated
cells between the two. The recorded pixels are written as their byte centres (b + 0.5) / 127.5 - 1, which the frame
writers' truncating quantiser maps back to the recorded bytes b (the value a dataset reads, b / 127.5 - 1, comes back one
lower for 63 of the 256 bytes). The result does not depend on the precision mode.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import ptr

MAX_FEATHER = 64
VIEWS = 6


def composite_frames(decoded: torch.Tensor, recorded: torch.Tensor, cells: torch.Tensor, feather: int):
    """decoded, recorded fp32 [F, 3, H, 6w] on the GPU; cells [F, H/cell, 6w/cell] (a cell > 0 was regenerated).
    Returns (frames [F, 3, H, 6w], alpha [F, H, 6w]): alpha is 1 in the regenerated cells, falls to 0 over `feather`
    pixels outside them within each panel, and frames = recorded byte centre + alpha (decoded - byte centre), exactly
    the decode where alpha = 1 and exactly the byte centre where alpha = 0 (pn_composite_frames)."""
    if decoded.dim() != 4 or decoded.shape[1] != 3 or decoded.shape[3] % VIEWS:
        raise ValueError(f"decoded: expected [F, 3, H, 6w], got {tuple(decoded.shape)}")
    if recorded.shape != decoded.shape:
        raise ValueError(f"recorded: expected {tuple(decoded.shape)}, got {tuple(recorded.shape)}")
    F, _, H, Wt = decoded.shape
    if cells.dim() != 3 or cells.shape[0] != F or cells.shape[1] == 0 or H % cells.shape[1] \
            or Wt != cells.shape[2] * (H // cells.shape[1]):
        raise ValueError(f"cells: expected [{F}, H/cell, 6w/cell] for frames of {H} x {Wt}, got {tuple(cells.shape)}")
    if not 0 <= int(feather) <= MAX_FEATHER:
        raise ValueError(f"feather must lie in 0 .. {MAX_FEATHER}, got {feather}")
    dev = decoded.device
    dec, rec = (t.to(dev, torch.float32).contiguous() for t in (decoded, recorded))
    cel = cells.to(dev, torch.float32).contiguous()
    out = torch.empty_like(dec)
    alpha = torch.empty(F, H, Wt, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().pn_composite_frames(ptr(dec), ptr(rec), ptr(cel), ptr(out), ptr(alpha), F, H, Wt // VIEWS,
                                               H // cells.shape[1], int(feather), _lib.stream(dev)), "pn_composite_frames")
    return out, alpha
