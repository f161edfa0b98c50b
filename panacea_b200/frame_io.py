"""Frame writers of the inference entry point (reference inference.py:110-205; SURVEY.md section 8f, row N3): the
on-disk layout the StreamPETR evaluation consumes — `fake/<scene>_<cam file stem>/_{frame:06}.jpg` per camera and frame —
plus the per-sample PNG strips and GIFs. Pure host code (PIL): it runs after the denoising loop and the VAE decode."""
from __future__ import annotations

import os

import numpy as np
import torch
from PIL import Image

# inference.py:110-125: view order of the panorama strip and the index of each camera in `filenames`
CAMERA_VIEWS = ["CAM_FRONT", "CAM_FRONT_RIGHT", "CAM_BACK_RIGHT", "CAM_BACK", "CAM_BACK_LEFT", "CAM_FRONT_LEFT"]
VIEW_ID = {"CAM_FRONT": 0, "CAM_FRONT_RIGHT": 1, "CAM_BACK_RIGHT": 5, "CAM_BACK": 3, "CAM_BACK_LEFT": 4, "CAM_FRONT_LEFT": 2}


def _to_uint8_hwc(img_chw: torch.Tensor) -> np.ndarray:
    """[-1, 1] CHW -> uint8 HWC (inference.py:160-166); maps with more than 4 channels collapse to min over the first 10."""
    a = ((img_chw.detach().float().cpu().clamp(-1.0, 1.0) + 1.0) / 2.0).permute(1, 2, 0).numpy()
    a = (a * 255).astype(np.uint8)
    if a.shape[-1] > 4:
        a = a[:, :, :10].min(-1)
    return a.squeeze(-1) if a.ndim == 3 and a.shape[-1] == 1 else a


def _stem(path: str) -> str:
    return path.split("/")[-1].split(".")[0]


def _name(entry) -> str:
    """DataLoader collates the per-frame, per-camera file names into nested lists of 1-tuples (batch size 1)."""
    return entry[0] if isinstance(entry, (list, tuple)) else entry


def logs_frames(jpgs: torch.Tensor, root: str, filenames, view_width: int | None = None) -> list[str]:
    """inference.py:171-196. jpgs [T, 3, H, 6*w] in [-1, 1]: one directory per camera named
    `<scene token>_<file stem of the LAST frame of that camera>`, files `_{frame:06}.jpg`."""
    T, _, _, Wtot = jpgs.shape
    w = view_width or Wtot // len(CAMERA_VIEWS)
    written = []
    for view in CAMERA_VIEWS:
        i = VIEW_ID[view]
        file_dir = _stem(_name(filenames[-1][i]))
        path_view = os.path.join(root, file_dir.split("__")[-2] + "_" + file_dir)
        os.makedirs(path_view, exist_ok=True)
        for frame_id in range(T):
            path = os.path.join(path_view, "_{:06}.jpg".format(frame_id))
            Image.fromarray(_to_uint8_hwc(jpgs[frame_id][:, :, w * i:w * i + w])).save(path)
            written.append(path)
    return written


def logs_all_images(outs: dict, root: str, filenames) -> list[str]:
    """inference.py:146-169: every logged tensor as one vertical PNG strip (frames stacked, nrow=1)."""
    written = []
    for k, v in outs.items():
        if not isinstance(v, torch.Tensor) or "cond_img" in k or "reconstructions" in k or v.dim() != 4:
            continue
        os.makedirs(os.path.join(root, k), exist_ok=True)
        strip = torch.cat(list(v.detach().float().cpu().clamp(-1.0, 1.0)), dim=1)       # make_grid(nrow=1), no padding
        path = os.path.join(root, k, _stem(_name(filenames[-1][0])) + ".png")
        Image.fromarray(_to_uint8_hwc(strip)).save(path)
        written.append(path)
    return written


def logs_scene(frames: torch.Tensor, inferdir: str, filenames) -> list[str]:
    """A scene of K chained clips sharing m frames (panacea_b200/scene.py): frames [K(T-m)+m, 3, H, 6*w] and their
    `filenames`, both in chronological order. Writes `fake/<scene>_<cam>/_{frame:06}.jpg` numbered `_000000` ..
    `_{K(T-m)+m-1:06}` over the whole scene (the directory named, as for one clip, after the last frame), one PNG strip
    under `allimages/samples/` and one GIF under `gifs/samples/`."""
    outs = {"samples": frames}
    return (logs_frames(frames, os.path.join(inferdir, "fake"), filenames)
            + logs_all_images(outs, os.path.join(inferdir, "allimages"), filenames)
            + logs_all_gifs(outs, os.path.join(inferdir, "gifs"), filenames, num_frames=frames.shape[0]))


def logs_all_gifs(outs: dict, root: str, filenames, num_frames: int = 8) -> list[str]:
    """inference.py:127-145: one GIF (4 fps, looping) per logged tensor and sequence."""
    written = []
    for k, v in outs.items():
        if not isinstance(v, torch.Tensor) or v.dim() != 4 or "txt" in k or "cond_img" in k or "reconstructions" in k:
            continue
        if v.shape[0] % num_frames:
            continue
        os.makedirs(os.path.join(root, k), exist_ok=True)
        seqs = v.reshape(-1, num_frames, *v.shape[1:])
        for b in range(seqs.shape[0]):
            frames = [Image.fromarray(_to_uint8_hwc(f)) for f in seqs[b]]
            path = os.path.join(root, k, _stem(_name(filenames[-1][0])) + ".gif")
            frames[0].save(path, save_all=True, append_images=frames[1:], duration=250, loop=0)
            written.append(path)
    return written
