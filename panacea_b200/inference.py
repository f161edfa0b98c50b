"""Inference entry point with the control flow of the reference's inference.py (main, :230-317): one process per GPU,
`DistributedSampler(shuffle=False)` + batch size 1 (one 6-view x 8-frame sequence per step and rank), seed = rank + 3407,
model built from `configs/inference_nuscenes.yaml`-style YAML via instantiate_from_config, `log_images` per batch, frame
writers. SURVEY.md section 8f rows N1 (engine / conditioner glue) and N3 (writers, gather -> rank-0 writer).

What is NOT here, and why: the nuScenes dataset itself (needs nuScenes and mmdet3d) is replaced by `SyntheticBEVDataset`
with the same batch contract, or, with `--layout scene.npz`, by `LayoutDataset`: a scene file of boxes, map polylines and
cameras whose 19-channel layout maps are rendered on the GPU (panacea_b200/layout.py, DESIGN.md section 12). The VAE (encoder and decoder) is native and random-init unless a
checkpoint provides `first_stage_model.*`. The OpenCLIP text tower is native too once it has weights: from the checkpoint
(`conditioner.embedders.0.model.*`) or from a stock open_clip file given as the embedder's `version`; prompts are
tokenized with the CLIP BPE vocabulary at the embedder's `bpe_path` (else open_clip's bundled copy). Without weights the
embedder is a deterministic stand-in. With the real modules importable, `--dataset module:Class` and the YAML targets
swap them in. `--clips K` generates scenes of K clips chained through their boundary frame, and `--overlap M` chains
them through M shared frames whose latents each clip keeps from the one before (DESIGN.md section 11).
`--strength S` edits each item's recorded frames instead of sampling from noise, and with `--layout EDITED.npz
--mask_from ORIGINAL.npz` regenerates only where the edited layout differs from the original (DESIGN.md section 13);
`--mask_image` takes a user-drawn mask, and `--composite F` pastes the recorded pixels back outside the edit.
Overrides use the dotlist form, and a numeric component indexes a list:

  torchrun --nproc-per-node 8 -m panacea_b200.inference --base configs.yaml --name run1 --inferdir out --gather
      --ckptpath panacea.ckpt model.params.conditioner_config.params.emb_models.0.params.bpe_path=bpe_simple_vocab_16e6.txt.gz
"""
from __future__ import annotations

import argparse
import importlib
import os
import time

from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist
import yaml
from PIL import Image
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.distributed import DistributedSampler

from . import dist_utils as D
from . import frame_io as IO
from . import layout as L
from .composite import MAX_FEATHER
from .scene import check_overlap, cond_index, condition_from_frame, scene_frame_number, scene_length
from .sgm.util import instantiate_from_config


def _check_scene(clips, overlap, num_frames):
    """A dataset item of `clips` clips of `num_frames` frames sharing `overlap` (scene.check_overlap)."""
    if clips < 1:
        raise ValueError(f"clips must be >= 1, got {clips}")
    check_overlap(overlap, num_frames)


class SyntheticBEVDataset(Dataset):
    """Batch contract of sgm/data/nuscenes_video/nuscenes_datasets_video.py:495-570 (`MyDataset.__getitem__`) with
    synthetic content: `jpg` target frames [T,3,H,6w] in [-1,1], `cond_img` the 19-channel BEV control maps [T,19,H,6w]
    in [0,1], `final_cond_zero` the image condition (zeros except the last — or first — frame, :559-566), `txt`,
    `filenames` (per frame, per camera).

    Scene form (`clips` = K > 1, DESIGN.md section 11): an item is `{"clips": [clip_0, ..., clip_{K-1}]}`. Clip 0 is the
    batch above; clips k > 0 carry only their layout, `cond_img`, `txt` and `filenames`, because their image condition
    is a frame that clip k-1 generates. A frame two clips share (the boundary frame, or the `overlap` shared frames)
    has the same file name in both clips that hold it."""

    def __init__(self, num_sequences=2, num_frames=8, image_hw=(256, 512), use_last_frame=True, seed=0, clips=1,
                 overlap=None):
        self.n, self.T, (self.h, self.w), self.use_last_frame, self.seed = num_sequences, num_frames, image_hw, use_last_frame, seed
        _check_scene(clips, overlap, num_frames)
        self.clips, self.overlap = clips, overlap

    def __len__(self):
        return self.n

    def _names(self, idx, clip):
        scene = f"n015-2018-07-24-11-22-45+0800__seq{idx:04d}"
        stamp = lambda f: 1532402927 + 50 * scene_frame_number(clip, f, self.clips, self.T, self.use_last_frame, self.overlap)
        return [[f"samples/{cam}/{scene}__{cam}__{stamp(f):d}.jpg" for cam in sorted(IO.VIEW_ID, key=IO.VIEW_ID.get)]
                for f in range(self.T)]

    def __getitem__(self, idx):
        g = torch.Generator().manual_seed(self.seed * 100003 + idx)
        W = 6 * self.w
        target = torch.rand(self.T, 3, self.h, W, generator=g) * 2.0 - 1.0
        cond = torch.zeros_like(target)
        k = -1 if self.use_last_frame else 0
        cond[k] = target[k]
        txt = "a driving scene, six surround-view cameras"
        first = {"jpg": target, "cond_img": torch.rand(self.T, 19, self.h, W, generator=g), "final_cond_zero": cond,
                 "txt": txt, "filenames": self._names(idx, 0)}
        if self.clips == 1:
            return first
        return {"clips": [first] + [{"cond_img": torch.rand(self.T, 19, self.h, W, generator=g), "txt": txt,
                                     "filenames": self._names(idx, c)} for c in range(1, self.clips)]}


class LayoutDataset(Dataset):
    """One scene file (panacea_b200/layout.py) as a dataset of one item with the batch contract of `MyDataset` (see
    `SyntheticBEVDataset`), without the ground-truth `jpg`: `cond_img` rendered on `device` by `render_layout`,
    `final_cond_zero`, `txt` and `filenames`. The scene must hold K(T-m)+m frames for K = `clips` and m = `overlap`
    shared frames (1 when None); clip k renders the scene frames that `scene.scene_frame_number` assigns to it, so the
    frames it shares with its neighbour render from the same scene frames. Clip 0 is
    conditioned on a real frame: `cond_frame` or the scene file's `cond_frame`, an RGB image of [H, 6w] in the
    panel order of the renderer, which becomes clip 0's frame at the conditioning index. The caption is the file's
    `prompt`, else one written from the classes of each clip's last frame (the reference captions a clip by its last
    frame, :541).

    A scene with `frame_files` also gives each clip its recorded frames as `jpg`. With `edit` (one clip only) those are
    required and clip 0's image condition is the recorded frame at the conditioning index instead of `cond_frame`."""

    def __init__(self, path, num_frames=8, image_hw=(256, 512), use_last_frame=True, clips=1, cond_frame=None,
                 device="cuda", edit=False, overlap=None):
        _check_scene(clips, overlap, num_frames)
        self.path, self.T, (self.h, self.w) = Path(path), num_frames, tuple(image_hw)
        self.use_last_frame, self.clips, self.device, self.edit, self.overlap = use_last_frame, clips, device, edit, overlap
        self.scene = L.load_scene(path)
        want = scene_length(clips, num_frames, overlap)
        if self.scene.num_frames != want:
            shared = "" if overlap is None else f" with {overlap} shared between neighbours"
            raise L.SceneError(f"{self.path.name}: {self.scene.num_frames} frames, but {clips} clips of {num_frames} "
                               f"frames{shared} need {want}")
        if edit:
            if clips != 1 or cond_frame is not None:
                raise ValueError("editing takes one clip, conditioned on its own recorded frame")
            if self.scene.frame_files is None:
                raise L.SceneError(f"{self.path.name}: editing needs the recorded frames ('frame_files')")
            self.cond_frame = None
            return
        src = cond_frame or self.scene.cond_frame
        if src is None:
            raise L.SceneError(f"{self.path.name}: clip 0 needs a conditioning frame (--cond_frame or 'cond_frame')")
        self.cond_frame = self._read(src, "conditioning frame")

    def _read(self, src, what):
        """An [H, 6w] RGB image as [3, H, 6w] in [-1, 1]."""
        img = np.asarray(Image.open(src).convert("RGB"))
        if img.shape != (self.h, 6 * self.w, 3):
            raise L.SceneError(f"{what} {src}: expected {6 * self.w} x {self.h}, got {img.shape[1]} x {img.shape[0]}")
        return torch.from_numpy(img.astype(np.float32) / 127.5 - 1.0).permute(2, 0, 1).contiguous()

    def __len__(self):
        return 1

    def frames(self, clip):
        """Scene frame of each of the clip's T frames."""
        return [scene_frame_number(clip, f, self.clips, self.T, self.use_last_frame, self.overlap) for f in range(self.T)]

    def _clip(self, clip):
        frames = self.frames(clip)
        stem = self.path.stem
        names = [[f"samples/{cam}/{stem}__{cam}__{f:06d}.jpg" for cam in IO.CAMERA_VIEWS] for f in frames]
        txt = self.scene.prompt or L.caption(self.scene.labels[frames[-1]])
        batch = {"cond_img": L.render_layout(self.scene, frames, self.h, self.w, self.device), "txt": txt, "filenames": names}
        if self.scene.frame_files is not None:
            batch["jpg"] = torch.stack([self._read(self.scene.frame_files[f], "recorded frame") for f in frames])
        if clip == 0:
            cond = batch["jpg"][cond_index(self.T, self.use_last_frame)] if self.edit else self.cond_frame
            batch["final_cond_zero"] = condition_from_frame(cond, self.T, self.use_last_frame)
        return batch

    def __getitem__(self, idx):
        if idx != 0:
            raise IndexError(idx)
        if self.clips == 1:
            return self._clip(0)
        return {"clips": [self._clip(k) for k in range(self.clips)]}


def load_config(paths, overrides=()):
    cfg = {}
    for p in paths:
        with open(p) as f:
            new = yaml.safe_load(f)
        cfg = _merge(cfg, new)
    for ov in overrides:                                       # key.sub.key=value (OmegaConf dotlist style)
        k, v = ov.split("=", 1)
        node = cfg
        parts = k.split(".")
        for part in parts[:-1]:
            node = _child(node, part, k)
        if isinstance(node, list):
            node[_list_index(node, parts[-1], k)] = yaml.safe_load(v)
        else:
            node[parts[-1]] = yaml.safe_load(v)
    return cfg


def _list_index(node: list, part: str, key: str) -> int:
    """A numeric path component indexes an existing list entry (emb_models.0.params...)."""
    if not part.isdigit() or int(part) >= len(node):
        raise KeyError(f"override {key!r}: {part!r} does not index the {len(node)}-entry list here")
    return int(part)


def _child(node, part: str, key: str):
    if isinstance(node, list):
        return node[_list_index(node, part, key)]
    return node.setdefault(part, {})


def _merge(a, b):
    if isinstance(a, dict) and isinstance(b, dict):
        out = dict(a)
        for k, v in b.items():
            out[k] = _merge(a[k], v) if k in a else v
        return out
    return b


def model_load_ckpt(model, path):
    """inference.py:198-228: engine checkpoints (.ckpt, DeepSpeed prefix `_forward_module.` stripped) or safetensors;
    loaded non-strictly like the reference."""
    if path.endswith("ckpt"):
        sd = torch.load(path, map_location="cpu")
        sd = sd.get("state_dict", sd.get("module", sd))
        sd = {k.replace("_forward_module.", ""): v for k, v in sd.items()}
    elif path.endswith("safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        raise NotImplementedError(path)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    print(f"Restored from {path} with {len(missing)} missing and {len(unexpected)} unexpected keys")
    return model


def get_parser():
    p = argparse.ArgumentParser()
    p.add_argument("-n", "--name", type=str, default="")
    p.add_argument("-b", "--base", nargs="*", default=[], help="YAML configs, merged left to right")
    p.add_argument("--inferdir", type=str, default="inferences")
    p.add_argument("--ckptpath", type=str, default=None)
    p.add_argument("--split", type=str, default="val")
    p.add_argument("--use_last_frame", type=lambda v: str(v).lower() in ("1", "true", "yes", "y", "t"), default=True)
    p.add_argument("-s", "--seed", type=int, default=D.BASE_SEED)
    p.add_argument("--bs", type=int, default=1)
    p.add_argument("--dataset", type=str, default=None, help="module:Class of a dataset with the MyDataset batch contract")
    p.add_argument("--num_sequences", type=int, default=2)
    p.add_argument("--image_hw", type=int, nargs=2, default=(256, 512), help="per-view image size of the synthetic or layout dataset")
    p.add_argument("--layout", type=str, default=None, help="scene file (.npz) whose layout maps condition the clips (DESIGN.md section 12)")
    p.add_argument("--cond_frame", type=str, default=None, help="conditioning frame of a --layout scene, an [H, 6w] RGB image")
    p.add_argument("--gather", action="store_true", help="gather decoded frames on rank 0 and let rank 0 write them")
    p.add_argument("--randomize_zero_init", action="store_true", help="re-draw the reference's zero-initialised tails (no checkpoint)")
    p.add_argument("--clips", type=_positive_int, default=1,
                   help="clips per scene: each clip after the first is conditioned on a frame of the one before (DESIGN.md section 11)")
    p.add_argument("--overlap", type=int, default=None,
                   help="frames consecutive clips of a scene share: each clip keeps the previous clip's latents for them and "
                        "generates the rest; needs --clips >= 2 and 1 <= M <= T-1 (DESIGN.md section 11)")
    p.add_argument("--strength", type=float, default=None,
                   help="edit each item's recorded frames: re-denoise their latent from this fraction of the schedule, in (0, 1] "
                        "(DESIGN.md section 13)")
    p.add_argument("--mask_from", type=str, default=None,
                   help="original scene file: with --layout EDITED.npz --strength, regenerate only where the layouts differ")
    p.add_argument("--mask_dilate", type=int, default=1, help="latent cells the --mask_from change mask grows by within a panel")
    p.add_argument("--mask_image", type=str, default=None,
                   help="user-drawn edit mask: an [H, 6w] image (>= 128 regenerates) for every frame, or a .npy bool/uint8 "
                        "[T, H, 6w]; needs --strength, grows by --mask_dilate cells and is united with --mask_from")
    p.add_argument("--composite", type=int, default=None,
                   help=f"paste the recorded pixels back outside the edit mask with a feather of F pixels (0 .. {MAX_FEATHER}); "
                        "needs --strength and --mask_from or --mask_image (DESIGN.md section 13)")
    return p


def check_args(opt):
    """The editing, mask and compositing options that cannot be combined, whatever the clip length; raises ValueError
    naming the flag. main runs this before it reads the config."""
    if opt.strength is not None:
        if not 0.0 < opt.strength <= 1.0:
            raise ValueError(f"--strength must lie in (0, 1], got {opt.strength}")
        if opt.clips > 1:
            raise ValueError("--strength edits one recorded clip; it cannot be combined with --clips > 1")
        if opt.cond_frame is not None:
            raise ValueError("--strength conditions on the clip's own recorded frame; --cond_frame cannot be given with it")
    if opt.mask_from is not None:
        if opt.layout is None:
            raise ValueError("--mask_from compares the --layout scene with the original: it needs --layout EDITED.npz")
        if opt.strength is None:
            raise ValueError("--mask_from regenerates part of a recorded clip: it needs --strength")
    if opt.mask_dilate < 0:
        raise ValueError(f"--mask_dilate must be >= 0, got {opt.mask_dilate}")
    if opt.mask_image is not None and opt.strength is None:
        raise ValueError("--mask_image regenerates part of a recorded clip: it needs --strength")
    if opt.composite is not None:
        if opt.strength is None:
            raise ValueError("--composite pastes the recorded pixels back into an edit: it needs --strength")
        if opt.mask_from is None and opt.mask_image is None:
            raise ValueError("--composite needs an edit mask (--mask_from or --mask_image): without one every cell is "
                             "regenerated and nothing is pasted back")
        if not 0 <= opt.composite <= MAX_FEATHER:
            raise ValueError(f"--composite must lie in 0 .. {MAX_FEATHER} pixels, got {opt.composite}")


def check_clip_args(opt, num_frames: int):
    """The scene and mask options checked against clips of `num_frames` frames, before any device work; raises
    ValueError naming the flag. Returns the --mask_image pixels, uint8 [T, H, 6w] on the host, or None."""
    if opt.overlap is not None:
        if opt.clips < 2:
            raise ValueError(f"--overlap shares frames between consecutive clips: it needs --clips >= 2, got {opt.clips}")
        check_overlap(opt.overlap, num_frames)
    if opt.mask_image is None:
        return None
    try:
        return L.read_edit_mask(opt.mask_image, num_frames, tuple(opt.image_hw))
    except (ValueError, OSError) as e:
        raise ValueError(f"--mask_image: {e}") from e


def num_frames(config) -> int:
    return config["model"]["params"]["network_config"]["params"].get("num_frames", 8)


def _positive_int(v) -> int:
    n = int(v)
    if n < 1:
        raise argparse.ArgumentTypeError(f"must be >= 1, got {v}")
    return n


def make_dataset(opt, config):
    """A `--layout` scene file, `--dataset module:Class` (constructed with `clips=` only for scenes and `overlap=` only
    when --overlap is given, so a one-clip dataset needs no such keyword) or the synthetic dataset; with --clips K > 1
    every item is a scene `{"clips": [K clip batches]}`."""
    T = num_frames(config)
    if opt.layout:
        return LayoutDataset(opt.layout, T, tuple(opt.image_hw), opt.use_last_frame, opt.clips, cond_frame=opt.cond_frame,
                             edit=opt.strength is not None, overlap=opt.overlap)
    if opt.dataset:
        mod, cls = opt.dataset.split(":")
        kw = {"clips": opt.clips} if opt.clips > 1 else {}
        if opt.overlap is not None:
            kw["overlap"] = opt.overlap
        return getattr(importlib.import_module(mod), cls)(split=opt.split, use_last_frame=opt.use_last_frame, **kw)
    return SyntheticBEVDataset(opt.num_sequences, T, tuple(opt.image_hw), opt.use_last_frame, seed=opt.seed, clips=opt.clips,
                               overlap=opt.overlap)


def main(argv=None):
    opt, unknown = get_parser().parse_known_args(argv)
    if not opt.name:
        raise ValueError("You must specify the experiment name!!")
    check_args(opt)
    assert opt.bs == 1, "the reference runs batch size 1 (one sequence per rank and step)"
    inferdir = os.path.join(opt.inferdir, opt.name)
    config = load_config(opt.base, unknown)
    drawn = check_clip_args(opt, num_frames(config))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group(backend="nccl", device_id=torch.device("cuda", local))
        rank = dist.get_rank()
    else:
        rank, local = 0, 0
        torch.cuda.set_device(0)
    seed = rank + opt.seed                                     # inference.py:250
    torch.manual_seed(seed)
    device = torch.device("cuda", local)

    dataset = make_dataset(opt, config)
    mask = None
    if opt.mask_from:
        mask = L.change_mask(L.load_scene(opt.mask_from), dataset.scene, dataset.frames(0), tuple(opt.image_hw),
                             opt.mask_dilate, device)
    if drawn is not None:
        cells = L.mask_cells(drawn, opt.mask_dilate, device)
        mask = cells if mask is None else torch.maximum(mask, cells)
    sampler = DistributedSampler(dataset, num_replicas=world, rank=rank, shuffle=False)
    loader = DataLoader(dataset, batch_size=opt.bs, sampler=sampler)

    model = instantiate_from_config(config["model"])
    if opt.ckptpath is not None:
        model = model_load_ckpt(model, opt.ckptpath)
    elif opt.randomize_zero_init:
        model.model.diffusion_model.randomize_zero_init(seed=opt.seed)
        model.model.diffusion_model.controlnet.randomize_zero_init(seed=opt.seed + 1)
    model.to(device).eval()

    all_time, written = 0.0, []
    for idx, batch in enumerate(loader):
        start = time.time()
        if opt.clips > 1:
            written += _run_scene(model, batch, opt, inferdir, world, device)
            all_time += time.time() - start
            if rank == 0:
                print(f"idx {idx}: time per scene {time.time() - start:.2f}s ({opt.clips} clips), avg {all_time / (idx + 1):.2f}s",
                      flush=True)
            continue
        for key in batch:
            if key not in ("txt", "filenames"):
                batch[key] = batch[key].to(device)
        with torch.no_grad():
            outs = model.log_images(batch) if opt.strength is None else \
                model.edit_images(batch, opt.strength, mask, composite=opt.composite)
        filenames = batch["filenames"]
        samples = outs["samples"]
        if opt.gather and world > 1:                           # BASELINE.json configs[2]: NCCL gather of decoded frames
            for frames, names in D.gather_named_on_rank0(samples, filenames):
                written += IO.logs_frames(frames, os.path.join(inferdir, "fake"), names)
        else:
            written += IO.logs_frames(samples, os.path.join(inferdir, "fake"), filenames)
        written += IO.logs_all_images(outs, os.path.join(inferdir, "allimages"), filenames)
        written += IO.logs_all_gifs(outs, os.path.join(inferdir, "gifs"), filenames, num_frames=samples.shape[0])
        all_time += time.time() - start
        if rank == 0:
            print(f"idx {idx}: time per iter {time.time() - start:.2f}s, avg {all_time / (idx + 1):.2f}s", flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return written


def _run_scene(model, item, opt, inferdir, world, device) -> list[str]:
    """One scene of `opt.clips` clips (`DiffusionEngine3D.sample_scene`, sharing `opt.overlap` frames), written as one
    chronological sequence per camera plus one PNG strip and one GIF; `--gather` gathers one scene per rank on rank 0."""
    clips = item["clips"]
    if len(clips) != opt.clips:
        raise ValueError(f"--clips {opt.clips}, but the dataset item holds {len(clips)} clips")
    with torch.no_grad():
        out = model.sample_scene(clips, use_last_frame=opt.use_last_frame, overlap=opt.overlap)
    frames, names = out["samples"], out["filenames"]
    if opt.gather and world > 1:
        return [w for f, n in D.gather_named_on_rank0(frames.to(device), names) for w in IO.logs_scene(f, inferdir, n)]
    return IO.logs_scene(frames, inferdir, names)


if __name__ == "__main__":
    main()
