"""Measures the editing path (DESIGN.md section 13) and prints one JSON line with the card's name and power limit:

  * wall time per clip of `log_images` (generation from noise) against `edit_images` at strength 0.6 with a change
    mask over half the latent, on the full-size bf16 engine (random weights, 8 frames at 256 x 512 per view), each
    timed by a host clock ending in a synchronise, after one warm-up call of each (packing, graph capture), alternated;
  * CUDA-event time of one pn_sampler_step launch against one pn_sampler_step_known launch (Euler, CFG halves, next
    network input written) on a state of 16 M elements (64 MB per buffer, larger than the 50 MB L2), with a soft mask
    (every element blended) and with mask 1 (no element blended);
  * CUDA-event time of pn_layout_change_mask (two launches, dilate 1) on two renders of the seeded 256 x 512 golden
    scene, T = 8.

  python tools/bench_edit.py [--steps 25] [--reps 2] [--kernel_reps 50]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def _events(fn, reps):
    for _ in range(3):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def step_kernels(reps):
    from panacea_b200.ops import SAMPLER_EULER, NativeOps
    ops = NativeOps()
    shape = (16, 4, 512, 512)                                    # 16 M elements
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(shape, device="cuda", generator=g)
    net = torch.randn((2 * shape[0],) + shape[1:], device="cuda", generator=g)
    x_in = torch.empty_like(net)
    known = torch.randn(shape, device="cuda", generator=g)
    soft = torch.rand((shape[0], *shape[2:]), device="cuda", generator=g)
    ones = torch.ones_like(soft)
    kw = dict(x_in_next=x_in, halves=2, sigma_q=3.0, cfg_scale=5.0, sigma=3.0, dt=-0.5, c_in_next=0.3)
    blend = lambda m: dict(known=known, mask=m, known_seed=7, known_draw=1, known_sigma=2.5)
    res = {"elements": x.numel(),
           "plain_ms": _events(lambda: ops.sampler_step(SAMPLER_EULER, x, net, **kw), reps),
           "known_soft_mask_ms": _events(lambda: ops.sampler_step(SAMPLER_EULER, x, net, **kw, **blend(soft)), reps),
           "known_mask_one_ms": _events(lambda: ops.sampler_step(SAMPLER_EULER, x, net, **kw, **blend(ones)), reps)}
    # bytes the plain launch must move: x read + write, 2 halves of net read, 2 halves of x_in written
    res["plain_gb_per_s"] = 6 * x.numel() * 4 / res["plain_ms"] / 1e6
    return res


def mask_kernel(reps):
    from panacea_b200 import _lib, layout as L
    from test_layout_cpu import golden, scene_arrays, write_scene
    g = golden("layout_512")
    H, w = g["image_hw"]
    arrays = scene_arrays(g)
    edited = dict(arrays, corners=arrays["corners"].copy())
    edited["corners"][0] += np.array([3.0, 0.0, 0.0], np.float32)
    with tempfile.TemporaryDirectory() as tmp:
        a = L.load_scene(write_scene(Path(tmp), arrays, "a.npz"))
        b = L.load_scene(write_scene(Path(tmp), edited, "b.npz"))
    frames = list(range(a.num_frames))
    ra, rb = L.render_layout(a, frames, H, w), L.render_layout(b, frames, H, w)
    out = torch.empty(len(frames), H // 8, 6 * w // 8, device="cuda")
    lib, ptr = _lib.load(), lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ms = _events(lambda: _lib.check(lib.pn_layout_change_mask(ptr(ra), ptr(rb), ptr(out), len(frames), H, w, 8, 1, stream),
                                    "pn_layout_change_mask"), reps)
    read = 2 * ra.numel() * 4
    return {"frames": len(frames), "image_hw": [H, w], "kernel_ms": ms, "read_gb_per_s": read / ms / 1e6,
            "changed_cells": int(out.sum().item())}


def clips(steps, reps):
    from tools.bench_scene import full_size_engine, scene_clips
    m = full_size_engine(steps=steps)
    batch = {k: v.cuda() if isinstance(v, torch.Tensor) else v for k, v in scene_clips(1)[0].items()}
    mask = torch.ones(8, 32, 6 * 64, device="cuda")
    mask[:, :, : 3 * 64] = 0.0                                    # three of the six views kept
    runs = {"log_images": lambda: m.log_images(batch), "edit_images": lambda: m.edit_images(batch, 0.6, mask=mask)}
    times = {k: [] for k in runs}
    for k, fn in runs.items():                                    # packing, graph capture
        fn()
    for _ in range(reps):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    return {"steps": steps, "strength": 0.6, "evaluations_edit": m.sampler.plan(None, 0.6)[1].__len__(),
            "log_images_s": times["log_images"], "edit_images_s": times["edit_images"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--kernel_reps", type=int, default=50)
    args = ap.parse_args()
    from tools.bench_vae import card
    assert torch.cuda.is_available(), "bench_edit needs a CUDA device"
    torch.manual_seed(0)
    rec = {"card": card(), "sampler_step": step_kernels(args.kernel_reps), "change_mask": mask_kernel(args.kernel_reps),
           "clip_bf16": clips(args.steps, args.reps)}
    print("EDIT_BENCH " + json.dumps(rec))


if __name__ == "__main__":
    main()
