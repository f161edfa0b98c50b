"""Measures pasting the recorded pixels back outside an edit (DESIGN.md section 13) and prints one JSON line with the
card's name and power limit:

  * CUDA-event time of pn_composite_frames at T = 8, 256 x 512 per view, feather 0, 8, 32 and 64, on seeded frames and
    a seeded cell mask (about a quarter of the cells regenerated, in blobs), after warm-up; GB/s against the bytes the
    algorithm must move: decoded and recorded read (2 x 75.5 MB), the frames written (75.5 MB) and alpha (25.2 MB);
  * CUDA-event time of pn_mask_cells (pooling plus dilation by 1) on a drawn uint8 mask of the same clip;
  * wall time of one full-size bf16 `edit_images` at strength 0.6 with the same mask, with and without composite=8,
    alternated after one warm-up call of each (packing, graph capture), each ending in a synchronise, and the peak
    device memory of each.

  python tools/bench_composite.py [--steps 25] [--reps 2] [--kernel_reps 100]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

T, H, W = 8, 256, 512


def _events(fn, reps):
    for _ in range(5):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def _cell_mask(g):
    """[T, H/8, 6W/8] regenerated blobs: random cells grown by two cells, about a quarter of the clip."""
    from panacea_b200 import layout as L
    seeds = (g.random((T, H, 6 * W)) < 2e-4).astype(np.uint8)
    return L.mask_cells(seeds, 2)


def kernels(reps):
    from panacea_b200 import layout as L
    from panacea_b200.composite import composite_frames
    g = np.random.default_rng(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    rec = torch.randint(0, 256, (T, 3, H, 6 * W), device="cuda", generator=gen).float() / 127.5 - 1.0
    dec = torch.rand((T, 3, H, 6 * W), device="cuda", generator=gen) * 2.0 - 1.0
    cells = _cell_mask(g)
    frame_bytes = dec.numel() * 4
    moved = 3 * frame_bytes + T * H * 6 * W * 4
    res = {"frames": T, "image_hw": [H, W], "regenerated_cells": float(cells.mean().item()),
           "bytes_moved": moved, "composite": {}}
    for f in (0, 8, 32, 64):
        ms = _events(lambda: composite_frames(dec, rec, cells, f), reps)
        res["composite"][str(f)] = {"ms": ms, "gb_per_s": moved / ms / 1e6}
    drawn = (g.random((T, H, 6 * W)) < 1e-3).astype(np.uint8)
    d_drawn = torch.from_numpy(drawn).cuda()
    import ctypes as C
    from panacea_b200 import _lib
    out = torch.empty(T, H // 8, 6 * W // 8, device="cuda")
    lib, stream = _lib.load(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res["mask_cells_ms"] = _events(lambda: _lib.check(lib.pn_mask_cells(C.c_void_p(d_drawn.data_ptr()), C.c_void_p(out.data_ptr()),
                                                                      T, H, W, 8, 1, stream), "pn_mask_cells"), reps)
    assert torch.equal(out, L.mask_cells(drawn, 1))
    return res


def clips(steps, reps):
    from tools.bench_scene import full_size_engine, scene_clips
    m = full_size_engine(steps=steps)
    batch = {k: v.cuda() if isinstance(v, torch.Tensor) else v for k, v in scene_clips(1)[0].items()}
    mask = _cell_mask(np.random.default_rng(1))
    runs = {"edit": lambda: m.edit_images(batch, 0.6, mask=mask),
            "edit_composite8": lambda: m.edit_images(batch, 0.6, mask=mask, composite=8)}
    times, peak = {k: [] for k in runs}, {}
    for k, fn in runs.items():                                    # packing, graph capture
        fn()
    for _ in range(reps):
        for k, fn in runs.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
            peak[k] = max(peak.get(k, 0), torch.cuda.max_memory_allocated())
    return {"steps": steps, "strength": 0.6, "regenerated_cells": float(mask.mean().item()),
            **{f"{k}_s": v for k, v in times.items()}, **{f"{k}_peak_gb": v / 1e9 for k, v in peak.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--kernel_reps", type=int, default=100)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_composite needs a CUDA device"
    from tools.bench_vae import card
    torch.manual_seed(0)
    rec = {"card": card(), "kernels": kernels(args.kernel_reps), "clip_bf16": clips(args.steps, args.reps)}
    print("COMPOSITE_BENCH " + json.dumps(rec))


if __name__ == "__main__":
    main()
