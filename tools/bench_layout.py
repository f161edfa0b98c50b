"""Times the rendering of one clip's 19-channel layout maps (panacea_b200/layout.py) at 256 x 512 per view, T = 8, on
the seeded 256 x 512 golden scene: the kernel alone (CUDA events around pn_render_layout, after warm-up) and the whole
`render_layout` call (host geometry, upload, launch; a host clock around work that ends in a synchronise). Prints one
JSON line with the card's name and power limit.

  python tools/bench_layout.py [--reps 50]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    from panacea_b200 import _lib, layout as L
    from panacea_b200.frame_io import CAMERA_VIEWS
    from test_layout_cpu import golden, scene_arrays, write_scene
    from tools.bench_vae import card
    assert torch.cuda.is_available(), "bench_layout needs a CUDA device"
    g = golden("layout_512")
    H, w = g["image_hw"]
    with tempfile.TemporaryDirectory() as tmp:
        scene = L.load_scene(write_scene(Path(tmp), scene_arrays(g)))
    frames = list(range(scene.num_frames))

    for _ in range(3):
        out = L.render_layout(scene, frames, H, w)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.reps):
        out = L.render_layout(scene, frames, H, w)
    torch.cuda.synchronize()
    call_ms = (time.perf_counter() - t0) / args.reps * 1e3

    per_panel = [L.panel_primitives(scene, f, cam, H, w) for f in frames for cam in CAMERA_VIEWS]
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum([len(p) for p in per_panel])]).astype(np.int32)).cuda()
    prims = torch.from_numpy(np.concatenate(per_panel)).cuda()
    rays = torch.from_numpy(L.ray_params(scene, H, w)).cuda()
    lib, ptr = _lib.load(), lambda t: C.c_void_p(t.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    launch = lambda: _lib.check(lib.pn_render_layout(ptr(prims), ptr(offsets), ptr(rays), ptr(out), len(frames), H, w, stream),
                                "pn_render_layout")
    for _ in range(5):
        launch()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.reps):
        launch()
    end.record()
    torch.cuda.synchronize()
    kernel_ms = start.elapsed_time(end) / args.reps
    out_bytes = out.numel() * out.element_size()
    print("LAYOUT_BENCH " + json.dumps({
        "card": card(), "frames": len(frames), "image_hw": [H, w], "primitives": int(prims.shape[0]),
        "kernel_ms": kernel_ms, "render_layout_call_ms": call_ms, "output_gb": out_bytes / 1e9,
        "kernel_write_gb_per_s": out_bytes / kernel_ms / 1e6}))


if __name__ == "__main__":
    main()
