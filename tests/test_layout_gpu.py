"""The layout renderer on the GPU (pn_render_layout, DESIGN.md section 12) against the reference's hints of two seeded
scenes (tests/golden/layout_*.pt, written by tools/make_layout_golden.py):

  * channels 3..12 (class depth) are bitwise the reference's;
  * channels 16..18 (rays) are within one level, and at least 99.99 % exact;
  * channels 0..2 (boxes) and 13..15 (map) differ almost only within 2 px of an edge pixel of the reference (a pixel
    whose 3 x 3 neighbourhood is not constant), and their ink masks (any channel < 255) overlap the reference's in
    every panel with >= 200 ink pixels. The kernel does not restate OpenCV's scan conversion, so lines 3 or 5 px wide
    land a pixel off here and there, which costs thin-line panels much of their IoU. Bounds, from the worst values
    measured on the two goldens (printed as LAYOUT lines): at most 0.01 % of a group's pixels farther than 2 px from
    an edge (measured 146 of 5.5 M, box fills that meet the canvas border), ink IoU >= 0.80 for boxes and >= 0.85
    for map lines (measured 0.83 and 0.89);
  * two renders are bitwise equal;
  * the inference entry point with --layout and --clips 2 writes the scene and feeds each clip the renderer's hint."""
import json
import os
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_layout_cpu import GOLDENS, golden, scene_arrays, write_scene

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
MIN_INK_IOU = {"boxes": 0.80, "map": 0.85}


def unpack(p):
    return torch.from_numpy(np.frombuffer(zlib.decompress(p["zlib"]), np.uint8).reshape(p["shape"]).copy())


def render(g, tmp_path):
    from panacea_b200 import layout as L
    H, w = g["image_hw"]
    scene = L.load_scene(write_scene(tmp_path, scene_arrays(g)))
    return L.render_layout(scene, range(scene.num_frames), H, w)


def as_levels(out):
    """The uint8 levels k of a hint, checking every value is fp32 k / 255 correctly rounded, as numpy divides."""
    out = out.cpu()
    levels = torch.round(out * 255.0).to(torch.int64).clamp(0, 255)
    table = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255.0))
    assert torch.equal(table[levels], out), "the hint holds values other than k / 255"
    return levels.to(torch.int16)


def panels(x, w):
    """[T, C, H, 6w] -> [T * 6, C, H, w]"""
    T, C, H, _ = x.shape
    return x.reshape(T, C, H, 6, w).permute(0, 3, 1, 2, 4).reshape(T * 6, C, H, w)


def edge_mask(ref):
    """Pixels whose 3 x 3 neighbourhood (inside the panel) is not constant in any channel: [N, H, w] bool."""
    x = ref.float()
    hi = F.max_pool2d(x, 3, 1, 1)
    lo = -F.max_pool2d(-x, 3, 1, 1)
    return (hi != lo).any(1)


@pytest.mark.parametrize("name", GOLDENS)
def test_layout_matches_the_reference(name, tmp_path):
    g = golden(name)
    H, w = g["image_hw"]
    got = as_levels(render(g, tmp_path))
    ref = unpack(g["hint_0_15"]).to(torch.int16)
    rays = unpack(g["rays"]).to(torch.int16)
    T = ref.shape[0]
    assert got.shape == (T, 19, H, 6 * w)
    assert torch.equal(got[:, 3:13], ref[:, 3:13]), f"depth channels: {(got[:, 3:13] != ref[:, 3:13]).sum()} pixels differ"

    dr = (got[:, 16:19] - rays[None]).abs()
    exact = (dr == 0).double().mean().item()
    report = {"case": name, "ray_max_level_diff": int(dr.max()), "ray_exact_fraction": exact}
    assert dr.max() <= 1 and exact >= 0.9999, report

    for label, lo, hi in (("boxes", 0, 3), ("map", 13, 16)):
        a, b = panels(got[:, lo:hi], w), panels(ref[:, lo:hi], w)
        differ = (a != b).any(1)
        near = F.max_pool2d(edge_mask(b).float()[:, None], 5, 1, 2)[:, 0] > 0        # within 2 px (Chebyshev)
        far = differ & ~near
        # the largest distance of a differing pixel to an edge pixel, for the report
        dist, reach = 0, edge_mask(b).float()[:, None]
        while (differ & ~(reach[:, 0] > 0)).any() and dist < 16:
            dist += 1
            reach = F.max_pool2d(reach, 3, 1, 1)
        ink_a, ink_b = (a < 255).any(1), (b < 255).any(1)
        inter = (ink_a & ink_b).flatten(1).sum(1).double()
        union = (ink_a | ink_b).flatten(1).sum(1).double()
        counted = ink_b.flatten(1).sum(1) >= 200
        iou = (inter / union.clamp(min=1))[counted]
        report.update({f"{label}_differing_pixels": int(differ.sum()), f"{label}_far_from_edge": int(far.sum()),
                       f"{label}_max_edge_distance_px": dist, f"{label}_worst_ink_iou": float(iou.min()),
                       f"{label}_panels_with_ink": int(counted.sum())})
        assert int(far.sum()) <= 1e-4 * differ.numel() and float(iou.min()) >= MIN_INK_IOU[label], report
    print("LAYOUT " + json.dumps(report))


def test_two_renders_are_bitwise_equal(tmp_path):
    g = golden("layout_512")
    a, b = render(g, tmp_path), render(g, tmp_path)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def _small_scene(tmp_path, T, clips):
    """The 256 x 512 golden scene shrunk to 64 x 128 per view, cut to the K(T-1)+1 frames of `clips` clips."""
    from PIL import Image
    arrays = scene_arrays(golden("layout_512"))
    n = clips * (T - 1) + 1
    keep, mkeep = arrays["box_frame"] < n, arrays["map_frame"] < n
    starts = np.concatenate([[0], np.cumsum(arrays["map_lengths"])[:-1]])
    pts = np.concatenate([arrays["map_points"][s:s + k] for s, k, m in zip(starts, arrays["map_lengths"], mkeep) if m])
    l2i = arrays["lidar2img"].copy()
    l2i[:, :2] *= 0.25
    rng = np.random.default_rng(0)
    Image.fromarray(rng.integers(0, 256, (64, 6 * 128, 3), dtype=np.uint8)).save(tmp_path / "first.png")
    return write_scene(tmp_path, {**arrays, "num_frames": np.array(n), "lidar2img": l2i,
                                  "box_frame": arrays["box_frame"][keep], "labels": arrays["labels"][keep],
                                  "corners": arrays["corners"][keep], "map_frame": arrays["map_frame"][mkeep],
                                  "map_labels": arrays["map_labels"][mkeep], "map_lengths": arrays["map_lengths"][mkeep],
                                  "map_points": pts, "cond_frame": np.array("first.png")}, "drive.npz")


def test_inference_entry_point_renders_each_clip_of_a_layout_scene(tmp_path, monkeypatch):
    from panacea_b200 import inference as INF
    from panacea_b200.frame_io import CAMERA_VIEWS
    from panacea_b200.sgm.models.diffusion import DiffusionEngine3D
    T, clips = 4, 2
    path = _small_scene(tmp_path, T, clips)
    fed = []
    log_images = DiffusionEngine3D.log_images

    def recording(self, batch, *a, **k):
        fed.append(batch["cond_img"].detach().clone())
        return log_images(self, batch, *a, **k)
    monkeypatch.setattr(DiffusionEngine3D, "log_images", recording)
    written = INF.main(["--name", "layout", "--base", CFG, "--inferdir", str(tmp_path / "out"), "--layout", str(path),
                        "--image_hw", "64", "128", "--clips", str(clips), "--randomize_zero_init"])
    fake = tmp_path / "out" / "layout" / "fake"
    dirs = sorted(os.listdir(fake))
    last = clips * (T - 1)
    assert dirs == sorted(f"{cam}_drive__{cam}__{last:06d}" for cam in CAMERA_VIEWS)
    for d in dirs:
        assert sorted(os.listdir(fake / d)) == [f"_{i:06}.jpg" for i in range(clips * (T - 1) + 1)]
    assert len([p for p in written if p.endswith(".gif")]) == 1 and len([p for p in written if p.endswith(".png")]) == 1
    want = INF.LayoutDataset(path, T, (64, 128), True, clips)[0]["clips"]
    assert len(fed) == clips
    for k in range(clips):
        assert fed[k].shape == (1, T, 19, 64, 768)
        assert torch.equal(fed[k][0], want[k]["cond_img"]), k
    assert not torch.equal(want[0]["cond_img"], want[1]["cond_img"])
