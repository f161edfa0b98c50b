"""Scene files and the host geometry of the layout renderer (panacea_b200/layout.py, DESIGN.md section 12), against
goldens of the reference's dataset code (tools/make_layout_golden.py): validation of scene files, clip slicing, the
box-corner helper, and the 2-D boxes, depths and kept polyline points, which must equal the reference's exactly."""
import numpy as np
import pytest
import torch

from panacea_b200 import layout as L
from panacea_b200.frame_io import CAMERA_VIEWS
from panacea_b200.scene import scene_slices

GOLDENS = ["layout_448", "layout_512"]


def golden(name):
    from pathlib import Path
    return torch.load(Path(__file__).resolve().parent / "golden" / f"{name}.pt", weights_only=True)


def scene_arrays(g):
    return {k: (np.array(v) if isinstance(v, list) else v.numpy()) for k, v in g["scene"].items()}


def write_scene(tmp_path, arrays, name="scene.npz"):
    path = tmp_path / name
    np.savez(path, **arrays)
    return path


@pytest.mark.parametrize("name", GOLDENS)
def test_corner_helper_matches_the_golden_corners(name):
    g = golden(name)
    got = L.box_corners(g["boxes"].numpy())
    want = g["scene"]["corners"].numpy()
    assert got.shape == want.shape
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-5)       # the golden's corners are mmdet3d's fp32 arithmetic


@pytest.mark.parametrize("name", GOLDENS)
def test_host_geometry_equals_the_reference_intermediates(name, tmp_path):
    g = golden(name)
    H, W = g["image_hw"]
    scene = L.load_scene(write_scene(tmp_path, scene_arrays(g)))
    dropped = partial = 0
    for t, want in enumerate(g["intermediates"]):
        for p, cam in enumerate(CAMERA_VIEWS):
            ann = L.project_boxes(scene.corners[t], scene.labels[t], scene.lidar2img[cam], H, W)
            assert np.array_equal(ann["bbox"], want["bbox"][p].numpy().reshape(-1, 4)), (t, cam)
            assert np.array_equal(ann["depth"], want["depth"][p].numpy()), (t, cam)
            assert np.array_equal(ann["label"], want["label"][p].numpy()), (t, cam)
            assert np.array_equal(ann["corners"], want["corners"][p].numpy().reshape(-1, 8, 2)), (t, cam)
            for (cls, pts), kept in zip(scene.polylines[t], want["lines"][p], strict=True):
                got = L.project_polyline(L.resample_polyline(pts), scene.lidar2img[cam], H, W)
                assert np.array_equal(got, kept.numpy().reshape(-1, 2)), (t, cam, cls)
                partial += 0 < len(got) < L.MAP_SAMPLES
            dropped += len(scene.corners[t]) - len(ann["bbox"])
    assert dropped > 0 and partial > 0


def _base(tmp_path):
    arrays = scene_arrays(golden("layout_512"))
    return arrays, lambda **changes: write_scene(tmp_path, {**arrays, **changes})


@pytest.mark.parametrize("change, message", [
    (lambda a: {"labels": a["labels"] * 0 + 10}, "labels"),
    (lambda a: {"labels": a["labels"][:-1]}, "labels|box_frame"),
    (lambda a: {"box_frame": a["box_frame"] + 8}, "box_frame"),
    (lambda a: {"corners": np.where(np.arange(a["corners"].size).reshape(a["corners"].shape) == 5, np.nan, a["corners"])}, "finite"),
    (lambda a: {"corners": a["corners"][:, :4]}, "corners"),
    (lambda a: {"lidar2img": a["lidar2img"][:5]}, "lidar2img"),
    (lambda a: {"lidar2img": a["lidar2img"] * np.array([1, 1, 1, 0])[None, :, None]}, "invertible"),
    (lambda a: {"cameras": np.array(["CAM_FRONT"] * 6)}, "cameras"),
    (lambda a: {"num_frames": np.array(0)}, "num_frames"),
    (lambda a: {"map_labels": a["map_labels"] + 3}, "map_labels"),
    (lambda a: {"map_lengths": a["map_lengths"] + 1}, "map_lengths"),
    (lambda a: {"map_points": np.full_like(a["map_points"], np.inf)}, "finite"),
])
def test_scene_validation_rejects_bad_input(tmp_path, change, message):
    arrays, write = _base(tmp_path)
    with pytest.raises(L.SceneError, match=message):
        L.load_scene(write(**change(arrays)))


def test_scene_validation_rejects_missing_and_doubled_keys(tmp_path):
    arrays, _ = _base(tmp_path)
    with pytest.raises(L.SceneError, match="lidar2img"):
        L.load_scene(write_scene(tmp_path, {k: v for k, v in arrays.items() if k != "lidar2img"}))
    boxes = np.zeros((len(arrays["labels"]), 7))
    with pytest.raises(L.SceneError, match="exactly one"):
        L.load_scene(write_scene(tmp_path, {**arrays, "boxes": boxes}))


def test_boxes_key_gives_the_helper_corners(tmp_path):
    g = golden("layout_448")
    arrays = scene_arrays(g)
    del arrays["corners"]
    scene = L.load_scene(write_scene(tmp_path, {**arrays, "boxes": g["boxes"].numpy()}))
    want = L.box_corners(g["boxes"].numpy()).astype(np.float32)
    assert np.array_equal(np.concatenate(scene.corners), want[np.argsort(arrays["box_frame"], kind="stable")])


def _layout_dataset(tmp_path, clips, T, use_last_frame, frames=None):
    from PIL import Image
    from panacea_b200.inference import LayoutDataset
    arrays = scene_arrays(golden("layout_512"))
    F = clips * (T - 1) + 1 if frames is None else frames
    keep = arrays["box_frame"] < F
    mkeep = arrays["map_frame"] < F
    starts = np.concatenate([[0], np.cumsum(arrays["map_lengths"])[:-1]])
    pts = np.concatenate([arrays["map_points"][s:s + n] for s, n, k in zip(starts, arrays["map_lengths"], mkeep) if k])
    Image.fromarray(np.zeros((32, 6 * 64, 3), np.uint8)).save(tmp_path / "cond.png")
    path = write_scene(tmp_path, {**arrays, "num_frames": np.array(F), "box_frame": arrays["box_frame"][keep],
                                  "labels": arrays["labels"][keep], "corners": arrays["corners"][keep],
                                  "map_frame": arrays["map_frame"][mkeep], "map_labels": arrays["map_labels"][mkeep],
                                  "map_lengths": arrays["map_lengths"][mkeep], "map_points": pts,
                                  "cond_frame": np.array("cond.png")})
    return LayoutDataset(path, T, (32, 64), use_last_frame, clips, device="cpu")


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("clips", [1, 2, 3])
def test_clip_frames_follow_scene_slices(tmp_path, clips, use_last_frame):
    T = 4
    ds = _layout_dataset(tmp_path, clips, T, use_last_frame)
    covered = []
    for k, lo, hi in scene_slices(clips, T, use_last_frame):
        covered += ds.frames(k)[lo:hi]
    assert covered == list(range(clips * (T - 1) + 1))             # chronological, every frame once
    a = T - 1 if use_last_frame else 0
    for k in range(1, clips):                   # clip k's conditioning frame is clip k-1's hand-off frame
        assert ds.frames(k)[a] == ds.frames(k - 1)[T - 1 - a]


def test_layout_dataset_rejects_a_wrong_frame_count_and_a_missing_frame(tmp_path):
    with pytest.raises(L.SceneError, match="frames"):
        _layout_dataset(tmp_path, 2, 4, True, frames=8)
    from panacea_b200.inference import LayoutDataset
    arrays = scene_arrays(golden("layout_512"))
    path = write_scene(tmp_path, arrays)
    with pytest.raises(L.SceneError, match="conditioning frame"):
        LayoutDataset(path, 8, (256, 512), True, 1, device="cpu")


def test_caption_counts_the_classes():
    assert L.caption([0, 0, 8, 9]) == ("A street scene seen by six surround-view cameras, with 4 objects: 2 car, "
                                       "1 pedestrian, 1 traffic cone.")
