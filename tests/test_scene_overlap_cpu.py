"""Scenes whose clips share m frames (panacea_b200/scene.py with `overlap`, DiffusionEngine3D.sample_scene(overlap=),
inference --overlap): the host logic without a GPU — frame accounting and hand-off indices for every m, the unchanged
results of `overlap=None`, the known region of a carrying clip, option checks that come before any device work, the
datasets' shared-frame contract, and the routing of carrying clips to `outpaint_images`."""
import sys
import types
from pathlib import Path

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from panacea_b200 import layout as L
from panacea_b200 import scene as S

ROOT = Path(__file__).resolve().parent.parent
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
CASES = [(T, m) for T in (2, 4, 8) for m in range(1, T)]


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("T,m", CASES)
def test_frame_numbers_cover_the_scene_once_and_shared_frames_agree(T, m, use_last_frame):
    a = S.cond_index(T, use_last_frame)
    h = S.handoff_index(T, use_last_frame, m)
    cur, prev = S.shared_frames(T, use_last_frame, m)
    assert len(cur) == len(prev) == m and a in cur
    for K in range(1, 5):
        num = [[S.scene_frame_number(k, f, K, T, use_last_frame, m) for f in range(T)] for k in range(K)]
        assert S.scene_order(num, use_last_frame, m) == list(range(K * (T - m) + m)) == list(range(S.scene_length(K, T, m)))
        assert S.scene_order([torch.tensor(n) for n in num], use_last_frame, m).tolist() == list(range(S.scene_length(K, T, m)))
        for k in range(1, K):
            assert [num[k][i] for i in cur] == [num[k - 1][j] for j in prev], (K, k)
            assert num[k][a] == num[k - 1][h], (K, k)                 # the hand-off frame is clip k's conditioning frame
            assert not set(num[k]) & set(num[k - 1]) - {num[k][i] for i in cur}
        covered = sorted(num[k][f] for k, lo, hi in S.scene_slices(K, T, use_last_frame, m) for f in range(lo, hi))
        assert covered == list(range(S.scene_length(K, T, m)))


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("T", [2, 4, 8])
def test_overlap_none_is_the_boundary_frame_scene(T, use_last_frame):
    """None keeps the boundary-frame results (restated from their definitions before `overlap` existed), and m = 1
    gives the same frame accounting."""
    a = T - 1 if use_last_frame else 0
    assert S.handoff_index(T, use_last_frame) == T - 1 - a == S.handoff_index(T, use_last_frame, 1)
    for K in range(1, 5):
        assert S.scene_length(K, T) == K * (T - 1) + 1 == S.scene_length(K, T, 1)
        want = [(k, 0, T - 1) for k in range(K - 1, 0, -1)] + [(0, 0, T)] if use_last_frame else \
            [(0, 0, T)] + [(k, 1, T) for k in range(1, K)]
        assert S.scene_slices(K, T, use_last_frame) == want == S.scene_slices(K, T, use_last_frame, 1)
        for k in range(K):
            for f in range(T):
                start = (K - 1 - k) if use_last_frame else k
                assert S.scene_frame_number(k, f, K, T, use_last_frame) == start * (T - 1) + f
                assert S.scene_frame_number(k, f, K, T, use_last_frame, 1) == start * (T - 1) + f
        per_clip = [[f"{k}:{f}" for f in range(T)] for k in range(K)]
        assert S.scene_order(per_clip, use_last_frame) == [x for k, lo, hi in want for x in per_clip[k][lo:hi]]


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("T,m", [(4, 1), (4, 2), (4, 3), (8, 4), (8, 7)])
def test_known_region_holds_the_previous_clips_shared_latents(T, m, use_last_frame):
    prev = torch.arange(T, dtype=torch.float32).reshape(T, 1, 1, 1) * 10.0 + torch.rand(T, 4, 3, 5)
    known, mask = S.known_region(prev, use_last_frame, m)
    assert known.shape == (T, 4, 3, 5) and mask.shape == (T, 3, 5) and known.dtype == mask.dtype == torch.float32
    kept = list(range(T - m, T)) if use_last_frame else list(range(m))
    src = list(range(m)) if use_last_frame else list(range(T - m, T))
    for i in range(T):
        if i in kept:
            assert torch.equal(known[i], prev[src[kept.index(i)]]) and mask[i].abs().max() == 0, i
        else:
            assert known[i].abs().max() == 0 and torch.equal(mask[i], torch.ones(3, 5)), i
    assert S.cond_index(T, use_last_frame) in kept                     # the conditioning frame is a kept frame


@pytest.mark.parametrize("bad", [0, 4, 5, -1, 2.0, True])
def test_overlap_outside_the_clip_is_refused(bad):
    with pytest.raises(ValueError, match=r"1 \.\. 3"):
        S.check_overlap(bad, 4)
    with pytest.raises(ValueError):
        S.known_region(torch.zeros(4, 4, 2, 2), True, bad)
    from panacea_b200.inference import SyntheticBEVDataset
    with pytest.raises(ValueError):
        SyntheticBEVDataset(1, 4, (16, 32), clips=3, overlap=bad)


def _main_refuses(argv, match):
    from panacea_b200 import inference as INF
    with pytest.raises(ValueError, match=match):
        INF.main(["--name", "x", "--base", CFG, "--image_hw", "16", "32", *argv])


def test_cli_refuses_an_overlap_that_cannot_work():
    """Raised before any device is touched: this machine may have none, and a ValueError is what comes back."""
    _main_refuses(["--overlap", "2"], "--clips >= 2")
    _main_refuses(["--clips", "1", "--overlap", "1"], "--clips >= 2")
    for bad in ("0", "4", "9", "-1"):
        _main_refuses(["--clips", "3", "--overlap", bad], r"1 \.\. 3")
    _main_refuses(["--clips", "3", "--overlap", "2", "--strength", "0.5"], "--clips > 1")
    from panacea_b200.inference import get_parser
    assert get_parser().parse_known_args(["--name", "x"])[0].overlap is None
    assert get_parser().parse_known_args(["--name", "x", "--overlap", "3"])[0].overlap == 3


def _stamp(name) -> int:
    from panacea_b200 import frame_io as IO
    return int(IO._name(name).split("__")[-1].split(".")[0])


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("m", [1, 2, 3])
def test_synthetic_dataset_shared_frames_carry_one_file_name(m, use_last_frame):
    from panacea_b200.inference import SyntheticBEVDataset
    K, T = 3, 4
    item = next(iter(DataLoader(SyntheticBEVDataset(1, T, (16, 32), use_last_frame, clips=K, overlap=m), batch_size=1)))
    clips = item["clips"]
    cur, prev = S.shared_frames(T, use_last_frame, m)
    for k in range(1, K):
        assert [clips[k]["filenames"][i] for i in cur] == [clips[k - 1]["filenames"][j] for j in prev]
    names = S.scene_order([c["filenames"] for c in clips], use_last_frame, m)
    assert len(names) == K * (T - m) + m
    for cam in range(6):
        stamps = [_stamp(f[cam]) for f in names]
        assert stamps == sorted(stamps) and len(set(stamps)) == len(names)
    plain = next(iter(DataLoader(SyntheticBEVDataset(1, T, (16, 32), use_last_frame, clips=K), batch_size=1)))["clips"]
    for c, p in zip(clips, plain):                                      # the overlap changes file names only
        assert torch.equal(c["cond_img"], p["cond_img"])


def _scene_file(tmp_path, n):
    """The 256 x 512 golden scene shrunk to 64 x 128 per view and cut to its first n frames."""
    from PIL import Image
    from test_layout_cpu import golden, scene_arrays, write_scene
    arrays = scene_arrays(golden("layout_512"))
    keep, mkeep = arrays["box_frame"] < n, arrays["map_frame"] < n
    starts = np.concatenate([[0], np.cumsum(arrays["map_lengths"])[:-1]])
    pts = np.concatenate([arrays["map_points"][s:s + k] for s, k, mk in zip(starts, arrays["map_lengths"], mkeep) if mk])
    l2i = arrays["lidar2img"].copy()
    l2i[:, :2] *= 0.25                                                  # the cameras at 64 x 128 per view
    Image.fromarray(np.random.default_rng(0).integers(0, 256, (64, 6 * 128, 3), dtype=np.uint8)).save(tmp_path / "first.png")
    return write_scene(tmp_path, {**arrays, "num_frames": np.array(n), "lidar2img": l2i, "box_frame": arrays["box_frame"][keep],
                                  "labels": arrays["labels"][keep], "corners": arrays["corners"][keep],
                                  "map_frame": arrays["map_frame"][mkeep], "map_labels": arrays["map_labels"][mkeep],
                                  "map_lengths": arrays["map_lengths"][mkeep], "map_points": pts,
                                  "cond_frame": np.array("first.png")}, f"drive{n}.npz")


@pytest.mark.parametrize("use_last_frame", [True, False])
def test_layout_dataset_counts_and_numbers_shared_frames(tmp_path, use_last_frame):
    from panacea_b200.inference import LayoutDataset
    K, T, m = 3, 4, 2
    ds = LayoutDataset(_scene_file(tmp_path, 8), T, (64, 128), use_last_frame, K, overlap=m)   # no render yet
    cur, prev = S.shared_frames(T, use_last_frame, m)
    frames = [ds.frames(k) for k in range(K)]
    assert sorted(set(sum(frames, []))) == list(range(8))
    for k in range(1, K):
        assert [frames[k][i] for i in cur] == [frames[k - 1][j] for j in prev]
    with pytest.raises(L.SceneError, match=r"8 frames, but 3 clips of 4 frames with 1 shared between neighbours need 10"):
        LayoutDataset(_scene_file(tmp_path, 8), T, (64, 128), use_last_frame, K, overlap=1)
    with pytest.raises(L.SceneError, match=r"10 frames, but 3 clips of 4 frames with 2 shared between neighbours need 8"):
        LayoutDataset(_scene_file(tmp_path, 10), T, (64, 128), use_last_frame, K, overlap=m)
    with pytest.raises(L.SceneError, match=r"8 frames, but 3 clips of 4 frames need 10"):
        LayoutDataset(_scene_file(tmp_path, 8), T, (64, 128), use_last_frame, K)


def test_make_dataset_passes_overlap_only_when_given(monkeypatch):
    from panacea_b200.inference import SyntheticBEVDataset, get_parser, load_config, make_dataset
    cfg = load_config([CFG])
    opt = get_parser().parse_known_args(["--name", "x", "--image_hw", "16", "32", "--clips", "2", "--overlap", "2"])[0]
    ds = make_dataset(opt, cfg)
    assert isinstance(ds, SyntheticBEVDataset) and ds.overlap == 2
    seen = []

    class Plugged:
        def __init__(self, **kw):
            seen.append(kw)
    monkeypatch.setitem(sys.modules, "plugged_ds", types.SimpleNamespace(Plugged=Plugged))
    for argv, want in ((["--clips", "4"], {"clips": 4}), (["--clips", "4", "--overlap", "3"], {"clips": 4, "overlap": 3})):
        opt = get_parser().parse_known_args(["--name", "x", "--dataset", "plugged_ds:Plugged", *argv])[0]
        make_dataset(opt, cfg)
        assert seen[-1] == {"split": "val", "use_last_frame": True, **want}


def _engine():
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.util import instantiate_from_config
    return instantiate_from_config(load_config([CFG])["model"])


@pytest.mark.parametrize("use_last_frame", [True, False])
def test_carrying_clips_go_to_outpaint_images_with_the_known_region(use_last_frame):
    """With stubs for the two clip methods: clip 0 is log_images, clip k > 0 outpaint_images with clip k-1's latent as
    its known region and the hand-off frame of `handoff_index(T, ., m)` in its image condition."""
    m = _engine()
    K, T, ov, calls = 3, 4, 2, []

    def clip(kind):
        def run(batch, *known_mask, **kw):
            calls.append((kind, batch, known_mask))
            g = torch.Generator().manual_seed(len(calls))
            return {"samples": torch.rand(T, 3, 16, 192, generator=g) * 2.4 - 1.2,
                    "sample_latents": torch.randn(T, 4, 2, 24, generator=g)}
        return run
    m.log_images, m.outpaint_images = clip("log"), clip("outpaint")
    from panacea_b200.inference import SyntheticBEVDataset
    item = next(iter(DataLoader(SyntheticBEVDataset(1, T, (16, 32), use_last_frame, clips=K, overlap=ov), batch_size=1)))
    out = m.sample_scene(item["clips"], use_last_frame=use_last_frame, overlap=ov)
    assert [c[0] for c in calls] == ["log", "outpaint", "outpaint"] and out["overlap"] == ov
    h = S.handoff_index(T, use_last_frame, ov)
    for k in range(1, K):
        known, mask = calls[k][2]
        want_k, want_m = S.known_region(out["sample_latents"][k - 1], use_last_frame, ov)
        assert torch.equal(known.cpu(), want_k) and torch.equal(mask.cpu(), want_m)
        frame = S.quantize_frame(out["clip_samples"][k - 1][h])
        assert torch.equal(out["handoff_frames"][k - 1], frame)
        assert torch.equal(calls[k][1]["final_cond_zero"].cpu(), S.condition_from_frame(frame, T, use_last_frame).unsqueeze(0))
        assert "jpg" not in calls[k][1]
    assert out["samples"].shape[0] == K * (T - ov) + ov and len(out["filenames"]) == K * (T - ov) + ov
    assert torch.equal(out["samples"], S.scene_order(out["clip_samples"], use_last_frame, ov))
    with pytest.raises(ValueError, match=r"1 \.\. 3"):
        m.sample_scene(item["clips"], overlap=4)
    calls.clear()
    assert m.sample_scene(item["clips"], use_last_frame=use_last_frame)["overlap"] is None
    assert [c[0] for c in calls] == ["log"] * K
