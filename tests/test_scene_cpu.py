"""Scenes of K chained clips (panacea_b200/scene.py, DiffusionEngine3D.sample_scene, inference --clips): the host logic
without a GPU — hand-off indices, the writer-exact quantise / dataset-exact dequantise round trip, chronological order
with the boundary frame once, continuous writer numbering, the dataset's scene contract, option parsing, and the
routing of K = 1 to the unchanged log_images path."""
from pathlib import Path

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from panacea_b200 import frame_io as IO
from panacea_b200 import scene as S

ROOT = Path(__file__).resolve().parent.parent
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")


def _stamp(name) -> int:
    return int(IO._name(name).split("__")[-1].split(".")[0])


@pytest.mark.parametrize("T", [4, 8])
def test_condition_and_handoff_indices(T):
    assert S.cond_index(T, True) == T - 1 and S.handoff_index(T, True) == 0
    assert S.cond_index(T, False) == 0 and S.handoff_index(T, False) == T - 1
    assert S.scene_length(3, T) == 3 * (T - 1) + 1


def test_handoff_quantisation_is_the_writers_then_the_datasets():
    g = torch.Generator().manual_seed(0)
    img = torch.randn(3, 16, 24, generator=g) * 0.8
    img[0, 0, :4] = torch.tensor([-3.0, -1.0, 1.0, 3.0])                      # clamped ends
    got = S.quantize_frame(img)
    u8 = (((img.clamp(-1.0, 1.0) + 1.0) / 2.0).permute(1, 2, 0).numpy() * 255).astype(np.uint8)   # inference.py:160-166
    assert np.array_equal(IO._to_uint8_hwc(img), u8)
    want = torch.from_numpy(u8.astype(np.float32) / 127.5 - 1.0).permute(2, 0, 1)               # dataset.py:551-552
    assert got.dtype == torch.float32 and got.shape == img.shape and torch.equal(got, want)
    assert got[0, 0, :4].tolist() == [-1.0, -1.0, 1.0, 1.0]
    assert (got - img.clamp(-1.0, 1.0)).abs().max().item() <= 2.0 / 255.0 + 1e-6
    cond = S.condition_from_frame(got, 4, True)
    assert cond.shape == (4, 3, 16, 24) and torch.equal(cond[3], got) and cond[:3].abs().max() == 0
    cond = S.condition_from_frame(got, 4, False)
    assert torch.equal(cond[0], got) and cond[1:].abs().max() == 0


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("K", [1, 2, 3])
def test_scene_order_is_chronological_with_the_boundary_once(K, use_last_frame):
    T = 4
    clips = [torch.tensor([[100.0 * k + f] for f in range(T)]) for k in range(K)]            # clip k, frame f -> 100k + f
    scene = S.scene_order(clips, use_last_frame)[:, 0].tolist()
    assert len(scene) == S.scene_length(K, T)
    pos = {(k, f): S.scene_frame_number(k, f, K, T, use_last_frame) for k in range(K) for f in range(T)}
    for k in range(K):
        for f in range(T):
            if k > 0 and f == S.cond_index(T, use_last_frame):
                # clip k's conditioning slot is clip k-1's hand-off frame, kept from clip k-1
                assert 100.0 * k + f not in scene
                assert pos[(k, f)] == pos[(k - 1, S.handoff_index(T, use_last_frame))]
                assert scene[pos[(k, f)]] == 100.0 * (k - 1) + S.handoff_index(T, use_last_frame)
            else:
                assert scene[pos[(k, f)]] == 100.0 * k + f
    if K > 1:
        # use_last_frame grows into the past: the latest-generated clip opens the scene
        assert scene[0] == (100.0 * (K - 1) if use_last_frame else 0.0)
    names = S.scene_order([[f"{k}:{f}" for f in range(T)] for k in range(K)], use_last_frame)
    assert names == [f"{int(v) // 100}:{int(v) % 100}" for v in scene]


def _scene_item(K, use_last_frame=True, T=4, hw=(16, 32), n=2, idx=0):
    from panacea_b200.inference import SyntheticBEVDataset
    ds = SyntheticBEVDataset(n, T, hw, use_last_frame, clips=K)
    return list(DataLoader(ds, batch_size=1))[idx]


@pytest.mark.parametrize("use_last_frame", [True, False])
def test_dataset_scene_contract(use_last_frame):
    from panacea_b200.inference import SyntheticBEVDataset
    K, T = 3, 4
    item = _scene_item(K, use_last_frame, T, idx=1)
    assert set(item) == {"clips"} and len(item["clips"]) == K
    first = item["clips"][0]
    plain = list(DataLoader(SyntheticBEVDataset(2, T, (16, 32), use_last_frame), batch_size=1))[1]
    assert set(first) == set(plain)
    for key in ("jpg", "cond_img", "final_cond_zero"):                     # clip 0 is the one-clip item, real frame included
        assert torch.equal(first[key], plain[key]), key
    a = S.cond_index(T, use_last_frame)
    assert first["final_cond_zero"][0, a].abs().max() > 0
    for c in item["clips"][1:]:
        assert set(c) == {"cond_img", "txt", "filenames"}
        assert c["cond_img"].shape == first["cond_img"].shape and not torch.equal(c["cond_img"], first["cond_img"])
    for k in range(1, K):                                                  # a boundary frame has one file name
        prev, cur = item["clips"][k - 1]["filenames"], item["clips"][k]["filenames"]
        assert cur[a] == prev[S.handoff_index(T, use_last_frame)]
    names = S.scene_order([c["filenames"] for c in item["clips"]], use_last_frame)
    for cam in range(6):
        stamps = [_stamp(f[cam]) for f in names]
        assert stamps == sorted(stamps) and len(set(stamps)) == S.scene_length(K, T)
    one = list(DataLoader(SyntheticBEVDataset(2, T, (16, 32), use_last_frame, clips=1), batch_size=1))[1]
    assert one["filenames"] == plain["filenames"]
    with pytest.raises(ValueError):
        SyntheticBEVDataset(1, T, (16, 32), clips=0)


def test_scene_writers_number_frames_continuously(tmp_path):
    from PIL import Image
    K, T, h, w = 3, 4, 16, 32
    item = _scene_item(K, True, T, (h, w))
    names = S.scene_order([c["filenames"] for c in item["clips"]], True)
    N = S.scene_length(K, T)
    frames = torch.linspace(-1.0, 1.0, N).reshape(N, 1, 1, 1).expand(N, 3, h, 6 * w).contiguous()
    written = IO.logs_scene(frames, str(tmp_path), names)
    jpgs = [p for p in written if p.endswith(".jpg")]
    assert len(jpgs) == 6 * N
    dirs = sorted(p.name for p in (tmp_path / "fake").iterdir())
    last = IO._stem(IO._name(names[-1][IO.VIEW_ID["CAM_FRONT"]]))
    assert len(dirs) == 6 and last.split("__")[-2] + "_" + last in dirs
    for d in dirs:
        assert sorted(p.name for p in (tmp_path / "fake" / d).iterdir()) == [f"_{i:06}.jpg" for i in range(N)]
    gifs = [p for p in written if p.endswith(".gif")]
    pngs = [p for p in written if p.endswith(".png")]
    assert len(gifs) == 1 and len(pngs) == 1
    assert Image.open(gifs[0]).n_frames == N and Image.open(pngs[0]).size == (6 * w, N * h)
    d = tmp_path / "fake" / dirs[0]
    px = [Image.open(d / f"_{i:06}.jpg").convert("L").getpixel((3, 3)) for i in range(N)]
    assert px == sorted(px) and px[0] < 10 and px[-1] > 245                # chronological order survives the writer


def test_clips_option_parsing():
    from panacea_b200.inference import get_parser
    p = get_parser()
    assert p.parse_known_args(["--name", "x"])[0].clips == 1
    assert p.parse_known_args(["--name", "x", "--clips", "3"])[0].clips == 3
    for bad in ("0", "-2", "two"):
        with pytest.raises(SystemExit):
            p.parse_known_args(["--name", "x", "--clips", bad])


def test_make_dataset_routes_scene_and_one_clip_forms(monkeypatch):
    import sys
    import types
    from panacea_b200.inference import SyntheticBEVDataset, get_parser, load_config, make_dataset
    cfg = load_config([CFG])
    opt = get_parser().parse_known_args(["--name", "x", "--image_hw", "16", "32"])[0]
    ds = make_dataset(opt, cfg)
    assert isinstance(ds, SyntheticBEVDataset) and ds.clips == 1 and "jpg" in ds[0]
    opt = get_parser().parse_known_args(["--name", "x", "--image_hw", "16", "32", "--clips", "2"])[0]
    assert len(make_dataset(opt, cfg)[0]["clips"]) == 2
    seen = []

    class Plugged:                                       # a --dataset class: `clips=` is passed only for scenes
        def __init__(self, **kw):
            seen.append(kw)
    monkeypatch.setitem(sys.modules, "plugged_ds", types.SimpleNamespace(Plugged=Plugged))
    for argv, want in ((["--clips", "1"], {}), (["--clips", "4"], {"clips": 4})):
        opt = get_parser().parse_known_args(["--name", "x", "--dataset", "plugged_ds:Plugged", *argv])[0]
        make_dataset(opt, cfg)
        assert seen[-1] == {"split": "val", "use_last_frame": True, **want}


def _engine():
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.util import instantiate_from_config
    return instantiate_from_config(load_config([CFG])["model"])


def _stub_log_images(m, calls, T=4, hw=(16, 192)):
    def log_images(batch, **kw):
        calls.append(batch)
        k = len(calls)
        g = torch.Generator().manual_seed(k)
        return {"samples": torch.rand(T, 3, *hw, generator=g) * 2.4 - 1.2, "sample_latents": torch.full((T, 4, 2, 24), float(k)),
                "inputs": torch.zeros(1)}
    m.log_images = log_images


def test_one_clip_scene_is_one_log_images_call():
    m = _engine()
    calls = []
    _stub_log_images(m, calls)
    item = _scene_item(1)
    out = m.sample_scene([item])
    assert len(calls) == 1
    assert set(calls[0]) == set(item) and all(calls[0][k] is item[k] or torch.equal(calls[0][k], item[k]) for k in item)
    assert out["handoff_frames"] == [] and torch.equal(out["samples"], out["clip_samples"][0])
    assert out["filenames"] == item["filenames"]


@pytest.mark.parametrize("use_last_frame", [True, False])
def test_scene_hands_each_clip_the_quantised_opposite_end_of_the_previous(use_last_frame):
    m = _engine()
    calls = []
    _stub_log_images(m, calls)
    K, T = 3, 4
    item = _scene_item(K, use_last_frame, T)
    out = m.sample_scene(item["clips"], use_last_frame=use_last_frame)
    assert len(calls) == K and "jpg" in calls[0] and torch.equal(calls[0]["final_cond_zero"], item["clips"][0]["final_cond_zero"])
    h = S.handoff_index(T, use_last_frame)
    for k in range(1, K):
        assert "jpg" not in calls[k] and torch.equal(calls[k]["cond_img"], item["clips"][k]["cond_img"])
        frame = S.quantize_frame(out["clip_samples"][k - 1][h])
        assert torch.equal(out["handoff_frames"][k - 1], frame)
        want = S.condition_from_frame(frame, T, use_last_frame).unsqueeze(0)
        assert torch.equal(calls[k]["final_cond_zero"], want)
    assert len(out["handoff_frames"]) == K - 1 and [float(z[0, 0, 0, 0]) for z in out["sample_latents"]] == [1.0, 2.0, 3.0]
    assert torch.equal(out["samples"], S.scene_order(out["clip_samples"], use_last_frame))
    assert len(out["filenames"]) == S.scene_length(K, T)
