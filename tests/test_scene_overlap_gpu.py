"""Scenes whose clips share m frames on the GPU (DiffusionEngine3D.sample_scene(overlap=m), DESIGN.md section 11), on
the tiny inference config and weights of test_scene_gpu (T = 4):

  * composition: a K = 3, m = 2 scene is bitwise clip 0's log_images followed by, per carrying clip, _log_inputs ->
    _initial_noise -> sampler(known, mask) -> decode with the hand-off and the known region built by hand, in bf16 and
    parity mode, for both use_last_frame values; the shared latents and their decoded frames equal clip k-1's bitwise;
  * the fused and the plain-callable sampler loops agree on a carrying clip, shared frames bitwise in both;
  * one graph: the scene replays one CUDA graph and never repacks the weights;
  * the inference entry point (synthetic and --layout) and the layout dataset's shared frames;
  * full size, bf16, K = 2, m = 4, T = 8: seconds per clip and per new frame, peak memory against one clip."""
import json
import os

import numpy as np
import pytest
import torch

from test_scene_cpu import CFG
from test_scene_gpu import T, _clips, _dev, _small
from test_scene_overlap_cpu import _scene_file

pytestmark = pytest.mark.gpu
K, M = 3, 2


def _clips_overlap(use_last_frame):
    from torch.utils.data import DataLoader
    from panacea_b200.inference import SyntheticBEVDataset
    ds = SyntheticBEVDataset(1, T, (64, 128), use_last_frame, clips=K, overlap=M)
    return next(iter(DataLoader(ds, batch_size=1)))["clips"]


def _handoff(decoded_frame):
    u8 = (((decoded_frame.clamp(-1.0, 1.0) + 1.0) / 2.0).permute(1, 2, 0).numpy() * 255).astype(np.uint8)
    return torch.from_numpy(u8.astype(np.float32) / 127.5 - 1.0).permute(2, 0, 1)


def _kept(use_last_frame):
    """(frames of clip k, frames of clip k-1) that are the same scene frames, restated by hand."""
    return (slice(T - M, T), slice(0, M)) if use_last_frame else (slice(0, M), slice(T - M, T))


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("precision", ["bf16", "parity"])
def test_overlap_scene_is_log_images_then_outpainting_by_hand(precision, use_last_frame):
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    m, _ = _small(precision)
    clips = _clips_overlap(use_last_frame)
    torch.manual_seed(11)
    out = m.sample_scene(clips, use_last_frame=use_last_frame, overlap=M)
    a = T - 1 if use_last_frame else 0
    h = M - 1 if use_last_frame else T - M
    cur, prev = _kept(use_last_frame)
    torch.manual_seed(11)
    decoded, latents = [], []
    for k, clip in enumerate(clips):
        b = _dev(clip)
        if k == 0:
            log = m.log_images(b)
            lat, dec = log["sample_latents"], log["samples"]
        else:
            frame = _handoff(decoded[-1][h])
            assert torch.equal(out["handoff_frames"][k - 1], frame)
            cond = torch.zeros(1, T, *frame.shape)
            cond[0, a] = frame
            b["final_cond_zero"] = cond.cuda()
            known = torch.zeros(latents[-1].shape)
            mask = torch.ones(T, *latents[-1].shape[2:])
            known[cur] = latents[-1][prev]
            mask[cur] = 0.0
            _, c, uc, N, shape, z = m._log_inputs(b, 8)
            assert z is None
            x = m._initial_noise(c, N * T, shape)
            lat = m.sampler(BoundDenoiser(m.denoiser, m.model), x, c, uc=uc, known=known.cuda(), mask=mask.cuda())
            dec = m.decode_first_stage(lat)
        decoded.append(dec.cpu())
        latents.append(lat.cpu())
    for k in range(K):
        assert torch.equal(out["sample_latents"][k], latents[k]), k
        assert torch.equal(out["clip_samples"][k], decoded[k]), k
    n = K * (T - M) + M
    want = torch.cat([decoded[2][:T - M], decoded[1][:T - M], decoded[0]]) if use_last_frame else \
        torch.cat([decoded[0], decoded[1][M:], decoded[2][M:]])
    assert out["samples"].shape == (n, 3, 64, 768) and torch.equal(out["samples"], want) and out["overlap"] == M
    assert torch.isfinite(out["samples"]).all()
    for k in range(1, K):                                               # the shared frames, bitwise
        assert torch.equal(latents[k][cur], latents[k - 1][prev]), k
        assert torch.equal(decoded[k][cur], decoded[k - 1][prev]), k
    torch.manual_seed(11)
    plain = m.sample_scene(_clips(K, use_last_frame), use_last_frame=use_last_frame)
    fresh = slice(0, T - M) if use_last_frame else slice(M, T)
    for k in range(1, K):
        assert not torch.equal(plain["sample_latents"][k][fresh], latents[k][fresh]), k
    print(f"OVERLAP {precision} use_last_frame={use_last_frame}: {n} frames, shared latents and frames bitwise")


def test_fused_and_plain_callable_loops_agree_on_a_carrying_clip():
    """In parity mode, so that a blend applied differently by the two loops cannot hide under bf16 network error."""
    from panacea_b200 import scene as S
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    from panacea_b200.sgm.util import instantiate_from_config
    m, _ = _small("parity")
    w, den = m.model, instantiate_from_config(DEFAULT_DENOISER)
    clips = _clips_overlap(True)
    torch.manual_seed(2)
    first = m.log_images(_dev(clips[0]))
    known, mask = S.known_region(first["sample_latents"], True, M)
    b = _dev(clips[1])
    b["final_cond_zero"] = S.condition_from_frame(S.quantize_frame(first["samples"][M - 1]), T, True).unsqueeze(0).cuda()
    _, c, uc, N, shape, _ = m._log_inputs(b, 8)
    x = torch.randn((N * T, *shape), generator=torch.Generator().manual_seed(5)).cuda()
    outs = []
    for d in (BoundDenoiser(den, w), lambda xx, sigma, cc: den(w, xx, sigma, cc)):
        torch.manual_seed(6)
        outs.append(m.sampler(d, x, c, uc, num_steps=10, known=known, mask=mask).cpu())
    fused, plain = outs
    rel = ((fused - plain).norm() / fused.norm()).item()
    print(f"OVERLAP fused vs plain-callable rel-L2 {rel:.3e}")
    assert rel < 5e-3, rel
    carried = first["sample_latents"][:M].cpu()
    assert torch.equal(fused[T - M:], carried) and torch.equal(plain[T - M:], carried)


def test_overlap_scene_replays_one_graph_and_keeps_the_packed_weights():
    m, _ = _small("bf16")
    w = m.model
    eng = w.diffusion_model.engine()                                 # packed once, before the scene
    gen = eng.generation
    captures, packs, after = [], [], []
    cap, pack = w._capture, eng.pack
    w._capture = lambda *a, **k: (captures.append(1), cap(*a, **k))[1]
    eng.pack = lambda *a, **k: (packs.append(1), pack(*a, **k))[1]
    for name in ("log_images", "outpaint_images"):
        inner = getattr(m, name)

        def logged(batch, *a, _inner=inner, **kw):
            log = _inner(batch, *a, **kw)
            after.append((w._graph, eng.cond["guided"].data_ptr(), sorted(v.data_ptr() for v in eng.cond["kv"].values())))
            return log
        setattr(m, name, logged)
    torch.manual_seed(0)
    out = m.sample_scene(_clips_overlap(True), overlap=M)
    assert len(after) == K and len(captures) == 1, f"{len(captures)} graph captures over a {K}-clip scene"
    assert all(x[0] is after[0][0] for x in after), "a clip replaced the captured graph"
    assert len({x[1] for x in after}) == 1 and all(x[2] == after[0][2] for x in after), "conditioning buffers moved"
    assert packs == [] and eng.generation == gen, "the packed weights were rebuilt during the scene"
    assert torch.isfinite(out["samples"]).all()


def test_inference_entry_point_writes_an_overlapping_scene(tmp_path):
    from panacea_b200 import inference as INF
    written = INF.main(["--name", "scene", "--base", CFG, "--inferdir", str(tmp_path), "--num_sequences", "1",
                        "--image_hw", "64", "128", "--clips", str(K), "--overlap", str(M), "--randomize_zero_init"])
    fake = tmp_path / "scene" / "fake"
    dirs = sorted(os.listdir(fake))
    assert len(dirs) == 6
    for d in dirs:
        assert sorted(os.listdir(fake / d)) == [f"_{i:06}.jpg" for i in range(K * (T - M) + M)]
    assert len([p for p in written if p.endswith(".gif")]) == 1 and len([p for p in written if p.endswith(".png")]) == 1


def test_layout_scene_with_overlap_renders_shared_frames_once(tmp_path):
    from panacea_b200 import inference as INF
    from panacea_b200.frame_io import CAMERA_VIEWS
    n = K * (T - M) + M
    path = _scene_file(tmp_path, n)
    written = INF.main(["--name", "layout", "--base", CFG, "--inferdir", str(tmp_path / "out"), "--layout", str(path),
                        "--image_hw", "64", "128", "--clips", str(K), "--overlap", str(M), "--randomize_zero_init"])
    fake = tmp_path / "out" / "layout" / "fake"
    dirs = sorted(os.listdir(fake))
    assert dirs == sorted(f"{cam}_drive{n}__{cam}__{n - 1:06d}" for cam in CAMERA_VIEWS)
    for d in dirs:
        assert sorted(os.listdir(fake / d)) == [f"_{i:06}.jpg" for i in range(n)]
    assert len([p for p in written if p.endswith(".gif")]) == 1 and len([p for p in written if p.endswith(".png")]) == 1
    for use_last_frame in (True, False):
        clips = INF.LayoutDataset(path, T, (64, 128), use_last_frame, K, overlap=M)[0]["clips"]
        cur, prev = _kept(use_last_frame)
        for k in range(1, K):
            assert torch.equal(clips[k]["cond_img"][cur], clips[k - 1]["cond_img"][prev]), (use_last_frame, k)
            assert not torch.equal(clips[k]["cond_img"], clips[k - 1]["cond_img"])


def test_full_size_overlap_scene_peak_memory_is_one_clip_plus_one_decoded_clip():
    from tools.bench_scene import full_size_engine, scene_clips, timed_scene
    from tools.bench_vae import card
    ov = 4
    m = full_size_engine(steps=10)
    clips = scene_clips(2)
    torch.manual_seed(0)
    timed_scene(m, clips[:1])                                         # packing and graph capture
    _, one, _, one_peak = timed_scene(m, clips[:1])
    out, per_clip, total, peak = timed_scene(m, clips, overlap=ov)
    frames = int(out["samples"].shape[0])
    decoded = out["clip_samples"][0].numel() * out["clip_samples"][0].element_size()
    rec = {"case": "scene_full_size_bf16_k2_overlap4", "card": card(), "steps": 10, "one_clip_s": one[0], "clip_s": per_clip,
           "scene_s": total, "scene_frames": frames, "s_per_scene_frame": total / frames,
           "s_per_new_frame_second_clip": per_clip[1] / (8 - ov), "one_clip_peak_gb": one_peak / 1e9,
           "scene_peak_gb": peak / 1e9, "decoded_clip_gb": decoded / 1e9}
    print("SCENE_OVERLAP " + json.dumps(rec))
    assert out["samples"].shape == (2 * (8 - ov) + ov, 3, 256, 3072) and torch.isfinite(out["samples"]).all()
    assert peak <= one_peak + decoded, rec
