"""Scenes of K chained clips on the GPU (DiffusionEngine3D.sample_scene, DESIGN.md section 11), on the tiny inference
config (the small head_dim-64 model with the seeded weights of the sampler cases, the config's VAE at a 64 x 768 image):

  * composition: a K = 3 rollout is bitwise three log_images calls with the hand-off done by hand, in bf16 and parity
    mode, for both use_last_frame values;
  * one graph: the wrapper captures one CUDA graph for the whole scene and the packed weights are not rebuilt;
  * per clip, teacher-forced: each clip's latent against the CPU oracle port given the same conditioning (the hand-off
    frame the GPU produced) and the same initial noise, at the parity bar;
  * full size, bf16, K = 2: peak memory of the scene against one clip, seconds per clip logged;
  * the inference entry point with --clips 3."""
import json
import os
from pathlib import Path

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from test_eps_parity_gpu import _report

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
T = 4


def _small(precision):
    from oracle import cases as Cs
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.util import instantiate_from_config
    m = instantiate_from_config(load_config([CFG], [f"model.params.precision={precision}"])["model"])
    sd = Cs.make_weights(Cs.SAMPLER_CASE)
    m.model.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


def _clips(K, use_last_frame):
    from panacea_b200.inference import SyntheticBEVDataset
    return next(iter(DataLoader(SyntheticBEVDataset(1, T, (64, 128), use_last_frame, clips=K), batch_size=1)))["clips"]


def _dev(batch):
    return {k: v.cuda() if isinstance(v, torch.Tensor) else v for k, v in batch.items()}


@pytest.mark.parametrize("use_last_frame", [True, False])
@pytest.mark.parametrize("precision", ["bf16", "parity"])
def test_scene_is_log_images_calls_with_the_handoff_by_hand(precision, use_last_frame):
    m, _ = _small(precision)
    clips = _clips(3, use_last_frame)
    torch.manual_seed(11)
    out = m.sample_scene(clips, use_last_frame=use_last_frame)
    a = T - 1 if use_last_frame else 0
    torch.manual_seed(11)
    decoded, latents, prev = [], [], None
    for k, clip in enumerate(clips):
        b = _dev(clip)
        if k:
            u8 = (((prev.clamp(-1.0, 1.0) + 1.0) / 2.0).permute(1, 2, 0).numpy() * 255).astype(np.uint8)
            frame = torch.from_numpy(u8.astype(np.float32) / 127.5 - 1.0).permute(2, 0, 1)
            assert torch.equal(out["handoff_frames"][k - 1], frame)
            cond = torch.zeros(1, T, *frame.shape)
            cond[0, a] = frame
            b["final_cond_zero"] = cond.cuda()
        log = m.log_images(b)
        decoded.append(log["samples"].cpu())
        latents.append(log["sample_latents"].cpu())
        assert ("inputs" in log) == (k == 0) and ("reconstructions" in log) == (k == 0)
        prev = decoded[-1][T - 1 - a]
    for k in range(3):
        assert torch.equal(out["sample_latents"][k], latents[k]), k
        assert torch.equal(out["clip_samples"][k], decoded[k]), k
    want = torch.cat([decoded[2][:-1], decoded[1][:-1], decoded[0]]) if use_last_frame else \
        torch.cat([decoded[0], decoded[1][1:], decoded[2][1:]])
    assert out["samples"].shape == (3 * (T - 1) + 1, 3, 64, 768) and torch.equal(out["samples"], want)
    assert torch.isfinite(out["samples"]).all() and not torch.equal(latents[1], latents[2])


def test_scene_replays_one_graph_and_keeps_the_packed_weights():
    m, _ = _small("bf16")
    w = m.model
    eng = w.diffusion_model.engine()                                 # packed once, before the scene
    gen = eng.generation
    captures, packs, prepares, after = [], [], [], []
    cap, pack, prep, log_images = w._capture, eng.pack, eng.prepare_condition, m.log_images
    w._capture = lambda *a, **k: (captures.append(1), cap(*a, **k))[1]
    eng.pack = lambda *a, **k: (packs.append(1), pack(*a, **k))[1]
    eng.prepare_condition = lambda *a, **k: (prepares.append(1), prep(*a, **k))[1]

    def logged(batch, **kw):
        log = log_images(batch, **kw)
        after.append((w._graph, eng.cond["guided"].data_ptr(), sorted(v.data_ptr() for v in eng.cond["kv"].values())))
        return log
    m.log_images = logged
    torch.manual_seed(0)
    out = m.sample_scene(_clips(3, True))
    assert len(after) == 3 and len(captures) == 1, f"{len(captures)} graph captures over a 3-clip scene"
    assert all(x[0] is after[0][0] for x in after), "a clip replaced the captured graph"
    assert len({x[1] for x in after}) == 1 and all(x[2] == after[0][2] for x in after), "conditioning buffers moved"
    assert packs == [] and eng.generation == gen, "the packed weights were rebuilt during the scene"
    assert len(prepares) == 3                                         # each clip's hint stem and text K/V, re-prepared in place
    assert torch.isfinite(out["samples"]).all()


@pytest.mark.parametrize("use_last_frame", [True, False])
def test_scene_clips_match_the_oracle_teacher_forced(use_last_frame):
    """Each clip's latent against the CPU oracle port's Euler/CFG loop, given the conditioning and initial noise the GPU
    clip used (its concat encodes the hand-off frame the GPU produced), so a rounding flip in one clip's uint8 hand-off
    cannot carry into the next clip's comparison. Latents normalised by the oracle's rms, as the sampler-loop tests do."""
    from oracle import cases as Cs, sampler_port as SP, unet_port as P
    m, sd = _small("parity")
    seen = []

    class Recorder:
        def __init__(self, inner):
            self.inner = inner

        def __call__(self, den, x, cond, uc=None, **kw):
            seen.append((x.cpu(), {k: v.cpu() for k, v in cond.items()}, {k: v.cpu() for k, v in uc.items()}))
            return self.inner(den, x, cond, uc=uc, **kw)
    m.sampler = Recorder(m.sampler)
    torch.manual_seed(5)
    out = m.sample_scene(_clips(3, use_last_frame), use_last_frame=use_last_frame)
    assert len(seen) == 3
    cfg = Cs.SAMPLER_CASE.net_config()
    net = lambda xx, t, cc: P.wrapper_forward(sd, cfg, xx, t, cc)
    steps, scale = m.sampler.inner.num_steps, m.sampler.inner.guider.scale
    for k, (x, c, uc) in enumerate(seen):
        ref = SP.euler_edm_sample(net, x, c, uc, steps, scale=scale)
        got = out["sample_latents"][k]
        rms = ref.double().pow(2).mean().sqrt().item()
        _report(f"scene_clip{k}{'_last_frame' if use_last_frame else ''}:latent_vs_oracle", got / rms, ref / rms, "parity",
                {"latent_rms": rms})


def test_full_size_scene_peak_memory_is_one_clip_plus_one_decoded_clip():
    from tools.bench_scene import full_size_engine, scene_clips, timed_scene
    from tools.bench_vae import card
    m = full_size_engine(steps=10)
    clips = scene_clips(2)
    torch.manual_seed(0)
    timed_scene(m, clips[:1])                                         # packing and graph capture
    _, one, _, one_peak = timed_scene(m, clips[:1])
    out, per_clip, total, peak = timed_scene(m, clips)
    decoded = out["clip_samples"][0].numel() * out["clip_samples"][0].element_size()
    rec = {"case": "scene_full_size_bf16_k2", "card": card(), "steps": 10, "one_clip_s": one[0], "clip_s": per_clip,
           "scene_s": total, "one_clip_peak_gb": one_peak / 1e9, "scene_peak_gb": peak / 1e9, "decoded_clip_gb": decoded / 1e9}
    print("SCENE " + json.dumps(rec))
    assert out["samples"].shape == (15, 3, 256, 3072) and torch.isfinite(out["samples"]).all()
    assert peak <= one_peak + decoded, rec


def test_inference_entry_point_writes_a_three_clip_scene(tmp_path):
    from panacea_b200 import inference as INF
    written = INF.main(["--name", "scene", "--base", CFG, "--inferdir", str(tmp_path), "--num_sequences", "1",
                        "--image_hw", "64", "128", "--clips", "3", "--randomize_zero_init"])
    fake = tmp_path / "scene" / "fake"
    dirs = sorted(os.listdir(fake))
    assert len(dirs) == 6
    for d in dirs:
        assert sorted(os.listdir(fake / d)) == [f"_{i:06}.jpg" for i in range(10)]
    assert len([p for p in written if p.endswith(".gif")]) == 1 and len([p for p in written if p.endswith(".png")]) == 1
