"""Time a scene of K chained clips at full size and report its peak memory against one clip.

  python tools/bench_scene.py [--clips 2] [--steps 25] [--precision bf16] [--out FILE]
  python tools/bench_scene.py --overlap M [--reps 2] [--steps 25] [--out FILE]

The engine is tests/configs/tiny_inference.yaml grown to the reference's sizes (FULL_SIZE_OVERRIDES: model_channels 320,
context_dim 1024, 8 frames; the SD VAE of that YAML is already full size) with random weights and the zero-initialised
tails re-drawn, on `SyntheticBEVDataset` at 256 x 512 per view (latent 32 x 64 x 6 views), EulerEDMSampler + CFG 5.
One warm-up clip (weight packing, graph capture) runs first. Then, with host clocks around work that ends in a device
synchronise:
  * a one-clip scene (= log_images): seconds and peak `torch.cuda.max_memory_allocated`;
  * a K-clip scene: seconds per clip and per scene, peak memory;
  * the hand-off's pieces, each timed alone (median of 5, CUDA events): the decode of the boundary frame alone, the
    encode of a clip's image condition through the conditioner's VAE embedder, and the host round trip of the frame
    (copy out, quantise, dequantise, build the condition) — each as a share of the mean clip time. In a scene the
    boundary frame is decoded with its clip and every clip encodes an image condition, so only the host round trip is
    work a one-clip run does not do.
With --overlap M the run instead compares the two ways of chaining a 2-clip scene, after one warm-up scene of each:
  * alternately, --reps times, the scene with `overlap` None (boundary frame regenerated) and with `overlap` M (clip 1
    keeps clip 0's latents of M frames): seconds per clip, and seconds per new frame (scene seconds over the scene's
    frames, and the second clip's seconds over the T-1 or T-M frames it adds);
  * CUDA-event time (median of 7 runs of 50 launches) of one pn_sampler_step launch against one pn_sampler_step_known
    launch with M of 8 frames kept (Euler, CFG halves, next network input written) on the benchmark's latent [8, 4,
    32, 336] (344 K elements), and the difference as a share of one denoising step (clip seconds / steps, which
    includes the clip's decode and so overstates the step).
The card name, power limit and clocks are read in the same run. Prints one JSON line (and writes it to --out).
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
_NET = "model.params.network_config.params."
_CN = _NET + "controlnet_config.params."
FULL_SIZE_OVERRIDES = [_NET + "model_channels=320", _NET + "context_dim=1024", _NET + "num_frames=8",
                       _CN + "model_channels=320", _CN + "context_dim=1024", _CN + "num_frames=8",
                       "model.params.conditioner_config.params.emb_models.0.params.context_dim=1024"]


def full_size_engine(steps: int, precision: str = "bf16"):
    """The full-size DiffusionEngine3D on the GPU, random weights with the zero-initialised tails re-drawn."""
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.util import instantiate_from_config
    cfg = load_config([CFG], FULL_SIZE_OVERRIDES + [f"model.params.sampler_config.params.num_steps={steps}",
                                                    f"model.params.precision={precision}"])
    m = instantiate_from_config(cfg["model"])
    m.model.diffusion_model.randomize_zero_init(seed=0)
    m.model.diffusion_model.controlnet.randomize_zero_init(seed=1)
    return m.cuda().eval()


def scene_clips(clips: int, use_last_frame: bool = True, image_hw=(256, 512)):
    from torch.utils.data import DataLoader
    from panacea_b200.inference import SyntheticBEVDataset
    item = next(iter(DataLoader(SyntheticBEVDataset(1, 8, image_hw, use_last_frame, clips=clips), batch_size=1)))
    return item["clips"] if clips > 1 else [item]


def timed_scene(m, clips, use_last_frame=True, overlap=None):
    """-> (output, seconds per clip, scene seconds, peak bytes), each clip timed by a host clock ending in a synchronise."""
    per_clip = []

    def timed(inner):
        def run(*a, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            log = inner(*a, **kw)
            torch.cuda.synchronize()
            per_clip.append(time.perf_counter() - t0)
            return log
        return run
    m.log_images, m.outpaint_images = timed(m.log_images), timed(m.outpaint_images)
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = m.sample_scene(clips, use_last_frame=use_last_frame, overlap=overlap)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        del m.log_images, m.outpaint_images
    return out, per_clip, total, torch.cuda.max_memory_allocated()


def _median_ms(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return statistics.median(ms)


def handoff_costs(m, out, use_last_frame=True):
    """ms of the hand-off's pieces, each alone: boundary-frame decode, condition encode, host round trip."""
    from panacea_b200 import scene as S
    from panacea_b200.sgm.modules.encoders.modules import VAEEmbedder
    T = m.num_frames
    h = S.handoff_index(T, use_last_frame)
    z = out["sample_latents"][0][h:h + 1].cuda()
    emb = [e for e in m.conditioner.embedders if isinstance(e, VAEEmbedder)][0]
    frame = out["clip_samples"][0][h].cuda()
    cond = S.condition_from_frame(S.quantize_frame(frame), T, use_last_frame).cuda()

    def host_round_trip():
        S.condition_from_frame(S.quantize_frame(frame), T, use_last_frame).cuda()
    return {"decode_boundary_frame_ms": _median_ms(lambda: m.decode_first_stage(z)),
            "condition_encode_ms": _median_ms(lambda: emb(cond)),
            "host_round_trip_ms": _median_ms(host_round_trip)}


def step_launches(overlap, T=8, reps=50, runs=7):
    """ms per pn_sampler_step launch, plain and with the known region of a carrying clip, on the benchmark's latent."""
    from panacea_b200 import scene as S
    from panacea_b200.ops import SAMPLER_EULER, NativeOps
    ops = NativeOps()
    shape = (T, 4, 32, 6 * 56)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(shape, device="cuda", generator=g)
    net = torch.randn((2 * T,) + shape[1:], device="cuda", generator=g)
    x_in = torch.empty_like(net)
    known, mask = S.known_region(torch.randn(shape, device="cuda", generator=g), True, overlap)
    kw = dict(x_in_next=x_in, halves=2, sigma_q=3.0, cfg_scale=5.0, sigma=3.0, dt=-0.5, c_in_next=0.3)
    blend = dict(known=known, mask=mask, known_seed=7, known_draw=1, known_sigma=2.5)

    def per_launch(fn):
        for _ in range(3):
            fn()
        ms = []
        for _ in range(runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / reps)
        return statistics.median(ms)
    plain, known_ms = [], []
    for _ in range(2):                                              # alternated
        plain.append(per_launch(lambda: ops.sampler_step(SAMPLER_EULER, x, net, **kw)))
        known_ms.append(per_launch(lambda: ops.sampler_step(SAMPLER_EULER, x, net, **kw, **blend)))
    return {"elements": x.numel(), "kept_frames": overlap, "plain_ms": plain, "known_ms": known_ms}


def compare_overlap(a):
    """The --overlap run: a 2-clip scene with and without the carried latents, alternated, and the step launches."""
    T = 8
    m = full_size_engine(a.steps, a.precision)
    clips = scene_clips(2)
    torch.manual_seed(0)
    modes = {"boundary": None, "overlap": a.overlap}
    for ov in modes.values():                                       # warm-up: packing, graph capture, module loads
        timed_scene(m, clips, overlap=ov)
    runs = {k: [] for k in modes}
    for _ in range(a.reps):
        for k, ov in modes.items():
            out, per_clip, total, peak = timed_scene(m, clips, overlap=ov)
            frames = int(out["samples"].shape[0])
            new = T - (1 if ov is None else ov)
            runs[k].append({"clip_s": per_clip, "scene_s": total, "scene_frames": frames, "s_per_scene_frame": total / frames,
                            "second_clip_new_frames": new, "s_per_new_frame_second_clip": per_clip[1] / new,
                            "peak_gb": peak / 1e9})
    step = step_launches(a.overlap, T)
    step_s = statistics.mean(r["clip_s"][1] for r in runs["overlap"]) / a.steps
    extra = statistics.median(step["known_ms"]) - statistics.median(step["plain_ms"])
    step.update({"known_extra_ms": extra, "clip_s_per_step": step_s, "known_extra_share_of_step": extra / 1e3 / step_s})
    return {"overlap": a.overlap, "reps": a.reps, "runs": runs, "step_launch": step}


def main(argv=None):
    from tools.bench_vae import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2)
    ap.add_argument("--steps", type=int, default=25, help="sampler steps per clip (the reference's config: 25)")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "parity"])
    ap.add_argument("--overlap", type=int, default=None, help="compare 2-clip scenes with and without M shared frames")
    ap.add_argument("--reps", type=int, default=2, help="alternations of the --overlap comparison")
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_scene.py: no CUDA device (the engine has no CPU path)")
    res = {"card": card(), "clips": a.clips, "steps": a.steps, "precision": a.precision, "frames_per_clip": 8,
           "image": [3, 256, 3072]}
    if a.overlap is not None:
        res.update(compare_overlap(a), clips=2)
        _emit(res, a.out)
        return
    m = full_size_engine(a.steps, a.precision)
    clips = scene_clips(a.clips)
    torch.manual_seed(0)
    timed_scene(m, clips[:1])                                        # warm-up: packing, graph capture, module loads
    _, one, one_total, one_peak = timed_scene(m, clips[:1])
    out, per_clip, total, peak = timed_scene(m, clips)
    clip_s = statistics.mean(per_clip)
    costs = handoff_costs(m, out)
    res.update({"one_clip_s": one[0], "one_clip_peak_gb": one_peak / 1e9, "scene_s": total, "scene_frames": int(out["samples"].shape[0]),
                "clip_s": per_clip, "scene_peak_gb": peak / 1e9,
                "decoded_clip_gb": out["clip_samples"][0].numel() * 4 / 1e9, **costs,
                "handoff_share_of_clip": {k.replace("_ms", ""): v / 1e3 / clip_s for k, v in costs.items()}})
    _emit(res, a.out)


def _emit(res, out):
    line = json.dumps(res)
    print(line, flush=True)
    if out:
        Path(out).parent.mkdir(parents=True, exist_ok=True)
        Path(out).write_text(line + "\n")


if __name__ == "__main__":
    main(sys.argv[1:])
