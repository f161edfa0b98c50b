"""Time the native VAE at the headline size in both precision modes and report its peak memory.

  python tools/bench_vae.py [--reps 5] [--frames 8] [--no-unet] [--out FILE]

Decode of z [F, 4, 32, 384] and encode of x [F, 3, 256, 3072] (F = 8 frames, 6 views of 32 x 64 latents / 256 x 512
pixels), each in bf16 and in parity mode (with the wrapper's default frames per call), on the inference config's
ddconfig with seeded random weights. Each case gets
one warm-up call, then `--reps` calls timed with CUDA events (one event pair per call); it reports the median and range.
Peak memory is `torch.cuda.max_memory_allocated` over the warm-up and timed calls.

Unless `--no-unet`, the full-size ControlNet + UNet is built in parity mode first and runs CFG-doubled eps-evaluations
at the benchmark shape (x [16, 8, 32, 336]) through its captured CUDA graph, as the sampler does; its weights and the
graph's memory pool stay resident while the VAE runs, so the VAE peaks show what a parity run needs next to a parity
UNet on one card.

The card name and power limit are read in the same run. Prints one JSON line (and writes it to --out).
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

DDCONFIG = dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                attn_resolutions=[], dropout=0.0)           # configs/inference_nuscenes.yaml first_stage_config


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "total_memory_gb": torch.cuda.get_device_properties(0).total_memory / 1e9}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["sm_max_mhz"] = float(q[0]), float(q[1])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        info["power_limit_w"] = None
    return info


def unet_parity_eval():
    """Full-size parity ControlNet + UNet, CFG-doubled eps-evaluations at the benchmark shape (graph capture + replay)."""
    from panacea_b200.pipeline import DenoisingPipeline
    g = torch.Generator().manual_seed(0)
    with torch.device("cuda"):
        pipe = DenoisingPipeline(use_cuda_graph=True, precision="parity")
    pipe.wrapper.hint_repeat = 2
    T, H, W = 8, 32, 336
    cc = {"cond_feat": torch.rand(T, 19, 8 * H, 8 * W, generator=g).cuda(), "concat": torch.randn(2 * T, 4, H, W, generator=g).cuda(),
          "crossattn": torch.randn(2, 77, 1024, generator=g).cuda()}
    x = torch.randn(2 * T, 4, H, W, generator=g).cuda()
    t = torch.full((2 * T,), 500, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(3):
        eps = pipe.wrapper(x, t, cc)
    torch.cuda.synchronize()
    res = {"peak_gb": torch.cuda.max_memory_allocated() / 1e9, "finite": bool(torch.isfinite(eps).all())}
    del eps, cc, x
    res["resident_gb"] = torch.cuda.memory_allocated() / 1e9
    res["reserved_gb"] = torch.cuda.memory_reserved() / 1e9
    return pipe, res


def time_case(fn, inp, reps: int) -> dict:
    torch.cuda.synchronize()
    torch.cuda.empty_cache()                             # the previous case's cached blocks do not count for this one
    torch.cuda.reset_peak_memory_stats()
    try:
        out = fn(inp)                                    # warm-up: packing, module load, allocator
    except torch.OutOfMemoryError as e:                  # a result too: this case does not fit next to what is resident
        torch.cuda.empty_cache()
        return {"out_of_memory": str(e).split(". ")[0], "peak_gb": torch.cuda.max_memory_allocated() / 1e9}
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(inp)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return {"ms_median": statistics.median(ms), "ms_min": min(ms), "ms_max": max(ms), "reps": reps,
            "peak_gb": torch.cuda.max_memory_allocated() / 1e9, "peak_reserved_gb": torch.cuda.max_memory_reserved() / 1e9,
            "finite": bool(torch.isfinite(out).all())}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--no-unet", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_vae.py: no CUDA device (the VAE has no CPU path)")
    from oracle.make_golden import vae_decoder_weights
    from panacea_b200.sgm.models.autoencoder import AutoencoderKLInferenceWrapper
    res = {"card": card(), "frames": a.frames, "z": [a.frames, 4, 32, 384], "x": [a.frames, 3, 256, 3072], "cases": {},
           "frames_per_call": {"bf16": "all", "parity": AutoencoderKLInferenceWrapper.PARITY_FRAMES_PER_CALL}}
    keep = None
    if not a.no_unet:
        keep, res["unet_parity_eps"] = unet_parity_eval()
        print(f"unet parity eps: {res['unet_parity_eps']}", file=sys.stderr, flush=True)
    g = torch.Generator().manual_seed(1)
    z = torch.randn(a.frames, 4, 32, 384, generator=g).cuda()
    x = (torch.rand(a.frames, 3, 256, 3072, generator=g) * 2.0 - 1.0).cuda()
    m = AutoencoderKLInferenceWrapper(embed_dim=4, ddconfig=DDCONFIG, lossconfig={"target": "torch.nn.Identity"}, precision="bf16")
    sd = vae_decoder_weights({k: tuple(v.shape) for k, v in m.state_dict().items()}, seed=2)
    m.load_state_dict(sd, strict=False)
    m = m.cuda()
    for precision in ("bf16", "parity"):
        m.set_precision(precision)
        for name, fn, inp in (("decode", m.decode, z), ("encode", m.encode_moments, x)):
            r = time_case(fn, inp, a.reps)
            res["cases"][f"{name}_{precision}"] = r
            print(f"{name} {precision}: {r}", file=sys.stderr, flush=True)
    res["resident_unet_gb"] = res.get("unet_parity_eps", {}).get("resident_gb", 0.0)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")
    del keep


if __name__ == "__main__":
    main(sys.argv[1:])
