"""TEST INFRASTRUCTURE — golden loops of the reference's other samplers (sampling.py:85-365), run UNMODIFIED around
the reference wrapper on the seeded cases of oracle/cases.py. Writes

  tests/golden/samplers_tiny_2to1.pt     10-step loops on tiny_2to1 (CPU tests): x_final, the timestep index of every
                                         network evaluation and the host scalars the reference computed
                                         (get_ancestral_step, the DPM++ multipliers, the LMS coefficients);
  tests/golden/samplers_small_hd64.pt    the CFG loops (the six other samplers and, as a control, EulerEDMSampler
                                         at the same 10 steps) on oracle.cases.SAMPLER_CASE with the use_last_frame
                                         shared-noise init (GPU tests): x_final, and x at the first evaluation of
                                         every step on a fixed 1-in-TRAJ_STRIDE subset of its elements (the
                                         error-vs-step curve; the whole trajectory would make the file 4x larger).

Noise is injected in draw order from a seeded CPU generator: through `sampler.noise_sampler` for the ancestral
samplers, and by standing in for `torch.randn_like` during the call for the EDM churn (the reference draws its churn
noise with it, sampling.py:99). The mirror samplers accept the same stream through their `noise_sampler` attribute.

Run where the reference tree is available:  python -m tools.make_sampler_golden [--only tiny,small]
"""
from __future__ import annotations

import argparse
import sys
import time
from pathlib import Path

import torch

from oracle import cases as Cs
from oracle import ref_loader as R
from oracle.make_golden import sampler_inputs

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
DISC = {"target": "sgm.modules.diffusionmodules.discretizer.LegacyDDPMDiscretization"}
NOISE_SEED = 20261015
NUM_STEPS = 10
SCALE = 5.0
TRAJ_STRIDE = 8         # trajectory: every 8th element of the flattened latent

# (name, reference class, constructor kwargs, guider)
LOOPS = [
    ("euler", "EulerEDMSampler", {}, "cfg"),              # the reference config's sampler: a control for the others
    ("heun", "HeunEDMSampler", {}, "cfg"),
    ("euler_churn", "EulerEDMSampler", {"s_churn": 1.0}, "cfg"),
    ("euler_ancestral", "EulerAncestralSampler", {}, "cfg"),
    ("dpmpp_2s_ancestral", "DPMPP2SAncestralSampler", {}, "cfg"),
    ("dpmpp_2m", "DPMPP2MSampler", {}, "cfg"),
    ("lms", "LinearMultistepSampler", {"order": 4}, "cfg"),
    ("dpmpp_2m_identity", "DPMPP2MSampler", {}, "identity"),
]


def guider_config(kind: str, scale: float = SCALE) -> dict:
    if kind == "identity":
        return {"target": "sgm.modules.diffusionmodules.guiders.IdentityGuider"}
    return {"target": "sgm.modules.diffusionmodules.guiders.VanillaCFG", "params": {"scale": scale}}


def noise_stream(seed: int = NOISE_SEED):
    """The injected noise: one standard-normal CPU draw per call, shaped like the sampler state."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return lambda x: torch.randn(x.shape, generator=g, dtype=torch.float32).to(x.device)


def _first(v):
    return float(v.reshape(-1)[0]) if torch.is_tensor(v) else float(v)


@torch.no_grad()
def golden_loop(case: Cs.EpsCase, cls_name: str, kwargs: dict, guider: str, num_steps: int = NUM_STEPS,
                use_last_frame: bool = False, share_noise_level: float = 0.07, trajectory: bool = False,
                model=None) -> dict:
    ref = R.import_reference()
    if model is None:
        model = R.build_reference_model(case.unet_kwargs())
        model.load_state_dict(Cs.make_weights(case), strict=True)
    den = ref.denoiser.DiscreteDenoiser(
        weighting_config={"target": "sgm.modules.diffusionmodules.denoiser_weighting.EpsWeighting"},
        scaling_config={"target": "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling"},
        num_idx=1000, discretization_config=DISC)
    sampler = getattr(ref.sampling, cls_name)(num_steps=num_steps, device="cpu", discretization_config=DISC,
                                              guider_config=guider_config(guider), **kwargs)
    x, c, uc = sampler_inputs(case, use_last_frame)
    if use_last_frame and share_noise_level > 0.0:
        x = x + c["concat"][-1].unsqueeze(0).expand_as(x) * share_noise_level     # diffusion.py:244-249
    n = x.shape[0]
    calls, traj, scalars = [], [], {"ancestral": [], "mult": [], "lms": []}
    state = {"step_start": True}
    draw = noise_stream()

    def denoise(xx, sigma, cc):
        calls.append(int(den.sigma_to_idx(sigma)[0]))
        if trajectory and (state["step_start"] or not hasattr(sampler, "sampler_step")):
            traj.append(xx[:n].clone())             # x at the first evaluation of the step (after any churn noise)
        state["step_start"] = False
        return den(model, xx, sigma, cc)

    if hasattr(sampler, "sampler_step"):
        inner_step = sampler.sampler_step

        def sampler_step(*a, **k):
            state["step_start"] = True
            return inner_step(*a, **k)
        sampler.sampler_step = sampler_step
    if hasattr(sampler, "get_mult"):
        inner_mult = sampler.get_mult

        def get_mult(*a, **k):
            m = inner_mult(*a, **k)
            scalars["mult"].append([_first(v) for v in m])
            return m
        sampler.get_mult = get_mult
    if hasattr(sampler, "noise_sampler"):
        sampler.noise_sampler = draw

    S = ref.sampling
    saved = (S.get_ancestral_step, S.linear_multistep_coeff, torch.randn_like)

    def get_ancestral_step(*a, **k):
        sd, su = saved[0](*a, **k)
        scalars["ancestral"].append((_first(sd), _first(su)))
        return sd, su

    def linear_multistep_coeff(order, t, i, j, *a, **k):
        v = saved[1](order, t, i, j, *a, **k)
        scalars["lms"].append((order, i, j, float(v)))
        return v

    S.get_ancestral_step, S.linear_multistep_coeff = get_ancestral_step, linear_multistep_coeff
    torch.randn_like = lambda t, **k: draw(t)                       # EDM churn (sampling.py:99)
    try:
        with R.view_height_shim(case.H, case.w):
            out = sampler(denoise, x.clone(), c, uc)
    finally:
        S.get_ancestral_step, S.linear_multistep_coeff, torch.randn_like = saved
    res = {"meta": case.meta(), "sampler": cls_name, "kwargs": dict(kwargs), "guider": guider, "num_steps": num_steps,
           "scale": SCALE, "noise_seed": NOISE_SEED, "x_final": out.contiguous(), "timestep_indices": calls,
           "use_last_frame": use_last_frame, "share_noise_level": share_noise_level, "scalars": scalars}
    if trajectory:
        res["x_steps"] = torch.stack(traj).reshape(len(traj), -1)[:, ::TRAJ_STRIDE].contiguous()
        res["x_steps_stride"] = TRAJ_STRIDE
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="", help="comma-separated subset of: tiny, small")
    a = ap.parse_args(argv)
    only = set(filter(None, a.only.split(",")))
    if not only or "tiny" in only:
        case = Cs.GOLDEN_CASES[0]
        model = R.build_reference_model(case.unet_kwargs())
        model.load_state_dict(Cs.make_weights(case), strict=True)
        out = {}
        for name, cls, kw, gd in LOOPS:
            t0 = time.time()
            out[name] = golden_loop(case, cls, kw, gd, model=model)
            print(f"tiny {name}: {len(out[name]['timestep_indices'])} evaluations {time.time() - t0:.1f}s", flush=True)
        torch.save(out, GOLDEN / f"samplers_{case.name}.pt")
    if not only or "small" in only:
        case = Cs.SAMPLER_CASE
        model = R.build_reference_model(case.unet_kwargs())
        model.load_state_dict(Cs.make_weights(case), strict=True)
        out = {}
        for name, cls, kw, gd in LOOPS:
            if gd != "cfg":
                continue
            t0 = time.time()
            out[name] = golden_loop(case, cls, kw, gd, use_last_frame=True, trajectory=True, model=model)
            print(f"small {name}: {len(out[name]['timestep_indices'])} evaluations {time.time() - t0:.1f}s", flush=True)
        torch.save(out, GOLDEN / f"samplers_{case.name}.pt")


if __name__ == "__main__":
    main(sys.argv[1:])
