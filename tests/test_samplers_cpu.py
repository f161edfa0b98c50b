"""The mirror samplers (panacea_b200/sgm/modules/diffusionmodules/sampling.py) on the CPU: host logic against loops of
the UNMODIFIED reference (tests/golden/samplers_tiny_2to1.pt, made by tools/make_sampler_golden.py), with
pn_sampler_step restated in torch (sampler_ref_ops.py) and the oracle network; the Philox restatement against the
published Random123 known-answer vectors; the C struct against its ctypes mirror."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import cases as Cs
from oracle import unet_port as P
from oracle.make_golden import sampler_inputs
from philox_ref import philox4x32_10, philox_normal
from sampler_ref_ops import TorchSamplerRefOps
from tools.make_sampler_golden import DISC, LOOPS, guider_config, noise_stream

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
NAMES = [name for name, *_ in LOOPS]


def make_sampler(cls, kwargs, guider, num_steps=10):
    from panacea_b200.sgm.util import instantiate_from_config
    return instantiate_from_config({"target": f"sgm.modules.diffusionmodules.sampling.{cls}",
                                    "params": dict(num_steps=num_steps, discretization_config=DISC,
                                                   guider_config=guider_config(guider), **kwargs)})


def _loop(name):
    return [entry for entry in LOOPS if entry[0] == name][0]


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN / "samplers_tiny_2to1.pt")


@pytest.mark.parametrize("name", NAMES)
def test_sampler_matches_reference_golden(name, golden):
    """Each sampler, fused path (BoundDenoiser) with the torch op set around the oracle network, with the reference's
    noise injected in draw order: same evaluation sequence and the reference's final latent within rel-L2 1e-4."""
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    from panacea_b200.sgm.util import instantiate_from_config
    _, cls, kw, guider = _loop(name)
    g = golden[name]
    case = Cs.GOLDEN_CASES[0]
    sd, cfg = Cs.make_weights(case), case.net_config()
    sampler = make_sampler(cls, kw, guider)
    sampler.ops = TorchSamplerRefOps()
    sampler.noise_sampler = noise_stream(g["noise_seed"])
    x, c, uc = sampler_inputs(case)
    den = instantiate_from_config(DEFAULT_DENOISER)
    out = sampler(BoundDenoiser(den, lambda xi, ti, ci: P.wrapper_forward(sd, cfg, xi, ti, ci)), x.clone(), c, uc)
    assert sampler.last_timestep_indices == g["timestep_indices"]
    rel = ((out - g["x_final"]).norm() / g["x_final"].norm()).item()
    assert rel < 1e-4, rel


@pytest.mark.parametrize("name", NAMES)
def test_host_scalars_equal_the_reference(name, golden):
    """get_ancestral_step, the DPM++ multipliers and the LMS coefficients computed before the loop equal the values the
    reference computed inside it (fp32 tensors, compared exactly; inf where the reference's torch.where discards them)."""
    _, cls, kw, guider = _loop(name)
    sampler = make_sampler(cls, kw, guider)
    init, evals = sampler.plan()
    assert sampler.host_scalars == golden[name]["scalars"]
    for e in [init] + [e.kw for e in evals]:            # the kernel never sees a non-finite coefficient
        vals = [v for k, v in e.items() if k in ("coef", "dt", "sigma", "noise_amp")]
        flat = [float(u) for v in vals for u in (v if isinstance(v, (list, tuple)) else [v])]
        assert all(np.isfinite(flat)), e
    assert len(evals) == len(golden[name]["timestep_indices"])


def test_dpmpp_2m_last_step_takes_x_standard():
    """sigma_next = 0: the reference computes -log 0 = inf and selects x_standard with torch.where; the host picks
    that branch (mode DPM, multipliers 0 and -1)."""
    from panacea_b200.sgm.modules.diffusionmodules.sampling import DPM
    sampler = make_sampler("DPMPP2MSampler", {}, "cfg")
    _, evals = sampler.plan()
    assert evals[-1].mode == DPM and list(evals[-1].kw["coef"]) == [0.0, -1.0]
    assert evals[0].mode == DPM and all(e.mode != DPM for e in evals[1:-1])


def test_philox_restatement_reproduces_random123_known_answers():
    """Philox4x32-10 known-answer vectors published with Random123 (kat_vectors: counter, key -> output)."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = philox4x32_10(np.array([ctr], np.uint32), np.array(key, np.uint32))[0]
        assert [int(v) for v in got] == list(want)
    z = philox_normal(7, 3, 200_000).astype(np.float64)
    assert abs(z.mean()) < 5 / np.sqrt(z.size) and abs(z.var() - 1.0) < 5 * np.sqrt(2.0 / z.size)


def test_default_noise_is_seeded_by_torch_manual_seed():
    """Without a noise_sampler the noise is the Philox stream under a seed drawn from torch's default CPU generator:
    the same torch.manual_seed gives the same sample, another seed a different one."""
    x = torch.randn(2, 4, 8, 96, generator=torch.Generator().manual_seed(0))
    net_eps = lambda xi, ti, ci: 0.1 * xi               # any deterministic network
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    from panacea_b200.sgm.util import instantiate_from_config
    den = instantiate_from_config(DEFAULT_DENOISER)
    outs = []
    for seed in (5, 5, 6):
        sampler = make_sampler("EulerAncestralSampler", {}, "identity", num_steps=3)
        sampler.ops = TorchSamplerRefOps()
        torch.manual_seed(seed)
        outs.append(sampler(BoundDenoiser(den, net_eps), x.clone(), {"crossattn": torch.zeros(1)}))
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])


def test_sampler_step_struct_matches_header_field_order():
    from panacea_b200 import _lib
    text = (ROOT / "include" / "panacea_b200.h").read_text()
    body = re.search(r"typedef struct pn_sampler_step_args \{(.*?)\} pn_sampler_step_args;", text, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            fields += [re.sub(r"\[.*?\]", "", part.strip().split()[-1].lstrip("*")) for part in decl.split(",")]
    assert fields == [f[0] for f in _lib.SamplerStepArgs._fields_]
    modes = re.search(r"enum pn_sampler_mode \{(.*?)\};", text, flags=re.S).group(1)
    modes = re.sub(r"/\*.*?\*/", "", modes, flags=re.S)
    from panacea_b200 import ops
    from panacea_b200.sgm.modules.diffusionmodules import sampling as S
    for name, value in re.findall(r"PN_SAMPLER_(\w+)\s*=\s*(\d+)", modes):
        assert getattr(ops, f"SAMPLER_{name}") == int(value) == getattr(S, name)


def test_every_reference_sampler_is_exported_for_the_sgm_namespace():
    from panacea_b200.sgm.util import get_obj_from_str
    for cls in ("BaseDiffusionSampler", "SingleStepDiffusionSampler", "EDMSampler", "AncestralSampler", "EulerEDMSampler",
                "HeunEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
                "LinearMultistepSampler"):
        obj = get_obj_from_str(f"sgm.modules.diffusionmodules.sampling.{cls}")
        assert obj.__module__.startswith("panacea_b200."), cls
    for fn in ("get_ancestral_step", "linear_multistep_coeff", "to_d", "to_neg_log_sigma", "to_sigma"):
        assert get_obj_from_str(f"sgm.modules.diffusionmodules.sampling_utils.{fn}").__module__.startswith("panacea_b200.")


def test_install_as_sgm_builds_and_runs_every_sampler():
    """With the mirror installed as `sgm`, every reference sampler class builds from its config — Euler with churn, and
    without a guider_config (the reference default IdentityGuider) — and samples."""
    import sys
    import panacea_b200.sgm as S
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    saved = {k: v for k, v in sys.modules.items() if k == "sgm" or k.startswith("sgm.")}
    for k in saved:
        del sys.modules[k]
    try:
        S.install_as_sgm()
        import sgm.modules.diffusionmodules.sampling as sampling
        from sgm.util import instantiate_from_config
        den = instantiate_from_config(DEFAULT_DENOISER)
        x = torch.randn(2, 4, 8, 48, generator=torch.Generator().manual_seed(1))
        c = {"crossattn": torch.zeros(1, 77, 8)}
        for cls, kw in (("EulerEDMSampler", {"s_churn": 1.0}), ("HeunEDMSampler", {}), ("EulerAncestralSampler", {}),
                        ("DPMPP2SAncestralSampler", {}), ("DPMPP2MSampler", {}), ("LinearMultistepSampler", {})):
            for guider in (None, {"target": "sgm.modules.diffusionmodules.guiders.VanillaCFG", "params": {"scale": 5.0}}):
                params = dict(kw, num_steps=4, discretization_config=DISC)
                if guider is not None:
                    params["guider_config"] = guider
                sampler = getattr(sampling, cls)(**params)
                assert type(sampler).__module__.startswith("panacea_b200.")
                sampler.ops = TorchSamplerRefOps()
                out = sampler(BoundDenoiser(den, lambda xi, ti, ci: 0.1 * xi), x.clone(), c, c)
                assert out.shape == x.shape and torch.isfinite(out).all(), (cls, guider)
    finally:
        for k in [k for k in sys.modules if k == "sgm" or k.startswith("sgm.")]:
            del sys.modules[k]
        sys.modules.update(saved)
