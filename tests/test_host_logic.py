"""CPU tests of the host side: plan/spec, state-dict compatibility of the drop-in modules, weight packing and the
engine's orchestration (run through a torch test op set, tests/torch_ref_ops.py) against the reference goldens."""
from pathlib import Path

import pytest
import torch

from oracle import cases as Cs
from oracle import unet_port as P
from panacea_b200 import engine as E
from panacea_b200 import netplan as NP
from torch_ref_ops import TorchFoldOps, TorchRefOps, TorchSplitOps

GOLDEN = Path(__file__).resolve().parent / "golden"


def _split(sd):
    up = {k[len("diffusion_model."):]: v for k, v in sd.items() if not k.startswith("diffusion_model.controlnet.")}
    cp = {k[len("diffusion_model.controlnet."):]: v for k, v in sd.items() if k.startswith("diffusion_model.controlnet.")}
    return up, cp


def test_param_spec_equals_reference_key_set():
    cfg = NP.config_from_kwargs(Cs.GOLDEN_CASES[4].unet_kwargs())
    full = {"diffusion_model." + k: v for k, v in NP.unet_param_spec(cfg).items()}
    full.update({"diffusion_model.controlnet." + k: v for k, v in NP.controlnet_param_spec(cfg).items()})
    assert full == P.state_spec(P.NetConfig())
    plan = NP.make_plan(cfg, True)
    kinds = [st.kind for st in plan.stages()]
    assert kinds.count("res") == 22 and kinds.count("stt") == 16          # SURVEY.md section 3.5
    assert [st.kind for st in NP.make_plan(cfg, False).stages()].count("stt") == 7


def test_unsupported_configurations_are_rejected_loudly():
    kw = Cs.GOLDEN_CASES[0].unet_kwargs()
    for bad in (dict(use_scale_shift_norm=True), dict(resblock_updown=True), dict(transformer_depth=2),
                dict(insert_crossview=False), dict(num_classes=10), dict(legacy=True)):
        with pytest.raises(NotImplementedError):
            NP.config_from_kwargs(dict(kw, **bad))


@pytest.mark.parametrize("name", ["tiny_2to1", "tiny_3to1", "small_hd64"])
def test_engine_orchestration_matches_reference_golden(name):
    case = [c for c in Cs.GOLDEN_CASES if c.name == name][0]
    cfg = NP.config_from_kwargs(case.unet_kwargs())
    eng = E.Engine(cfg, TorchRefOps())
    eng.pack(*_split(Cs.make_weights(case)))
    x, t, c = Cs.make_inputs(case)
    eng.prepare_condition(c["cond_feat"], c["crossattn"])
    eps = eng.eps(x, c["concat"], t)
    g = torch.load(GOLDEN / f"eps_{name}.pt")["eps"]
    assert (eps - g).abs().max().item() < 2e-5
    # CFG: hint given once for both halves
    half = x.shape[0] // case.b
    if case.b == 2:
        eng.prepare_condition(c["cond_feat"][:half], c["crossattn"], hint_repeat=1)
        eng.prepare_hint(torch.cat([c["cond_feat"][:half]] * 1), hint_repeat=1)


@pytest.mark.parametrize("name", ["tiny_3to1", "small_hd64"])
def test_parity_mode_split_operands_reach_fp32_class_accuracy(name):
    """Parity mode on CPU: the engine packs weights [W_hi | W_hi | W_lo] and every producer stores [hi | lo | hi]
    (emulated by TorchSplitOps with exact bf16-value products). Against the reference golden the literal BASELINE
    tolerance rtol 1e-3 / atol 1e-4 must hold on (essentially) every element — the same packing runs on the GPU through
    the wgmma kernel."""
    case = [c for c in Cs.GOLDEN_CASES if c.name == name][0]
    cfg = NP.config_from_kwargs(case.unet_kwargs())
    eng = E.Engine(cfg, TorchSplitOps())
    eng.pack(*_split(Cs.make_weights(case)))
    x, t, c = Cs.make_inputs(case)
    eng.prepare_condition(c["cond_feat"], c["crossattn"])
    eps = eng.eps(x, c["concat"], t)
    g = torch.load(GOLDEN / f"eps_{name}.pt")["eps"]
    d = (eps - g).abs()
    frac = (d <= 1e-4 + 1e-3 * g.abs()).float().mean().item()
    rel = ((eps - g).norm() / g.norm()).item()
    assert frac >= 0.999 and rel < 1e-4, (frac, rel)


def test_layernorm_fold_orchestration_matches_reference_golden():
    """Fast-path orchestration with the three LayerNorms of every transformer block folded into the GEMMs around the
    token stream (row sums from the producer epilogue, W diag(gamma) + rank-1 correction in the consumer): must reproduce
    the reference golden up to the bf16 rounding of the folded weights."""
    case = [c for c in Cs.GOLDEN_CASES if c.name == "small_hd64"][0]
    cfg = NP.config_from_kwargs(case.unet_kwargs())
    ops = TorchFoldOps()
    eng = E.Engine(cfg, ops)
    eng.pack(*_split(Cs.make_weights(case)))
    assert any(v is True for k, v in eng.wu.items() if k.endswith(".fold"))
    x, t, c = Cs.make_inputs(case)
    eng.prepare_condition(c["cond_feat"], c["crossattn"])
    eps = eng.eps(x, c["concat"], t)
    g = torch.load(GOLDEN / "eps_small_hd64.pt")["eps"]
    rel = ((eps - g).norm() / g.norm()).item()
    assert rel < 3e-3, rel                                  # bf16-rounded W diag(gamma); a wrong fold is O(1) off


def test_dropin_modules_share_the_reference_state_dict():
    from panacea_b200.pipeline import default_network_config
    from panacea_b200.sgm.modules.diffusionmodules import OpenAIWrapperControlLDM3D
    from panacea_b200.sgm.util import instantiate_from_config
    case = Cs.GOLDEN_CASES[0]
    kw = case.unet_kwargs()
    model = instantiate_from_config(default_network_config(**{k: kw[k] for k in ("model_channels", "num_head_channels", "context_dim", "num_frames")}))
    w = OpenAIWrapperControlLDM3D(model)
    ref_sd = Cs.make_weights(case)
    assert {k: tuple(v.shape) for k, v in w.state_dict().items()} == {k: tuple(v.shape) for k, v in ref_sd.items()}
    # reference default init reproduces the zero_module()'d tails
    z = [k for k, v in w.state_dict().items() if v.abs().sum() == 0 and k.endswith("weight")]
    assert any("proj_out_crossview" in k for k in z) and any("zero_convs" in k for k in z) and "diffusion_model.out.2.weight" in z
    res = w.load_state_dict(ref_sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(w.state_dict()["diffusion_model.controlnet.input_hint_block.14.weight"],
                       ref_sd["diffusion_model.controlnet.input_hint_block.14.weight"])
    with pytest.raises(RuntimeError):
        w.load_state_dict({**ref_sd, "diffusion_model.bogus.weight": torch.zeros(1)}, strict=True)
    # engine checkpoints carry a "model." prefix and DeepSpeed's "_forward_module." (inference.py:209-211)
    wrapped = {"model." + k: v for k, v in ref_sd.items()}

    class Host(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.model = w
    assert not Host().load_state_dict(wrapped, strict=True).missing_keys
    with pytest.raises(RuntimeError):
        w(torch.zeros(4, 4, 8, 96), torch.zeros(4, dtype=torch.int64), {})       # CPU tensors: no CPU path


def test_denoiser_and_sampler_host_scalars():
    from panacea_b200.pipeline import DEFAULT_DENOISER, default_sampler_config
    from panacea_b200.sgm.util import instantiate_from_config
    kat = torch.load(GOLDEN / "kat.pt")
    den = instantiate_from_config(DEFAULT_DENOISER)
    assert torch.equal(den.sigmas, kat["denoiser_sigmas"])
    assert torch.equal(den.sigma_to_idx(kat["sigmas_50"][:-1]), kat["idx_of_sigmas_50"])
    sampler = instantiate_from_config(default_sampler_config(25, 5.0))
    assert torch.equal(sampler.sigmas(), kat["sigmas_25"]) and torch.equal(sampler.sigmas(50), kat["sigmas_50"])
    idx, sq, c_in = den.step_scalars(float(kat["sigmas_25"][3]))
    assert idx == 999 - 3 * 40 and sq == float(kat["sigmas_25"][3]) and abs(c_in - (sq * sq + 1) ** -0.5) < 1e-7
    assert sampler.guider.scale == 5.0
    # a plain callable is accepted (the reference passes a lambda, diffusion.py:251-254); without a CUDA device the first
    # native op of the loop fails loudly — there is no CPU path
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError):
            sampler(lambda *a: None, torch.zeros(1, 4, 8, 8), {}, {})


def test_install_as_sgm_resolves_reference_targets():
    import sys
    import panacea_b200.sgm as S
    saved = {k: v for k, v in sys.modules.items() if k == "sgm" or k.startswith("sgm.")}
    for k in saved:
        del sys.modules[k]
    try:
        S.install_as_sgm()
        import sgm.modules.diffusionmodules.controlmodel as cm
        assert cm.ControlledUNetModel3D.__module__.startswith("panacea_b200.")
    finally:
        for k in [k for k in sys.modules if k == "sgm" or k.startswith("sgm.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_geglu_pack_is_the_layout_the_epilogue_contract_states():
    """include/panacea_b200.h: GEGLU columns come in blocks of 32 = 16 value columns then the 16 gate columns of the same
    outputs; packing the reference's [value rows | gate rows] projection (attention.py:94-99) and applying the blockwise
    rule must reproduce value * gelu(gate)."""
    import torch.nn.functional as F
    from panacea_b200.ops import geglu_pack
    g = torch.Generator().manual_seed(5)
    inner, C, M = 64, 48, 7
    w = torch.randn(2 * inner, C, generator=g)
    b = torch.randn(2 * inner, generator=g)
    x = torch.randn(M, C, generator=g)
    wp, bp = geglu_pack(w), geglu_pack(b)
    assert wp.shape == w.shape and bp.shape == b.shape
    # block structure: rows [32k, 32k+16) are value rows 16k.., rows [32k+16, 32k+32) the matching gate rows
    assert torch.equal(wp[0:16], w[0:16]) and torch.equal(wp[16:32], w[inner:inner + 16])
    assert torch.equal(wp[32:48], w[16:32]) and torch.equal(wp[48:64], w[inner + 16:inner + 32])
    y = x @ w.t() + b
    ref = y[:, :inner] * F.gelu(y[:, inner:])
    got = TorchRefOps().gemm(x, wp, bias=bp, geglu=True, out_dtype=torch.float32)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError):
        geglu_pack(torch.zeros(40, 4))


def test_geglu_erfc_constants_in_the_kernel_source_are_accurate():
    """The GEGLU epilogue evaluates Phi(-t) = 0.5 * 2^(-t Q(t)) with a fitted degree-4 Q and NO clamp of t = |g|
    (ptx.cuh::geglu_f32, generated by tools/fit_erfc.py). Re-evaluate the constants found in the kernel source in fp32
    on the CPU against the exact erf GELU of the reference (attention.py:97-99 -> F.gelu), far beyond the fitted range too."""
    import re
    import numpy as np
    src = (Path(__file__).resolve().parent.parent / "panacea_b200" / "csrc" / "ptx.cuh").read_text()
    body = src[src.index("__device__ __forceinline__ float geglu_f32"):]
    body = body[:body.index("\n}\n")]
    coef = [float(x) for x in re.findall(r"(-?[0-9]+\.[0-9]+(?:e[-+]?[0-9]+)?)f\b", body)]
    # Horner order in the source: c4, c3, ..., c0, then the -0.5 / 0.5 / 0.5 of the final combination
    c = np.array(coef[:5], dtype=np.float32)
    assert len(coef) >= 5 and abs(c[-1] - 1.1510913) < 1e-6 and c[0] > 0          # positive leading coefficient: no clamp needed
    assert "fminf" not in body
    g = np.concatenate([np.linspace(-9.0, 9.0, 200001), np.array([-1e30, -1e4, -50.0, 50.0, 1e4, 1e30])]).astype(np.float32)
    t = np.abs(g)
    q = np.full_like(t, c[0])
    with np.errstate(over="ignore"):
        for k in range(1, 5):
            q = (q * t + c[k]).astype(np.float32)
        e = np.exp2((-(q * t)).astype(np.float32)).astype(np.float32)
    r = (np.float32(0.5) - np.float32(0.5) * e).astype(np.float32)
    gelu = (np.float32(0.5) * g + np.abs(g) * r).astype(np.float32)
    ref = torch.nn.functional.gelu(torch.from_numpy(g).double()).numpy()
    assert np.abs(gelu[:200001] - ref[:200001]).max() < 2e-6
    assert np.all(np.abs(gelu[200001:] - ref[200001:]) <= 1e-6 * np.abs(ref[200001:]))
