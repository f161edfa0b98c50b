"""The VAE in parity precision, without a GPU: the parity orchestration of `VAEDecoderEngine` / `VAEEncoderEngine`
(split-bf16 operands everywhere, the mid-block attention with its device-made weight-form operands) on a CPU emulation
of the split encoding, against the UNMODIFIED reference's outputs at the shrunk width (tests/golden/vae_decode_small.pt)
and at the real channel width, C = 512 in the mid block (tests/golden/vae_full_width.pt, `python -m tools.make_vae_golden`).
Also the precision plumbing of the first-stage wrapper that needs no device."""
from pathlib import Path

import pytest
import torch

from oracle.make_golden import VAE_DDCONFIG, vae_decoder_input, vae_decoder_weights, vae_encoder_input
from panacea_b200.vae import VAEDecoderEngine, VAEEncoderEngine, decoder_param_spec, encoder_param_spec
from test_eps_parity_gpu import BOUNDS
from tools.make_vae_golden import FULL_WIDTH_DDCONFIG, full_width_inputs
from torch_ref_ops import TorchSplitOps

GOLDEN = Path(__file__).resolve().parent / "golden"


def _check_parity(name, got, ref):
    b_rel, b_max, b_frac = BOUNDS["parity"]
    d = (got - ref).double()
    rel = (d.norm() / ref.double().norm()).item()
    rms = ref.double().pow(2).mean().sqrt().item()
    frac = (d.abs() <= 1e-4 + 1e-3 * ref.double().abs()).double().mean().item()
    assert got.shape == ref.shape and torch.isfinite(got).all()
    assert rel <= b_rel, f"{name}: rel-L2 {rel:.3e} > {b_rel}"
    assert d.abs().max().item() <= b_max * rms, f"{name}: max-abs {d.abs().max().item():.3e} vs rms {rms:.3e}"
    assert frac >= b_frac, f"{name}: only {frac:.5f} of the elements inside rtol 1e-3 / atol 1e-4"


def _cases():
    small = torch.load(GOLDEN / "vae_decode_small.pt")
    full = torch.load(GOLDEN / "vae_full_width.pt")
    z, x = full_width_inputs()
    return {
        "small": (VAE_DDCONFIG, small, 7, 9, vae_decoder_input(), vae_encoder_input()),
        "full_width": (FULL_WIDTH_DDCONFIG, full, full["decoder_seed"], full["encoder_seed"], z, x),
    }


@pytest.mark.parametrize("case", ["small", "full_width"])
def test_parity_decoder_orchestration_matches_the_reference(case):
    dd, g, dseed, _, z, _ = _cases()[case]
    eng = VAEDecoderEngine(dd, TorchSplitOps())
    eng.pack(vae_decoder_weights(eng.spec, seed=dseed))
    _check_parity(f"vae_decode_{case}", eng.decode(z), g["image"])


@pytest.mark.parametrize("case", ["small", "full_width"])
def test_parity_encoder_orchestration_matches_the_reference(case):
    dd, g, _, eseed, _, x = _cases()[case]
    eng = VAEEncoderEngine(dd, TorchSplitOps())
    eng.pack(vae_decoder_weights(eng.spec, seed=eseed))
    _check_parity(f"vae_encode_{case}", eng.encode_moments(x), g["moments"])


def test_full_width_golden_keys_are_the_engine_specs():
    g = torch.load(GOLDEN / "vae_full_width.pt")
    assert g["ddconfig"] == FULL_WIDTH_DDCONFIG and FULL_WIDTH_DDCONFIG["ch"] * FULL_WIDTH_DDCONFIG["ch_mult"][-1] == 512
    assert g["keys"] == sorted(decoder_param_spec(FULL_WIDTH_DDCONFIG, 4))
    assert g["encoder_keys"] == sorted(encoder_param_spec(FULL_WIDTH_DDCONFIG, 4))
    assert tuple(g["image"].shape) == (2, 3, 64, 384) and tuple(g["moments"].shape) == (2, 8, 8, 48)


def test_weight_form_emulation_is_split3():
    from panacea_b200.ops import split3
    w = torch.randn(24, 40, generator=torch.Generator().manual_seed(5))
    assert torch.equal(TorchSplitOps().cast_operand(w, weight_form=True), split3(w))


def _wrapper(**kw):
    from panacea_b200.sgm.models.autoencoder import AutoencoderKLInferenceWrapper
    return AutoencoderKLInferenceWrapper(embed_dim=4, ddconfig=VAE_DDCONFIG, lossconfig={"target": "torch.nn.Identity"}, **kw)


def test_wrapper_precision_resolves_like_the_unet(monkeypatch):
    monkeypatch.delenv("PN_PRECISION", raising=False)
    assert _wrapper().precision == "bf16"
    assert _wrapper(precision="parity").precision == "parity"
    monkeypatch.setenv("PN_PRECISION", "parity")
    assert _wrapper().precision == "parity"
    assert _wrapper(precision="bf16").precision == "bf16"
    m = _wrapper(precision="bf16")
    m.set_precision("parity")
    assert m.precision == "parity"
    with pytest.raises(ValueError):
        m.set_precision("fp8")
    with pytest.raises(ValueError):
        _wrapper(precision="fp8")


@pytest.mark.parametrize("precision", ["bf16", "parity"])
def test_wrapper_has_no_cpu_path(precision):
    m = _wrapper(precision=precision)
    with pytest.raises(RuntimeError):
        m.decode(torch.zeros(2, 4, 8, 48))
    with pytest.raises(RuntimeError):
        m.encode(torch.zeros(2, 3, 32, 192))


def test_engine_precision_reaches_the_first_stage():
    """`model.params.precision=parity` on the inference command line sets the UNet, the text tower and the VAE (which
    the VAEEmbedder of the image condition shares)."""
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.modules.encoders.modules import VAEEmbedder
    from panacea_b200.sgm.util import instantiate_from_config
    cfg = str(Path(__file__).resolve().parent / "configs" / "tiny_inference.yaml")
    m = instantiate_from_config(load_config([cfg], ["model.params.precision=parity"])["model"])
    assert m.first_stage_model.precision == "parity"
    emb = [e for e in m.conditioner.embedders if isinstance(e, VAEEmbedder)]
    assert emb and emb[0].first_stage_model is m.first_stage_model


def test_frame_chunks_keep_every_groupnorm_split():
    """The planner allows a chunk size only where GroupNorm splits each frame the same way as one call over all frames
    (here a stand-in geometry: one frame per call doubles the split), and uses as few calls as possible."""
    eng = VAEDecoderEngine(FULL_WIDTH_DDCONFIG, TorchSplitOps())
    eng.ops = type("Geometry", (), {"groupnorm_ctas_per_frame": staticmethod(lambda f, P, C: 132 // min(f, 2))})()
    assert eng.frame_chunks(8, (32, 384), 8) == [8]
    assert eng.frame_chunks(8, (32, 384), 2) == [2, 2, 2, 2]
    assert eng.frame_chunks(7, (32, 384), 2) == [7]            # a 1-frame call would change the split: no chunking
    assert sorted(eng.frame_chunks(7, (32, 384), 3)) == [2, 2, 3]
    eng.ops = type("Geometry", (), {"groupnorm_ctas_per_frame": staticmethod(lambda f, P, C: 66)})()
    assert sorted(eng.frame_chunks(5, (32, 384), 2)) == [1, 2, 2]


def test_wrapper_frames_per_call_defaults():
    assert _wrapper(precision="parity").frames_per_call is None
    m = _wrapper(precision="parity", frames_per_call=4)
    assert m.frames_per_call == 4


def _groupnorm_shapes_of_a_run(Eng, dd, inp):
    """(pixels, channels) of every groupnorm call an engine run makes (CPU, fp32 torch op set)"""
    from torch_ref_ops import TorchRefOps

    class Recording(TorchRefOps):
        seen = set()

        def groupnorm(self, x, *a, **k):
            self.seen.add((x.numel() // (x.shape[0] * x.shape[-1]), x.shape[-1]))
            return super().groupnorm(x, *a, **k)
    eng = Eng(dd, Recording())
    eng.pack(vae_decoder_weights(eng.spec))
    eng.decode(inp) if Eng is VAEDecoderEngine else eng.encode_moments(inp)
    return eng, sorted(Recording.seen)


@pytest.mark.parametrize("Eng", [VAEDecoderEngine, VAEEncoderEngine])
def test_frame_chunk_planner_knows_every_groupnorm_shape(Eng):
    z, x = full_width_inputs()
    inp = z[:1] if Eng is VAEDecoderEngine else x[:1]
    eng, seen = _groupnorm_shapes_of_a_run(Eng, FULL_WIDTH_DDCONFIG, inp)
    assert eng._gn_shapes(tuple(inp.shape[2:])) == seen

