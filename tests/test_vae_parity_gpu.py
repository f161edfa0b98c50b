"""The VAE in parity precision on the GPU: the two operand forms its mid-block attention adds (the weight-form
`pn_cast_operand` and `pn_softmax_rows_operand`), the parity decoder / encoder against the UNMODIFIED reference at the
shrunk and the real channel width, one full-size frame against an fp32 torch run of the same orchestration, and the
precision plumbing of the first stage inside the inference engine. Parity rates go to parity.jsonl through
test_eps_parity_gpu._report."""
import ctypes as C
from pathlib import Path

import pytest
import torch

from op_check import _decode
from oracle.make_golden import VAE_DDCONFIG, vae_decoder_input, vae_decoder_weights, vae_encoder_input
from panacea_b200.vae import decoder_param_spec, encoder_param_spec
from test_eps_parity_gpu import _report
from tools.make_vae_golden import FULL_WIDTH_DDCONFIG, full_width_inputs

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")


def _wrapper(dd, precision=None, sd=None, **kw):
    from panacea_b200.sgm.models.autoencoder import AutoencoderKLInferenceWrapper
    if precision is not None:
        kw["precision"] = precision
    m = AutoencoderKLInferenceWrapper(embed_dim=4, ddconfig=dd, lossconfig={"target": "torch.nn.Identity"}, **kw)
    if sd is not None:
        m.load_state_dict(sd, strict=False)
    return m.cuda()


# ------------------------------------------------------------------------------------------------ kernels
def test_weight_form_cast_is_host_split3():
    from panacea_b200.ops import ParityOps, split3, split_encode
    ops = ParityOps()
    for rows, cols in ((300, 520), (64, 12288), (7, 4)):
        w = torch.randn(rows, cols, generator=torch.Generator().manual_seed(rows)) * 3.0
        got = ops.cast_operand(w.cuda(), weight_form=True).cpu()
        assert torch.equal(got, split3(w)), (rows, cols)
        assert torch.equal(ops.cast_operand(w.cuda()).cpu(), split_encode(w)), (rows, cols)


def _softmax_operand(lib, s, mode, out, scale):
    from panacea_b200.ops import _stream
    return lib.pn_softmax_rows_operand(C.c_void_p(s.data_ptr()), C.c_void_p(out.data_ptr()), s.shape[0], s.shape[1], s.stride(0),
                                       out.stride(0), scale, mode, _stream())


@pytest.mark.parametrize("rows,N", [(7, 768), (300, 12288), (4, 51200)])
def test_softmax_rows_operand(rows, N):
    from panacea_b200.ops import OP_BF16, NativeOps, ParityOps
    ops, pops = NativeOps(), ParityOps()
    scale = 512 ** -0.5
    s = (torch.randn(rows, N, generator=torch.Generator().manual_seed(N)) * 20).cuda()
    ref_bf16 = ops.softmax_rows(s, scale)
    got_bf16 = torch.empty_like(ref_bf16)
    assert _softmax_operand(ops.lib, s, OP_BF16, got_bf16, scale) == 0
    assert torch.equal(got_bf16, ref_bf16), "bf16 mode must be bitwise NativeOps.softmax_rows"
    p3 = pops.softmax_rows(s, scale)
    assert p3.shape == (rows, 3 * N) and p3.dtype == torch.bfloat16
    ref = torch.softmax(s.double() * scale, dim=-1)
    rel = ((_decode(p3, "split3") - ref).abs() / ref).max().item()
    assert rel <= 1e-5, rel


def test_softmax_rows_operand_rejects_what_it_cannot_do():
    from panacea_b200.ops import OP_F32, OP_SPLIT3, OP_SPLIT3_B, ParityOps, _ptr, _stream
    pops = ParityOps()
    lib = pops.lib
    N = 51204                                          # one float4 past the 200 KB shared-memory row buffer
    s = torch.zeros(2, N, device="cuda")
    out = torch.empty(2, 3 * N, device="cuda", dtype=torch.bfloat16)
    assert _softmax_operand(lib, s, OP_SPLIT3, out, 1.0) != 0
    assert b"exceeds the shared-memory row buffer" in lib.pn_last_error()
    s = torch.zeros(2, 64, device="cuda")
    for mode in (OP_F32, OP_SPLIT3_B):
        assert _softmax_operand(lib, s, mode, out, 1.0) != 0 and b"operand_mode" in lib.pn_last_error()
    x = torch.zeros(1, 4, 4, 64, device="cuda")       # the weight form is pn_cast_operand's only
    y = torch.empty(1, 8, 8, 192, device="cuda", dtype=torch.bfloat16)
    assert lib.pn_upsample2x(_ptr(x), _ptr(y), 1, 4, 4, 64, OP_SPLIT3_B, _stream()) != 0
    assert b"operand_mode 3" in lib.pn_last_error()
    assert lib.pn_gelu_operand(_ptr(x), _ptr(y), 16, 64, OP_SPLIT3_B, _stream()) != 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ vs the reference
def _golden_case(name):
    if name == "small":
        g = torch.load(GOLDEN / "vae_decode_small.pt")
        return VAE_DDCONFIG, g, 7, 9, vae_decoder_input(), vae_encoder_input()
    g = torch.load(GOLDEN / "vae_full_width.pt")
    z, x = full_width_inputs()
    return FULL_WIDTH_DDCONFIG, g, g["decoder_seed"], g["encoder_seed"], z, x


@pytest.mark.parametrize("name", ["small", "full_width"])
def test_parity_decoder_matches_the_reference(name):
    dd, g, dseed, _, z, _ = _golden_case(name)
    m = _wrapper(dd, "parity", vae_decoder_weights(decoder_param_spec(dd, 4), seed=dseed))
    out = m.decode(z.cuda()).cpu()
    _report(f"vae_decode_{name}:vs_reference_golden", out, g["image"], "parity")


@pytest.mark.parametrize("name", ["small", "full_width"])
def test_parity_encoder_matches_the_reference(name):
    dd, g, _, eseed, _, x = _golden_case(name)
    m = _wrapper(dd, "parity", vae_decoder_weights(encoder_param_spec(dd, 4), seed=eseed))
    mom = m.encode_moments(x.cuda()).cpu()
    _report(f"vae_encode_{name}:vs_reference_golden", mom, g["moments"], "parity")


def _fp32_torch(fn):
    """run fn with the fp32 torch op set on the GPU: TF32 off, factory functions on cuda"""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.device("cuda"):
            return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def test_parity_full_size_frame_matches_fp32_torch():
    """One frame at the headline size: latent 32 x 384 (P = 12,288 tokens in the mid attention), image 256 x 3072."""
    from panacea_b200.ops import ParityOps
    from panacea_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    from torch_ref_ops import TorchRefOps
    dd = FULL_WIDTH_DDCONFIG
    g = torch.Generator().manual_seed(41)
    z = torch.randn(1, 4, 32, 384, generator=g).cuda()
    x = (torch.rand(1, 3, 256, 3072, generator=g) * 2.0 - 1.0).cuda()
    for Eng, seed, run, inp, name in ((VAEDecoderEngine, 31, "decode", z, "vae_decode_full_size"),
                                      (VAEEncoderEngine, 32, "encode_moments", x, "vae_encode_full_size")):
        eng = Eng(dd, ParityOps())
        P = {k: v.cuda() for k, v in vae_decoder_weights(eng.spec, seed=seed).items()}
        eng.pack(P)
        got = getattr(eng, run)(inp).cpu()
        del eng
        ref_eng = Eng(dd, TorchRefOps())
        ref = _fp32_torch(lambda: (ref_eng.pack(P), getattr(ref_eng, run)(inp))[1]).cpu()
        del ref_eng
        torch.cuda.empty_cache()
        _report(name + ":vs_fp32_torch", got, ref, "parity")


# ------------------------------------------------------------------------------------------------ frame chunks
@pytest.mark.parametrize("run", ["decode", "encode_moments"])
def test_frame_chunked_parity_is_bitwise_one_call_at_full_size(run):
    """A parity run splits 8 full-size frames into calls of 2 (the default): bitwise the output of one 8-frame call."""
    dd = FULL_WIDTH_DDCONFIG
    sd = {**vae_decoder_weights(decoder_param_spec(dd, 4), seed=31), **vae_decoder_weights(encoder_param_spec(dd, 4), seed=32)}
    g = torch.Generator().manual_seed(43)
    inp = torch.randn(8, 4, 32, 384, generator=g) if run == "decode" else torch.rand(8, 3, 256, 3072, generator=g) * 2.0 - 1.0
    inp = inp.cuda()
    chunked = _wrapper(dd, "parity", sd)
    a = getattr(chunked, run)(inp)
    eng = chunked._engine if run == "decode" else chunked._enc_engine
    assert eng.frame_chunks(8, tuple(inp.shape[2:]), chunked.PARITY_FRAMES_PER_CALL) == [2, 2, 2, 2]
    del chunked, eng
    whole = _wrapper(dd, "parity", sd, frames_per_call=8)
    b = getattr(whole, run)(inp)
    assert torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.parametrize("precision", ["parity", "bf16"])
def test_frame_chunked_small_frames_are_bitwise_one_call(precision):
    """5 small frames, at most 2 per call: whatever split the planner picks (or none) reproduces one call bit for bit."""
    sd = {**vae_decoder_weights(decoder_param_spec(VAE_DDCONFIG, 4)), **vae_decoder_weights(encoder_param_spec(VAE_DDCONFIG, 4), seed=9)}
    g = torch.Generator().manual_seed(44)
    z = torch.randn(5, 4, 8, 48, generator=g).cuda()
    x = (torch.rand(5, 3, 64, 384, generator=g) * 2.0 - 1.0).cuda()
    split, whole = _wrapper(VAE_DDCONFIG, precision, sd, frames_per_call=2), _wrapper(VAE_DDCONFIG, precision, sd, frames_per_call=5)
    assert torch.equal(split.decode(z), whole.decode(z))
    assert torch.equal(split.encode_moments(x), whole.encode_moments(x))


# ------------------------------------------------------------------------------------------------ plumbing
def test_default_and_explicit_bf16_agree_and_survive_a_parity_round_trip(monkeypatch):
    monkeypatch.delenv("PN_PRECISION", raising=False)
    dd = FULL_WIDTH_DDCONFIG
    sd = {**vae_decoder_weights(decoder_param_spec(dd, 4), seed=31), **vae_decoder_weights(encoder_param_spec(dd, 4), seed=32)}
    z, x = (t.cuda() for t in full_width_inputs())
    d_default = _wrapper(dd, None, sd)
    m = _wrapper(dd, "bf16", sd)
    img, mom = m.decode(z), m.encode_moments(x)
    assert d_default.precision == "bf16"
    assert torch.equal(d_default.decode(z), img) and torch.equal(d_default.encode_moments(x), mom)
    m.set_precision("parity")
    img_p, mom_p = m.decode(z), m.encode_moments(x)
    assert not torch.equal(img_p, img)
    m.set_precision("bf16")
    assert torch.equal(m.decode(z), img) and torch.equal(m.encode_moments(x), mom)


def test_parity_engine_runs_log_images_on_a_parity_first_stage():
    """tiny_inference.yaml with model.params.precision=parity: log_images runs, and c["concat"] (the VAEEmbedder's
    encoding of the image condition) is bitwise a standalone parity wrapper's scale_factor * encode with the same
    weights and the same CPU generator state."""
    from torch.utils.data import DataLoader
    from panacea_b200.inference import SyntheticBEVDataset, load_config
    from panacea_b200.ops import ParityOps
    from panacea_b200.sgm.modules.encoders.modules import VAEEmbedder
    from panacea_b200.sgm.util import instantiate_from_config
    m = instantiate_from_config(load_config([CFG], ["model.params.precision=parity"])["model"]).cuda().eval()
    assert m.first_stage_model.precision == "parity"
    emb = [e for e in m.conditioner.embedders if isinstance(e, VAEEmbedder)][0]
    calls, seen = [], {}
    inner_emb, inner_cond = emb.forward, m.conditioner.get_unconditional_conditioning

    def record_emb(x):
        state = torch.get_rng_state()
        out = inner_emb(x)
        calls.append((x.clone(), state))
        return out

    def record_cond(*a, **k):
        seen["c"], seen["uc"] = inner_cond(*a, **k)
        return seen["c"], seen["uc"]
    emb.forward, m.conditioner.get_unconditional_conditioning = record_emb, record_cond
    batch = next(iter(DataLoader(SyntheticBEVDataset(1, 4, (64, 128)), batch_size=1)))
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
    torch.manual_seed(0)
    log = m.log_images(batch)
    for k in ("samples", "reconstructions"):
        assert torch.isfinite(log[k]).all() and log[k].shape == (4, 3, 64, 768), k
    assert isinstance(m.first_stage_model._engine.ops, ParityOps) and isinstance(m.first_stage_model._enc_engine.ops, ParityOps)
    alone = _wrapper(m.first_stage_model.ddconfig, "parity", m.first_stage_model.state_dict())
    x, state = calls[0]
    torch.set_rng_state(state)
    want = m.scale_factor * alone.encode(x)
    assert torch.equal(seen["c"]["concat"], want)
