"""Every kernel call of real network runs, checked one by one against an fp64 reference of that call (tests/op_check.py):
the UNet + ControlNet (one epsilon evaluation with its conditioning, small model; first call of each distinct signature
of the full-size model at the benchmarked shape), the VAE decoder and encoder and the text towers, in both precision
modes. One JSON line per (run, precision, op class) is printed (OP_REPLAY ...) and appended to the file PN_OP_REPLAY_LOG
names, if set.

The last test shows that the bounds can fail: the real kernels run on deliberately altered inputs at full-size
signatures, and the checker must reject their output as the output of the unaltered call."""
import pytest
import torch

from op_check import OpCheckError, checked, log_records
from test_eps_parity_gpu import _build, _full_model

pytestmark = pytest.mark.gpu
PRECISIONS = ["bf16", "parity"]


def _ops_cls(precision):
    from panacea_b200.ops import NativeOps, ParityOps
    return ParityOps if precision == "parity" else NativeOps


def _finish(ops, run, precision):
    assert not ops.unchecked, ops.unchecked
    recs = ops.records(run, precision)
    for r in recs:
        r["peak_alloc_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    log_records(recs)
    return recs


def _replay_eps(case, precision, first_only):
    from oracle import cases as Cs
    if case.model_channels == 320:
        w = _full_model(case.num_frames)                # built once, switched between precisions in place
        w.diffusion_model.set_precision(precision)
        w.invalidate()
    else:
        w, _ = _build(case, precision=precision)
    eng = w.diffusion_model.engine()
    ops = checked(type(eng.ops))()
    ops.first_only = first_only
    eng.ops = ops
    x, t, c = Cs.make_inputs(case)
    cg = {k: v.cuda() for k, v in c.items()}
    eps = w(x.cuda(), t.cuda(), cg)                     # prepare_condition (hint stem, text K/V) + one evaluation
    assert torch.isfinite(eps).all()
    ops.first_only = True                               # equal conditioning in new tensors: the fingerprint path
    w(x.cuda(), t.cuda(), {k: v.clone() for k, v in cg.items()})
    assert "fingerprint" in ops.stats
    return ops


@pytest.mark.parametrize("precision", PRECISIONS)
def test_unet_controlnet_every_call(precision):
    from oracle import cases as Cs
    case = [c for c in Cs.GOLDEN_CASES if c.name == "small_hd64"][0]
    ops = _replay_eps(case, precision, first_only=False)
    assert ops.stats["gemm"]["calls"] > 300
    _finish(ops, "unet_controlnet:small_hd64", precision)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_unet_controlnet_full_size_first_call_of_each_signature(precision):
    from oracle import cases as Cs
    case = [c for c in Cs.GOLDEN_CASES if c.name == "full_t8_cfg"][0]
    ops = _replay_eps(case, precision, first_only=True)
    _finish(ops, "unet_controlnet:full_t8_cfg", precision)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("dd_name", ["small", "full_width"])
def test_vae_every_call(dd_name, precision):
    from oracle.make_golden import VAE_DDCONFIG, vae_decoder_input, vae_decoder_weights, vae_encoder_input
    from panacea_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    from tools.make_vae_golden import FULL_WIDTH_DDCONFIG, full_width_inputs
    dd, (z, x) = ((VAE_DDCONFIG, (vae_decoder_input(), vae_encoder_input())) if dd_name == "small"
                  else (FULL_WIDTH_DDCONFIG, full_width_inputs()))
    for Eng, run, inp, seed in ((VAEDecoderEngine, "decode", z, 31), (VAEEncoderEngine, "encode_moments", x, 32)):
        ops = checked(_ops_cls(precision))()
        eng = Eng(dd, ops)
        eng.pack({k: v.cuda() for k, v in vae_decoder_weights(eng.spec, seed=seed).items()})
        assert torch.isfinite(getattr(eng, run)(inp.cuda())).all()
        _finish(ops, f"vae_{run}:{dd_name}", precision)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("case", ["small", "full"])
def test_text_tower_every_call(case, precision):
    from pathlib import Path
    from panacea_b200.text_encoder import TextEncoderEngine
    from tools.make_clip_golden import clip_text_weights
    gd = torch.load(Path(__file__).resolve().parent / "golden" / "clip_text.pt")[case]
    c = gd["config"]
    ops = checked(_ops_cls(precision))()
    eng = TextEncoderEngine(ops)
    eng.pack({k: v.cuda() for k, v in clip_text_weights(c["vocab"], c["width"], c["layers"], c["seed"]).items()})
    assert torch.isfinite(eng.encode(gd["tokens"].cuda(), gd["layer_idx"])).all()
    _finish(ops, f"text:{case}", precision)


# ------------------------------------------------------------------------------------------------ the bounds can fail
def _rejects(ops, name, got, *args, **kw):
    """the checker's verdict on `got` as the output of ops.name(*args, **kw)"""
    probe = checked(type(ops))()
    with pytest.raises(OpCheckError, match="elements out of bound"):
        probe._check(name, 0, "altered input", (name,), got, args, kw, list(args), dict(kw))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_altered_inputs_are_rejected_at_full_size_signatures(precision):
    """Full-size geometry (latent 32 x 336, 16 frames, C = 320 .. 1280) on seeded N(0,1) data: each case runs the real
    kernel on an altered input and hands the result to the checker as the output of the unaltered call."""
    from panacea_b200.netplan import CROSS_VIEW_NEIGHBOURS
    from panacea_b200.ops import geglu_pack
    ops = _ops_cls(precision)()
    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    opnd = lambda x: ops.cast_operand(x.contiguous())

    # conv 3x3 at level 3 (1280 channels, 4 x 42): one 64-wide k-block of the last tap zeroed
    C = 1280
    a = opnd(rn(16, 4, 42, C))
    w = rn(C, 9 * C) * C ** -0.5 / 3
    b = rn(C)
    wp = ops.pack_matrix(w, 9)
    wz = w.clone()
    wz[:, 8 * C + 128:8 * C + 192] = 0
    _rejects(ops, "gemm", ops.gemm(a, ops.pack_matrix(wz, 9), bias=b, taps=(3, 3)), a, wp, bias=b, taps=(3, 3))
    # ... and one bias column shifted by 2^-6 rms
    y = ops.gemm(a, wp, bias=b, taps=(3, 3))
    b2 = b.clone()
    b2[77] += 2.0 ** -6 * y.float().pow(2).mean().sqrt()
    _rejects(ops, "gemm", ops.gemm(a, wp, bias=b2, taps=(3, 3)), a, wp, bias=b, taps=(3, 3))

    # K = 320 linear over the level-0 tokens: a k-block zeroed; bias shifts in the bf16-out and GEGLU epilogues
    C = 320
    a = opnd(rn(16 * 32 * 336 // 4, C))
    w = rn(C, C) * C ** -0.5
    wz = w.clone()
    wz[:, 64:128] = 0
    b = rn(C)
    _rejects(ops, "gemm", ops.gemm(a, ops.pack_matrix(wz), bias=b), a, ops.pack_matrix(w), bias=b)
    out_dt = torch.bfloat16 if precision == "bf16" else torch.float32
    y = ops.gemm(a, ops.pack_matrix(w), bias=b, out_dtype=out_dt)
    b2 = b.clone()
    b2[5] += 2.0 ** -6 * y.float().pow(2).mean().sqrt()
    _rejects(ops, "gemm", ops.gemm(a, ops.pack_matrix(w), bias=b2, out_dtype=out_dt), a, ops.pack_matrix(w), bias=b, out_dtype=out_dt)
    w1, b1 = geglu_pack(rn(8 * C, C) * C ** -0.5), geglu_pack(rn(8 * C))
    gdt = ops.act_dtype
    y = ops.gemm(a, ops.pack_matrix(w1), bias=b1, geglu=True, out_dtype=gdt)
    b2 = b1.clone()
    b2[3] += 2.0 ** -6 * 1.0
    _rejects(ops, "gemm", ops.gemm(a, ops.pack_matrix(w1), bias=b2, geglu=True, out_dtype=gdt), a, ops.pack_matrix(w1), bias=b1,
             geglu=True, out_dtype=gdt)
    if precision == "bf16":
        # the stream producer's row statistics with its two column halves swapped
        xs = rn(a.shape[0], C).to(torch.bfloat16)
        wo = ops.pack_matrix(w)
        yy, st = ops.gemm(a, wo, residual=xs, out_dtype=torch.bfloat16, ln_stats_out=True)
        sw = st.view(st.shape[0], -1, 2, 2).flip(2).reshape(st.shape).contiguous()
        _rejects(ops, "gemm", (yy, sw), a, wo, residual=xs, out_dtype=torch.bfloat16, ln_stats_out=True)

    # attention: the V rows of one key block zeroed (view, text and temporal)
    qdt = ops.qkv_dtype
    C = 320
    qkv = rn(4, 32, 6, 56, 3 * C).to(qdt)
    q2 = qkv.clone()
    q2[:, :2, 1, :, 2 * C:] = 0                       # keys of rows 0-1 of view 1 = one 112-key block
    for cross in (False, True):
        _rejects(ops, "attention_view", ops.attention_view(q2, 5, cross, CROSS_VIEW_NEIGHBOURS), qkv, 5, cross, CROSS_VIEW_NEIGHBOURS)
    q = rn(16, 32 * 336 // 4, C).to(qdt)
    kv = rn(16, 77, 2 * C).to(qdt)
    kv2 = kv.clone()
    kv2[:, 64:77, C:] = 0
    _rejects(ops, "attention_text", ops.attention_text(q, kv2, 5), q, kv, 5)
    qkv = rn(2, 8, 32 * 336 // 4, 3 * C).to(qdt)
    q2 = qkv.clone()
    q2[:, 3, :, 2 * C:] = 0
    _rejects(ops, "attention_temporal", ops.attention_temporal(q2, 5), qkv, 5)

    # norms: one channel's gamma scaled by 1 + 2^-6
    x = rn(16, 32, 336, 320) * 2 + 0.5
    gm, bt = 1 + 0.1 * rn(320), 0.1 * rn(320)
    gm2 = gm.clone()
    gm2[17] *= 1 + 2.0 ** -6
    _rejects(ops, "groupnorm", ops.groupnorm(x, gm2, bt, 1e-5, True), x, gm, bt, 1e-5, True)
    xp = x.view(2, 8, 32 * 336, 320)
    _rejects(ops, "groupnorm_pixel", ops.groupnorm_pixel(xp, gm2, bt, 1e-5, True), xp, gm, bt, 1e-5, True)
    xl = x.view(-1, 320)[:200000].contiguous()
    _rejects(ops, "layernorm", ops.layernorm(xl, gm2, bt), xl, gm, bt)
