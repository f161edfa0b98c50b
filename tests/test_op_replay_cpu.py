"""The per-call replay checker (tests/op_check.py) on the CPU: the fp32 torch emulations of both precision modes pass it
call by call on real engine runs with complete coverage, and op sets with one planted defect each are rejected with the
defective op and its engine call site named."""
import pytest
import torch
import torch.nn.functional as F

from oracle import cases as Cs
from op_check import CHECKED, EXCLUDED, OpCheckError, checked
from panacea_b200 import engine as E
from panacea_b200 import netplan as NP
from torch_ref_ops import TorchFoldOps, TorchRefOps, TorchRefOps64, TorchSplitOps


def _split(sd):
    up = {k[len("diffusion_model."):]: v for k, v in sd.items() if not k.startswith("diffusion_model.controlnet.")}
    cp = {k[len("diffusion_model.controlnet."):]: v for k, v in sd.items() if k.startswith("diffusion_model.controlnet.")}
    return up, cp


def _eps_run(ops, name="tiny_3to1"):
    case = [c for c in Cs.GOLDEN_CASES if c.name == name][0]
    eng = E.Engine(NP.config_from_kwargs(case.unet_kwargs()), ops)
    eng.pack(*_split(Cs.make_weights(case)))
    x, t, c = Cs.make_inputs(case)
    eng.prepare_condition(c["cond_feat"], c["crossattn"])
    return eng.eps(x, c["concat"], t)


def _text_run(ops):
    """the small text tower of tests/golden/clip_text.pt on its golden tokens"""
    from pathlib import Path
    from panacea_b200.text_encoder import TextEncoderEngine
    from tools.make_clip_golden import clip_text_weights
    g = torch.load(Path(__file__).resolve().parent / "golden" / "clip_text.pt")["small"]
    c = g["config"]
    eng = TextEncoderEngine(ops)
    eng.pack({k: v.to(g["tokens"].device) for k, v in clip_text_weights(c["vocab"], c["width"], c["layers"], c["seed"]).items()})
    return eng.encode(g["tokens"], g["layer_idx"])


def test_every_public_op_is_checked_or_excluded():
    from panacea_b200.ops import NativeOps, ParityOps
    for cls in (NativeOps, ParityOps):
        public = {n for n in dir(cls) if not n.startswith("_") and callable(getattr(cls, n))}
        assert public - set(CHECKED) - set(EXCLUDED) == set(), cls
    assert not set(CHECKED) & set(EXCLUDED)


def test_an_op_without_a_checker_is_refused():
    class WithNewKernel(TorchFoldOps):
        def new_kernel(self, x):
            return x
    ops = checked(WithNewKernel)()
    with pytest.raises(OpCheckError, match="new_kernel"):
        ops.new_kernel(torch.zeros(4))


def test_fp64_reference_matches_fp32_reference():
    """TorchRefOps64 is TorchRefOps in fp64 (before store rounding): same semantics, to fp32 accuracy."""
    g = torch.Generator().manual_seed(3)
    a = torch.randn(2, 4, 6, 64, generator=g)
    w = torch.randn(160, 9 * 64, generator=g)
    b = torch.randn(160, generator=g)
    y32, s32 = TorchRefOps().gemm(a, w, bias=b, taps=(3, 3), ln_stats_out=True)
    y64, s64 = TorchRefOps64().gemm(a, w, bias=b, taps=(3, 3), ln_stats_out=True)
    assert y64.dtype == torch.float64 and s64.shape == s32.shape == (48, 2, 2)
    assert torch.allclose(y64.float(), y32, rtol=1e-5, atol=1e-3) and torch.allclose(s64.float(), s32, rtol=1e-4)
    assert torch.allclose(s64[:, 0, 0], y64.reshape(48, 160)[:, :80].sum(1))       # part 0: the first 80 columns


@pytest.mark.parametrize("name", ["tiny_3to1", "small_hd64"])
@pytest.mark.parametrize("base", [TorchFoldOps, TorchSplitOps], ids=["fold", "split"])
def test_clean_emulation_passes_every_call(name, base):
    ops = checked(base)()
    eps = _eps_run(ops, name)
    assert torch.isfinite(eps).all() and not ops.unchecked
    seen = set(ops.stats)
    assert {"gemm", "groupnorm", "groupnorm_pixel", "attention_view", "attention_text", "attention_temporal", "linear_small",
            "conv3x3_direct", "im2col_s2", "upsample2x", "concat_add", "add_", "nchw_to_nhwc", "nhwc_to_nchw",
            "timestep_embedding", "cast_operand"} <= seen
    assert all(st["worst_ratio"] <= 1.0 for st in ops.stats.values())


@pytest.mark.parametrize("parity", [False, True])
def test_clean_vae_and_text_emulations_pass(parity):
    from oracle.make_golden import VAE_DDCONFIG, vae_decoder_input, vae_decoder_weights, vae_encoder_input
    from panacea_b200.text_encoder import TextEncoderEngine
    from panacea_b200.vae import VAEDecoderEngine, VAEEncoderEngine
    base = TorchSplitOps if parity else TorchRefOps
    for Eng, run, inp in ((VAEDecoderEngine, "decode", vae_decoder_input()), (VAEEncoderEngine, "encode_moments", vae_encoder_input())):
        ops = checked(base)()
        eng = Eng(VAE_DDCONFIG, ops)
        eng.pack(vae_decoder_weights(eng.spec))
        assert torch.isfinite(getattr(eng, run)(inp)).all()
        assert "gemm" in ops.stats and "groupnorm" in ops.stats
    ops = checked(base)()
    _text_run(ops)
    assert {"token_embedding", "layernorm", "attention_causal", "gelu_operand", "gemm"} <= set(ops.stats)


# ------------------------------------------------------------------------------------------------ planted defects
class _Once:
    """fire a defect on the `at`-th call of one op (0-based) whose arguments satisfy `when`"""
    at = 0

    def _fire(self, name, ok=True):
        n = self.__dict__.setdefault("_n", {})
        if not ok:
            return False
        n[name] = n.get(name, -1) + 1
        return n[name] == self.at


class SkipKBlock(_Once, TorchFoldOps):
    def gemm(self, a, w, **kw):
        if self._fire("gemm", w.shape[1] >= 256):
            w = w.clone()
            w[:, 128:192] = 0                       # the third 64-wide k-block is never accumulated
        return super().gemm(a, w, **kw)


class ShiftedTap(_Once, TorchFoldOps):
    def gemm(self, a, w, *, taps=(1, 1), **kw):
        if self._fire("gemm", taps == (3, 3)):
            C = a.shape[-1]
            y = super().gemm(a, w, taps=taps, **{**kw, "out": None, "ln_stats_out": False})
            # tap (2, 2) read one pixel too far to the right
            a2 = torch.roll(a, -1, dims=2) - a
            extra = super().gemm(F.pad(a2, (0, 0, 0, 0, 0, 0)).contiguous(), torch.cat(
                [torch.zeros_like(w[:, :8 * C]), w[:, 8 * C:]], 1), taps=taps)
            y = y + extra
            if kw.get("out") is not None:
                kw["out"].copy_(y.reshape(kw["out"].shape))
                return kw["out"]
            return y
        return super().gemm(a, w, taps=taps, **kw)


class RowvecOffByOne(_Once, TorchFoldOps):
    def gemm(self, a, w, *, rowvec=None, rows_per_group=0, n_groups=0, **kw):
        if self._fire("gemm", rowvec is not None and not torch.equal(rowvec[0], rowvec[1])):
            rowvec = torch.roll(rowvec, 1, dims=0)   # group g gets the vector of group g - 1
        return super().gemm(a, w, rowvec=rowvec, rows_per_group=rows_per_group, n_groups=n_groups, **kw)


class SwappedQueryRows(_Once, TorchFoldOps):
    def attention_view(self, qkv, heads, cross, neighbours):
        out = super().attention_view(qkv, heads, cross, neighbours)
        if self._fire("attention_view", cross):
            out = out.clone()
            out[0, 0, 0, [0, 1]] = out[0, 0, 0, [1, 0]]
        return out


class WideChannelWrite(_Once, TorchFoldOps):
    def nchw_to_nhwc(self, x, out=None, ch_off=0):
        r = super().nchw_to_nhwc(x, out=out, ch_off=ch_off)
        if self._fire("nchw_to_nhwc", out is not None and out.shape[-1] > ch_off + x.shape[1]):
            out[..., ch_off + x.shape[1]] = 1.0      # one channel past the slice
        return r


class ModifiesInput(_Once, TorchFoldOps):
    def groupnorm(self, x, *a, **k):
        r = super().groupnorm(x, *a, **k)
        if self._fire("groupnorm"):
            x.view(-1)[7] += 1.0
        return r


@pytest.mark.parametrize("mutant,op,site", [
    (SkipKBlock, "gemm", "engine.py"),
    (ShiftedTap, "gemm", "_run_block [input_blocks.0.0]"),
    (RowvecOffByOne, "gemm", "_stt"),
    (SwappedQueryRows, "attention_view", "_transformer"),
    (WideChannelWrite, "nchw_to_nhwc", "prepare_hint"),
    (ModifiesInput, "groupnorm", "_res"),
], ids=["skip_k_block", "shifted_tap", "rowvec_off_by_one", "swapped_query_rows", "write_outside_channel_slice",
        "modifies_input"])
def test_planted_defect_is_rejected_with_op_and_site(mutant, op, site):
    ops = checked(mutant)()
    with pytest.raises(OpCheckError) as e:
        _eps_run(ops, "small_hd64")
    msg = str(e.value)
    assert msg.startswith(f"{op} call #") and site in msg, msg
