"""OpenCLIP text encoder on the GPU: the new kernels (pn_attention_causal in bf16 and fp32, pn_gelu_operand,
pn_token_embedding) against torch, the whole tower in both precision modes against the UNMODIFIED reference
(tests/golden/clip_text.pt), and the embedder inside the inference engine on tests/configs/tiny_inference.yaml."""
import time
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from op_check import _decode
from tools.make_clip_golden import clip_text_weights, golden_subset

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
BF16 = torch.bfloat16
# bf16 mode against the fp32 golden, for these seeded random weights. Measured on an H100 80GB HBM3 (700 W limit):
# full rel-L2 5.99e-3 / max abs 2.59e-2 on the stored elements, small 5.80e-3 / 2.61e-2 (outputs have rms 1.0); the bounds are twice that.
# Real CLIP activations have outlier channels, so they are not a claim about the released weights.
BF16_BOUND = {"full": (1.2e-2, 6e-2), "small": (1.2e-2, 6e-2)}     # (rel-L2, max abs)


def _causal_ref(qkv, heads):
    b, L, C3 = qkv.shape
    C = C3 // 3
    q, k, v = (t.reshape(b, L, heads, C // heads).transpose(1, 2) for t in qkv.float().split(C, dim=-1))
    return F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(b, L, C)


@pytest.mark.parametrize("L", [1, 16, 77, 128])
@pytest.mark.parametrize("b", [1, 3])
def test_attention_causal_kernel(L, b):
    from panacea_b200.ops import NativeOps
    g = torch.Generator().manual_seed(L * 10 + b)
    qkv = (torch.randn(b, L, 3 * 1024, generator=g) * 2).to(BF16)
    out = NativeOps().attention_causal(qkv.cuda(), 16).float().cpu()
    ref = _causal_ref(qkv, 16)
    rel = ((out - ref).norm() / ref.norm()).item()
    assert out.shape == (b, L, 1024) and rel < 1e-2, rel                 # bf16 P and output (attention tests: < 2e-2)


@pytest.mark.parametrize("L", [1, 16, 77, 128])
@pytest.mark.parametrize("b", [1, 3])
def test_attention_causal_f32_kernel(L, b):
    from panacea_b200.ops import ParityOps
    g = torch.Generator().manual_seed(L * 10 + b + 1)
    qkv = torch.randn(b, L, 3 * 1024, generator=g) * 2
    out = ParityOps().attention_causal(qkv.cuda(), 16).cpu()             # split3 operand [hi | lo | hi]
    dec = _decode(out, "split3")
    ref = _causal_ref(qkv.double(), 16).float()
    rel = ((dec - ref).norm() / ref.norm()).item()
    assert rel <= 1e-5, rel


def test_attention_causal_rejects_bad_shapes():
    from panacea_b200.ops import NativeOps
    with pytest.raises(ValueError):
        NativeOps().attention_causal(torch.zeros(1, 129, 3 * 128, device="cuda", dtype=BF16), 2)
    with pytest.raises(ValueError):
        NativeOps().attention_causal(torch.zeros(1, 77, 3 * 160, device="cuda", dtype=BF16), 2)   # head_dim 80


def test_gelu_operand_kernel_in_each_mode():
    import ctypes
    from panacea_b200 import _lib
    from panacea_b200.ops import OP_F32, NativeOps, ParityOps
    x = torch.randn(77, 4096, generator=torch.Generator().manual_seed(5)) * 3
    ref = F.gelu(x.double()).float()
    yb = NativeOps().gelu_operand(x.cuda()).cpu()
    assert yb.dtype == BF16 and (yb.float() - ref).abs().max().item() <= 2 ** -8 * ref.abs().max().item()
    ys = ParityOps().gelu_operand(x.cuda()).cpu()
    assert ys.shape == (77, 3 * 4096) and torch.equal(ys[:, :4096], ys[:, 8192:])
    # hi + lo keeps 16 significant bits of the fp32 value: |error| <= 2^-17 |v| plus erff's last bits
    assert (((ys[:, :4096].float() + ys[:, 4096:8192].float()) - ref).abs() <= 2 ** -17 * ref.abs() + 2e-6).all()
    ops = NativeOps()
    xc, yf = x.cuda(), torch.empty(77, 4096, device="cuda")
    _lib.check(ops.lib.pn_gelu_operand(ctypes.c_void_p(xc.data_ptr()), ctypes.c_void_p(yf.data_ptr()), 77, 4096, OP_F32,
                                       ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pn_gelu_operand")
    assert (yf.cpu() - ref).abs().max().item() < 2e-6


def test_token_embedding_kernel_is_exact():
    from panacea_b200.ops import NativeOps
    g = torch.Generator().manual_seed(6)
    table, pos = torch.randn(49408, 1024, generator=g), torch.randn(77, 1024, generator=g)
    tok = torch.randint(0, 49408, (3, 77), generator=g)
    tok[:, 0], tok[0, -1] = 0, 49407
    ops = NativeOps()
    out = ops.token_embedding(tok.cuda(), table.cuda(), pos.cuda()).cpu()
    assert torch.equal(out, table[tok] + pos)
    for bad in (49408, -1):
        t2 = tok.clone()
        t2[1, 5] = bad
        with pytest.raises(ValueError, match="token ids"):
            ops.token_embedding(t2.cuda(), table.cuda(), pos.cuda())


@pytest.mark.parametrize("case", ["small", "full"])
@pytest.mark.parametrize("precision", ["parity", "bf16"])
def test_tower_matches_the_reference(case, precision):
    from panacea_b200.ops import NativeOps, ParityOps
    from panacea_b200.text_encoder import TextEncoderEngine
    gd = torch.load(GOLDEN / "clip_text.pt")[case]
    c = gd["config"]
    P = {k: v.cuda() for k, v in clip_text_weights(c["vocab"], c["width"], c["layers"], c["seed"]).items()}
    eng = TextEncoderEngine(ParityOps() if precision == "parity" else NativeOps())
    eng.pack(P)
    tokens = gd["tokens"].cuda()
    out = eng.encode(tokens, gd["layer_idx"])
    torch.cuda.synchronize()
    if case == "full":                                              # one CFG pair per sample: the prompt and ""
        for _ in range(3):
            eng.encode(tokens[:1], gd["layer_idx"])
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        n = 20
        ev[0].record()
        for _ in range(n):
            eng.encode(tokens[:1], gd["layer_idx"])
            eng.encode(tokens[1:2], gd["layer_idx"])
        ev[1].record()
        torch.cuda.synchronize()
        print(f"TIMING clip_text_{case}_{precision} {ev[0].elapsed_time(ev[1]) / n:.3f} ms per sample (2 calls of batch 1) "
              f"on {torch.cuda.get_device_name()}")
    assert tuple(out.shape) == gd["out_shape"] and torch.isfinite(out).all()
    out = golden_subset(out, gd["out_stride"])
    ref = gd["out"]
    rel = ((out - ref).norm() / ref.norm()).item()
    mx = (out - ref).abs().max().item()
    frac = ((out - ref).abs() <= 1e-4 + 1e-3 * ref.abs()).float().mean().item()
    print(f"PARITY clip_text_{case}_{precision} rel_l2 {rel:.3e} max_abs {mx:.3e} within_tol {frac * 100:.3f} %")
    if precision == "parity":
        assert frac >= 0.999, frac
    else:
        assert rel < BF16_BOUND[case][0] and mx < BF16_BOUND[case][1], (rel, mx)


def test_embedder_feeds_the_tower_output_to_the_engine(tmp_path):
    """tiny_inference.yaml (context_dim 128, penultimate): bpe_path through a list-index override, seeded small-tower
    weights through load_state_dict; log_images runs and its c / uc crossattn are the tower's encodings."""
    from torch.utils.data import DataLoader
    from test_clip_text_cpu import PREFIX, write_tiny_vocab
    from panacea_b200.clip_tokenizer import ClipTokenizer
    from panacea_b200.inference import SyntheticBEVDataset, load_config
    from panacea_b200.ops import NativeOps
    from panacea_b200.sgm.util import instantiate_from_config
    from panacea_b200.text_encoder import TextEncoderEngine
    vocab = write_tiny_vocab(tmp_path)
    key = "model.params.conditioner_config.params.emb_models.0.params.bpe_path"
    m = instantiate_from_config(load_config([CFG], [f"{key}={vocab}"])["model"])
    tok = ClipTokenizer(vocab)
    P = clip_text_weights(tok.vocab_size, 128, 3, seed=21)
    m.load_state_dict({PREFIX + k: v for k, v in P.items()}, strict=False)
    m = m.cuda().eval()
    seen = {}
    inner = m.conditioner.get_unconditional_conditioning

    def record(*a, **k):
        seen["c"], seen["uc"] = inner(*a, **k)
        return seen["c"], seen["uc"]
    m.conditioner.get_unconditional_conditioning = record
    batch = next(iter(DataLoader(SyntheticBEVDataset(1, 4, (64, 128)), batch_size=1)))
    batch = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
    torch.manual_seed(0)
    log = m.log_images(batch)
    assert torch.isfinite(log["samples"]).all()
    eng = TextEncoderEngine(NativeOps())
    eng.pack({k: v.cuda() for k, v in P.items()})
    want_c = eng.encode(tok.tokenize(batch["txt"]).cuda(), 1)
    want_uc = eng.encode(tok.tokenize([""]).cuda(), 1)
    assert torch.equal(seen["c"]["crossattn"], want_c) and torch.equal(seen["uc"]["crossattn"], want_uc)
    emb = m.conditioner.embedders[0]
    assert not torch.equal(want_c, emb._stand_in(batch["txt"]))
