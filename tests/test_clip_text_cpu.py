"""OpenCLIP text encoder, host side: the CLIP BPE tokenizer rules, TextEncoderEngine's orchestration against the
UNMODIFIED reference `FrozenOpenCLIPEmbedder` (tests/golden/clip_text.pt, made by tools/make_clip_golden.py), the
embedder's weight loading, and list-index overrides in load_config."""
import gzip
from pathlib import Path

import pytest
import torch

from tools.make_clip_golden import CASES, clip_text_weights, golden_subset

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
PREFIX = "conditioner.embedders.0.model."
# a tiny merges file: "the" and "and" become single symbols, everything else falls back to byte symbols
TINY_MERGES = ["#version: 0.2", "t h", "th e</w>", "a n", "an d</w>"]
NUSCENES_CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
                    "pedestrian", "traffic_cone"]


def write_tiny_vocab(dirpath: Path) -> Path:
    p = Path(dirpath) / "tiny_bpe.txt.gz"
    with gzip.open(p, "wt", encoding="utf-8") as f:
        f.write("\n".join(TINY_MERGES) + "\n")
    return p


def byte_id(ch: str, end: bool = False) -> int:
    from panacea_b200.clip_tokenizer import bytes_to_unicode
    return list(bytes_to_unicode().values()).index(ch) + (256 if end else 0)


@pytest.fixture()
def tok(tmp_path):
    from panacea_b200.clip_tokenizer import ClipTokenizer
    return ClipTokenizer(write_tiny_vocab(tmp_path))


def test_tokenizer_vocabulary_and_special_ids(tok):
    assert tok.vocab_size == 512 + 4 + 2
    assert (tok.sot, tok.eot) == (tok.vocab_size - 2, tok.vocab_size - 1)


def test_tokenizer_merges_and_end_of_word(tok):
    the, and_ = 512 + 1, 512 + 3                                  # "th e</w>" and "an d</w>" are merges 1 and 3
    assert tok.encode("the and") == [the, and_]
    # inside one word "e" does not end it, so "th e</w>" cannot apply; "an d</w>" can, at the word's end
    assert tok.encode("theand") == [512 + 0, byte_id("e"), and_]
    assert tok.encode("th") == [byte_id("t"), byte_id("h", True)]        # "t h" only merges inside a word: "h</w>" ends it


def test_tokenizer_byte_fallback_and_punctuation(tok):
    assert tok.encode("x") == [byte_id("x", True)]
    assert tok.encode("zq") == [byte_id("z"), byte_id("q", True)]
    assert tok.encode("a,b") == [byte_id("a", True), byte_id(",", True), byte_id("b", True)]
    assert tok.encode("7") == [byte_id("7", True)]


def test_tokenizer_lowercase_and_whitespace(tok):
    assert tok.encode("  THE \n\t And  ") == tok.encode("the and")
    assert tok.encode("&amp;") == tok.encode("&")                  # html.unescape


def test_tokenizer_padding_truncation_and_empty(tok):
    t = tok.tokenize(["the and", "", "the " * 100])
    assert t.dtype == torch.int64 and t.shape == (3, 77)
    assert t[0, :4].tolist() == [tok.sot, 513, 515, tok.eot] and t[0, 4:].abs().sum() == 0
    assert t[1, :2].tolist() == [tok.sot, tok.eot] and t[1, 2:].abs().sum() == 0
    assert t[2, 0] == tok.sot and t[2, 76] == tok.eot and (t[2, 1:76] == 513).all()


def test_tokenizer_rejects_non_ascii_without_ftfy(tok):
    try:
        import ftfy  # noqa: F401
        pytest.skip("ftfy is installed: non-ASCII text is cleaned by it")
    except ImportError:
        pass
    with pytest.raises(NotImplementedError, match="ftfy"):
        tok.encode("café")


def test_missing_vocabulary_names_both_sources(tmp_path):
    from panacea_b200.clip_tokenizer import find_bpe_path
    with pytest.raises(FileNotFoundError):
        find_bpe_path(tmp_path / "nope.txt.gz")
    try:
        find_bpe_path()
    except FileNotFoundError as e:
        assert "bpe_path" in str(e) and "open_clip" in str(e)


def test_real_vocabulary_matches_open_clip():
    from panacea_b200.clip_tokenizer import ClipTokenizer, find_bpe_path
    try:
        find_bpe_path()
    except FileNotFoundError:
        pytest.skip("no CLIP BPE vocabulary available (open_clip not installed)")
    tok = ClipTokenizer()
    assert tok.vocab_size == 49408 and (tok.sot, tok.eot) == (49406, 49407)
    open_clip = pytest.importorskip("open_clip")
    g = torch.Generator().manual_seed(0)
    prompts = []
    for tmpl in torch.load(GOLDEN / "clip_text.pt")["prompt_templates"]:
        for n in (3, 40):
            objs = [NUSCENES_CLASSES[i] for i in torch.randint(0, len(NUSCENES_CLASSES), (n,), generator=g).tolist()]
            prompts.append(tmpl.format(str(n)) + ", ".join(objs))
    ours = tok.tokenize(prompts)
    assert (ours[:, -1] == 49407).any()                          # the long lists are truncated
    assert torch.equal(ours, open_clip.tokenize(prompts))


# ------------------------------------------------------------------ engine orchestration
def test_engine_orchestration_matches_the_reference_on_cpu():
    from torch_ref_ops import TorchRefOps
    from panacea_b200.text_encoder import TextEncoderEngine, text_param_spec
    g = torch.load(GOLDEN / "clip_text.pt")["small"]
    c = g["config"]
    P = clip_text_weights(c["vocab"], c["width"], c["layers"], c["seed"])
    spec = text_param_spec(c["vocab"], g["ctx"], c["width"], c["layers"])
    assert sorted(spec) == sorted(set(g["keys"]) - {"text_projection", "logit_scale"})
    eng = TextEncoderEngine(TorchRefOps())
    eng.pack(P)
    assert eng.heads == c["heads"]
    out = eng.encode(g["tokens"], g["layer_idx"])
    assert tuple(out.shape) == g["out_shape"] and g["out_stride"] == 1
    assert (golden_subset(out, 1) - g["out"]).abs().max().item() < 5e-5


def test_engine_rejects_bad_head_dim_and_out_of_range_tokens():
    from torch_ref_ops import TorchRefOps
    from panacea_b200.text_encoder import TextEncoderEngine
    eng = TextEncoderEngine(TorchRefOps())
    with pytest.raises(NotImplementedError, match="head_dim"):
        eng.pack(clip_text_weights(50, 96, 1, 0))
    eng.pack(clip_text_weights(50, 64, 2, 0))
    with pytest.raises(ValueError):
        eng.encode(torch.full((1, 77), 50, dtype=torch.int64), 0)


def test_full_size_spec_is_the_vit_h_14_text_tower():
    from panacea_b200.text_encoder import text_param_spec
    spec = text_param_spec(49408, 77, 1024, 24)
    n = sum(int(torch.tensor(s).prod()) for s in spec.values())
    assert sorted(spec) == sorted(set(torch.load(GOLDEN / "clip_text.pt")["full"]["keys"]) - {"text_projection", "logit_scale"})
    assert 352_900_000 < n < 353_100_000         # + text_projection (1024^2) and logit_scale: open_clip's 354 M


# ------------------------------------------------------------------ embedder
def _small_sd(vocab=1000):
    return clip_text_weights(vocab, 128, 3, CASES["small"]["seed"])


def _engine_model():
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.util import instantiate_from_config
    return instantiate_from_config(load_config([CFG])["model"])


def _stand_in(s, dim):
    import hashlib
    seed = int.from_bytes(hashlib.sha256(str(s).encode()).digest()[:8], "little") % (2 ** 63)
    return torch.randn(77, dim, generator=torch.Generator().manual_seed(seed))


def test_embedder_without_weights_is_the_unchanged_stand_in():
    from panacea_b200.sgm.modules.encoders.modules import FrozenOpenCLIPEmbedder
    e = FrozenOpenCLIPEmbedder(context_dim=128)
    out = e(["a driving scene", ""])
    assert not e.has_tower and e.state_dict() == {}
    assert torch.equal(out, torch.stack([_stand_in("a driving scene", 128), _stand_in("", 128)]))


def test_checkpoint_keys_activate_the_tower_and_round_trip():
    m = _engine_model()
    emb = m.conditioner.embedders[0]
    sd = {PREFIX + k: v for k, v in _small_sd().items()}
    res = m.load_state_dict(sd, strict=False)
    assert emb.has_tower and not [k for k in res.missing_keys if k.startswith(PREFIX)]
    out = m.state_dict()
    assert all(torch.equal(out[k], v) for k, v in sd.items())
    with pytest.raises(RuntimeError, match="no CPU path"):
        emb(["a driving scene"])
    with pytest.raises(RuntimeError, match="no CPU path"):
        emb(torch.zeros(1, 77, dtype=torch.int64))


def test_partial_tower_keys_raise():
    m = _engine_model()
    sd = {PREFIX + k: v for k, v in _small_sd().items() if k != "transformer.resblocks.1.mlp.c_fc.bias"}
    with pytest.raises(RuntimeError, match=r"transformer\.resblocks\.1\.mlp\.c_fc\.bias"):
        m.load_state_dict(sd, strict=False)
    assert not m.conditioner.embedders[0].has_tower


def test_tower_width_must_match_context_dim():
    from panacea_b200.sgm.modules.encoders.modules import FrozenOpenCLIPEmbedder
    e = FrozenOpenCLIPEmbedder(context_dim=1024)
    with pytest.raises(RuntimeError, match="context_dim"):
        e.load_state_dict({"model." + k: v for k, v in _small_sd().items()})


@pytest.mark.parametrize("suffix", [".pt", ".safetensors"])
def test_version_file_loads_a_stock_open_clip_file(tmp_path, suffix):
    from panacea_b200.sgm.modules.encoders.modules import FrozenOpenCLIPEmbedder
    sd = _small_sd()
    stock = {**sd, "visual.conv1.weight": torch.zeros(4, 3, 2, 2), "visual.proj": torch.zeros(4, 4)}
    path = tmp_path / ("open_clip_pytorch_model" + suffix)
    if suffix == ".safetensors":
        from safetensors.torch import save_file
        save_file(stock, str(path))
    else:
        torch.save(stock, path)
    e = FrozenOpenCLIPEmbedder(version=str(path), context_dim=128, layer="last")
    assert e.has_tower and sorted(e.state_dict()) == sorted("model." + k for k in sd)
    assert FrozenOpenCLIPEmbedder(context_dim=128).has_tower is False         # a pretrained tag loads nothing
    with pytest.raises(FileNotFoundError):
        FrozenOpenCLIPEmbedder(version=str(tmp_path / "missing.bin"), context_dim=128)


def test_load_config_list_index_override(tmp_path):
    from panacea_b200.inference import load_config
    key = "model.params.conditioner_config.params.emb_models.0.params.bpe_path"
    cfg = load_config([CFG], [f"{key}={tmp_path / 'v.txt.gz'}"])
    emb = cfg["model"]["params"]["conditioner_config"]["params"]["emb_models"]
    assert emb[0]["params"]["bpe_path"] == str(tmp_path / "v.txt.gz") and emb[0]["params"]["context_dim"] == 128
    assert len(emb) == 3 and "params" not in emb[1]
    with pytest.raises(KeyError):
        load_config([CFG], ["model.params.conditioner_config.params.emb_models.7.params.x=1"])
