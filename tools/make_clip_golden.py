"""TEST INFRASTRUCTURE — golden outputs of the reference's `FrozenOpenCLIPEmbedder` text tower
(sgm/modules/encoders/modules.py:559-632), run UNMODIFIED on seeded weights. Writes tests/golden/clip_text.pt:

  full    the ViT-H-14 text tower (vocab 49408, width 1024, 24 blocks, 16 heads), layer "penultimate", over three
          token rows: a normal prompt, the unconditional "" and a row truncated to 77 that ends in <end_of_text>;
  small   vocab 1000, width 128, 3 blocks, 2 heads, layer "last" (CPU tests);
  prompt_templates   the Panacea prompt templates of the reference's nuScenes dataset (nuscenes_datasets_video.py:91),
          for the tokenizer test against open_clip.tokenize.

Each case stores its token rows, config, layer, the sorted state-dict key list of the embedder's model and the fp32
output: whole for the small tower; for the full tower every OUT_STRIDE-th element of the flattened [3, 77, 1024] output
(every other channel of every position), which keeps the file under 0.6 MB; all 77 positions and every block still
feed the stored values, and LayerNorm statistics and the next block's GEMMs mix every channel. `golden_subset` selects
the same elements from a computed output. The weights are re-derived from seeds by `clip_text_weights`, which tests
import.

open_clip is not installed and the reference only imports it, so `create_model_and_transforms` is given a stand-in
for the duration of the run: open_clip's published text-tower architecture restated with plain torch.nn
(nn.Embedding, positional_embedding, resblocks of ln_1 / nn.MultiheadAttention in LND layout / ln_2 /
mlp = Sequential(c_fc, GELU, c_proj), the -inf upper-triangular attn_mask, ln_final, text_projection). Its module
names follow open_clip's, so the golden key list pins the names the loader must accept.

Run where the reference tree is available:  python -m tools.make_clip_golden [--only full,small]
"""
from __future__ import annotations

import argparse
import ast
import sys
from collections import OrderedDict
from pathlib import Path

import torch
import torch.nn as nn

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
CTX = 77
CASES = {
    "full": {"arch": "ViT-H-14", "vocab": 49408, "width": 1024, "layers": 24, "heads": 16, "layer": "penultimate", "seed": 11},
    "small": {"arch": "pn-text-small", "vocab": 1000, "width": 128, "layers": 3, "heads": 2, "layer": "last", "seed": 12},
}
OUT_STRIDE = {"full": 2, "small": 1}


def golden_subset(out: torch.Tensor, stride: int) -> torch.Tensor:
    """The elements of an encoder output [b, 77, width] that a golden case stores: every stride-th of the flattened
    tensor, on the CPU in fp32."""
    return out.detach().float().cpu().reshape(-1)[::stride].contiguous()


def clip_text_weights(vocab: int, width: int, layers: int, seed: int, ctx: int = CTX) -> dict:
    """Seeded parameters of an open_clip text tower under its state-dict names: token / positional embeddings
    N(0, 0.02) / N(0, 0.01), linear weights and biases N(0, 1/fan_in), LayerNorm gamma = 1 + 0.1 N(0,1) and
    beta = 0.05 N(0,1). Also text_projection and logit_scale, which the embedder does not use."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    P = {"token_embedding.weight": rn(vocab, width) * 0.02, "positional_embedding": rn(ctx, width) * 0.01}
    lin = lambda n, k: (rn(n, k) * k ** -0.5, rn(n) * k ** -0.5)
    ln = lambda: (1 + 0.1 * rn(width), 0.05 * rn(width))
    for i in range(layers):
        k = f"transformer.resblocks.{i}."
        P[k + "ln_1.weight"], P[k + "ln_1.bias"] = ln()
        P[k + "attn.in_proj_weight"], P[k + "attn.in_proj_bias"] = lin(3 * width, width)
        P[k + "attn.out_proj.weight"], P[k + "attn.out_proj.bias"] = lin(width, width)
        P[k + "ln_2.weight"], P[k + "ln_2.bias"] = ln()
        P[k + "mlp.c_fc.weight"], P[k + "mlp.c_fc.bias"] = lin(4 * width, width)
        P[k + "mlp.c_proj.weight"], P[k + "mlp.c_proj.bias"] = lin(width, 4 * width)
    P["ln_final.weight"], P["ln_final.bias"] = ln()
    P["text_projection"] = rn(width, width) * width ** -0.5
    P["logit_scale"] = torch.tensor(4.6052)
    return P


def clip_text_tokens(case: str) -> torch.Tensor:
    """The token rows of a case: [sot, ids, eot, 0...]; [sot, eot, 0...]; a truncated row ending in eot (full only)."""
    c = CASES[case]
    sot, eot = c["vocab"] - 2, c["vocab"] - 1
    g = torch.Generator().manual_seed(c["seed"] + 100)
    ids = lambda n: torch.randint(1, sot, (n,), generator=g).tolist()
    rows = [[sot] + ids(21) + [eot], [sot, eot]]
    if case == "full":
        rows.append(([sot] + ids(120))[:CTX - 1] + [eot])
    out = torch.zeros(len(rows), CTX, dtype=torch.int64)
    for r, row in enumerate(rows):
        out[r, :len(row)] = torch.tensor(row)
    return out


# ------------------------------------------------------------------ open_clip stand-in (published architecture)
class _ResidualAttentionBlock(nn.Module):
    def __init__(self, width, heads):
        super().__init__()
        self.ln_1 = nn.LayerNorm(width)
        self.attn = nn.MultiheadAttention(width, heads)
        self.ln_2 = nn.LayerNorm(width)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(width, 4 * width)), ("gelu", nn.GELU()),
                                              ("c_proj", nn.Linear(4 * width, width))]))

    def forward(self, x, attn_mask=None):
        y = self.ln_1(x)
        x = x + self.attn(y, y, y, need_weights=False, attn_mask=attn_mask)[0]
        return x + self.mlp(self.ln_2(x))


class _Transformer(nn.Module):
    def __init__(self, width, layers, heads):
        super().__init__()
        self.grad_checkpointing = False
        self.resblocks = nn.ModuleList([_ResidualAttentionBlock(width, heads) for _ in range(layers)])


class _TextCLIP(nn.Module):
    def __init__(self, vocab, width, layers, heads, ctx=CTX):
        super().__init__()
        self.visual = nn.Identity()
        self.transformer = _Transformer(width, layers, heads)
        self.token_embedding = nn.Embedding(vocab, width)
        self.positional_embedding = nn.Parameter(torch.empty(ctx, width))
        self.ln_final = nn.LayerNorm(width)
        self.text_projection = nn.Parameter(torch.empty(width, width))
        self.logit_scale = nn.Parameter(torch.ones([]))
        self.register_buffer("attn_mask", torch.full((ctx, ctx), float("-inf")).triu_(1), persistent=False)


def _create_model_and_transforms(arch, device=None, pretrained=None, cache_dir=None, **kw):
    c = [c for c in CASES.values() if c["arch"] == arch][0]
    m = _TextCLIP(c["vocab"], c["width"], c["layers"], c["heads"])
    text = clip_text_weights(c["vocab"], c["width"], c["layers"], c["seed"])
    missing, unexpected = m.load_state_dict(text, strict=False)
    assert not unexpected and missing == [], (missing, unexpected)
    return m, None, None


def prompt_templates() -> list:
    """`prompt_list` of the reference's nuScenes dataset module, read without importing it (it needs mmdet3d)."""
    from oracle import ref_loader as R
    src = (R.REFERENCE_ROOT / "sgm" / "data" / "nuscenes_video" / "nuscenes_datasets_video.py").read_text()
    for node in ast.parse(src).body:
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "prompt_list" for t in node.targets):
            return ast.literal_eval(node.value)
    raise RuntimeError("prompt_list not found")


@torch.no_grad()
def golden_case(case: str) -> dict:
    from oracle import ref_loader as R
    R.import_reference()
    import open_clip
    from sgm.modules.encoders import modules as M
    c = CASES[case]
    saved = getattr(open_clip, "create_model_and_transforms", None)
    open_clip.create_model_and_transforms = _create_model_and_transforms
    try:
        emb = M.FrozenOpenCLIPEmbedder(arch=c["arch"], device="cpu", layer=c["layer"])
    finally:
        if saved is None:
            del open_clip.create_model_and_transforms
        else:
            open_clip.create_model_and_transforms = saved
    tokens = clip_text_tokens(case)
    out = emb.encode_with_transformer(tokens)
    return {"config": {k: c[k] for k in ("vocab", "width", "layers", "heads", "seed")}, "ctx": CTX, "layer": c["layer"],
            "layer_idx": emb.layer_idx, "tokens": tokens, "keys": sorted(emb.model.state_dict()),
            "out_shape": tuple(out.shape), "out_stride": OUT_STRIDE[case], "out": golden_subset(out, OUT_STRIDE[case])}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="", help="comma-separated subset of: full, small")
    a = ap.parse_args(argv)
    only = set(filter(None, a.only.split(","))) or set(CASES)
    path = GOLDEN / "clip_text.pt"
    res = torch.load(path) if path.exists() else {}
    for case in CASES:
        if case in only:
            res[case] = golden_case(case)
            print(f"{case}: out {tuple(res[case]['out'].shape)} rms {res[case]['out'].pow(2).mean().sqrt():.4f}", flush=True)
    res["prompt_templates"] = prompt_templates()
    torch.save(res, path)


if __name__ == "__main__":
    main(sys.argv[1:])
