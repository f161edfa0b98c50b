"""OpenCLIP text tower on the hot path's own kernels: the prompt encoder of `FrozenOpenCLIPEmbedder`.

Executes the reference's `FrozenOpenCLIPEmbedder.encode_with_transformer` (sgm/modules/encoders/modules.py:609-629):
x = token_embedding[tokens] + positional_embedding, then the first `layers - layer_idx` residual blocks of open_clip's
text transformer (pre-LN, causal multi-head attention with head_dim 64, MLP c_fc -> exact-erf GELU -> c_proj), then
ln_final. All positions are computed and returned, including the padding after <end_of_text>: the UNet's text
cross-attention reads every one of them.

Per block, on an fp32 residual stream [b*L, width]:
  pn_layernorm (ln_1) -> pn_gemm (in_proj + bias) -> pn_attention_causal -> pn_gemm (out_proj + bias + x)
  pn_layernorm (ln_2) -> pn_gemm (c_fc + bias) -> pn_gelu_operand -> pn_gemm (c_proj + bias + x)
with pn_token_embedding before the blocks and pn_layernorm (fp32 output) after them. bf16 operands with fp32
accumulation in the default op set; split-bf16 operands and fp32 attention in the parity op set. Parameters are
addressed by open_clip's state-dict names, so a stock open_clip file or an engine checkpoint loads unchanged."""
from __future__ import annotations

import torch

F32 = torch.float32
HEAD_DIM = 64


def text_param_spec(vocab: int, ctx: int, width: int, layers: int) -> dict:
    """Keys/shapes of open_clip's text tower (CLIP.token_embedding, positional_embedding, transformer.resblocks.*,
    ln_final) that the embedder reads; text_projection / logit_scale are not used by it."""
    spec = {"token_embedding.weight": (vocab, width), "positional_embedding": (ctx, width)}
    for i in range(layers):
        k = f"transformer.resblocks.{i}."
        spec.update({
            k + "ln_1.weight": (width,), k + "ln_1.bias": (width,),
            k + "attn.in_proj_weight": (3 * width, width), k + "attn.in_proj_bias": (3 * width,),
            k + "attn.out_proj.weight": (width, width), k + "attn.out_proj.bias": (width,),
            k + "ln_2.weight": (width,), k + "ln_2.bias": (width,),
            k + "mlp.c_fc.weight": (4 * width, width), k + "mlp.c_fc.bias": (4 * width,),
            k + "mlp.c_proj.weight": (width, 4 * width), k + "mlp.c_proj.bias": (width,),
        })
    spec.update({"ln_final.weight": (width,), "ln_final.bias": (width,)})
    return spec


def text_config_from_params(P: dict) -> dict:
    """(vocab, ctx, width, layers) read off the shapes of a parameter dict under open_clip's names."""
    vocab, width = tuple(P["token_embedding.weight"].shape)
    ctx = P["positional_embedding"].shape[0]
    layers = 0
    while f"transformer.resblocks.{layers}.ln_1.weight" in P:
        layers += 1
    return {"vocab": vocab, "ctx": ctx, "width": width, "layers": layers}


class TextEncoderEngine:
    def __init__(self, ops):
        self.ops = ops
        self.W = None
        self.cfg = None

    def pack(self, P: dict) -> None:
        cfg = text_config_from_params(P)
        if cfg["width"] % HEAD_DIM:
            raise NotImplementedError(f"text tower width {cfg['width']} is not a multiple of head_dim {HEAD_DIM}")
        spec = text_param_spec(**cfg)
        bad = [k for k, s in spec.items() if k not in P or tuple(P[k].shape) != s]
        if bad:
            raise ValueError(f"text tower parameters missing or misshaped: {bad[:8]}{' ...' if len(bad) > 8 else ''}")
        f = lambda t: t.detach().to(F32).contiguous()
        mat = self.ops.pack_matrix
        W = {"tok": f(P["token_embedding.weight"]), "pos": f(P["positional_embedding"]),
             "lnf.g": f(P["ln_final.weight"]), "lnf.b": f(P["ln_final.bias"])}
        for i in range(cfg["layers"]):
            k = f"transformer.resblocks.{i}."
            W[f"{i}.ln1.g"], W[f"{i}.ln1.b"] = f(P[k + "ln_1.weight"]), f(P[k + "ln_1.bias"])
            W[f"{i}.ln2.g"], W[f"{i}.ln2.b"] = f(P[k + "ln_2.weight"]), f(P[k + "ln_2.bias"])
            W[f"{i}.qkv.w"], W[f"{i}.qkv.b"] = mat(P[k + "attn.in_proj_weight"]), f(P[k + "attn.in_proj_bias"])
            W[f"{i}.out.w"], W[f"{i}.out.b"] = mat(P[k + "attn.out_proj.weight"]), f(P[k + "attn.out_proj.bias"])
            W[f"{i}.fc.w"], W[f"{i}.fc.b"] = mat(P[k + "mlp.c_fc.weight"]), f(P[k + "mlp.c_fc.bias"])
            W[f"{i}.proj.w"], W[f"{i}.proj.b"] = mat(P[k + "mlp.c_proj.weight"]), f(P[k + "mlp.c_proj.bias"])
        self.W, self.cfg = W, cfg

    @property
    def heads(self) -> int:
        return self.cfg["width"] // HEAD_DIM

    @torch.no_grad()
    def encode(self, tokens: torch.Tensor, layer_idx: int) -> torch.Tensor:
        """tokens int64 [b, ctx] -> fp32 [b, ctx, width]: ln_final of the stream after `layers - layer_idx` blocks
        (layer_idx 0 = "last", 1 = "penultimate")."""
        ops, W, cfg = self.ops, self.W, self.cfg
        assert W is not None, "pack() the text tower parameters first"
        n_blocks = cfg["layers"] - layer_idx
        if not 0 < n_blocks <= cfg["layers"]:
            raise ValueError(f"layer_idx {layer_idx} out of range for a {cfg['layers']}-block tower")
        b, L = tokens.shape
        if L != cfg["ctx"]:
            raise ValueError(f"tokens must be [b, {cfg['ctx']}], got {tuple(tokens.shape)}")
        width, heads = cfg["width"], self.heads
        x = ops.token_embedding(tokens.to(W["tok"].device).contiguous(), W["tok"], W["pos"]).view(b * L, width)
        for i in range(n_blocks):
            a = ops.layernorm(x, W[f"{i}.ln1.g"], W[f"{i}.ln1.b"], 1e-5)
            qkv = ops.gemm(a, W[f"{i}.qkv.w"], bias=W[f"{i}.qkv.b"], out_dtype=ops.qkv_dtype)
            o = ops.attention_causal(qkv.view(b, L, 3 * width), heads)
            ops.gemm(o.view(b * L, -1), W[f"{i}.out.w"], bias=W[f"{i}.out.b"], residual=x, out=x)
            a = ops.layernorm(x, W[f"{i}.ln2.g"], W[f"{i}.ln2.b"], 1e-5)
            h = ops.gemm(a, W[f"{i}.fc.w"], bias=W[f"{i}.fc.b"])
            ops.gemm(ops.gelu_operand(h), W[f"{i}.proj.w"], bias=W[f"{i}.proj.b"], residual=x, out=x)
        return ops.layernorm(x, W["lnf.g"], W["lnf.b"], 1e-5, out_f32=True).view(b, L, width)
