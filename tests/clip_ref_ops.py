"""TEST INFRASTRUCTURE — the text-encoder ops (panacea_b200.ops attention_causal / gelu_operand / token_embedding and
layernorm's fp32 output) added to the plain-torch op sets of torch_ref_ops.py, so TextEncoderEngine's orchestration
runs on the CPU. Never imported by the package."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from torch_ref_ops import TorchRefOps, TorchSplitOps, _enc

F32 = torch.float32


class TextRefOps(TorchRefOps):
    def layernorm(self, x, gamma, beta, eps=1e-5, out_f32=False):
        return F.layer_norm(self._c(x), (x.shape[-1],), self._c(gamma), self._c(beta), eps)

    def attention_causal(self, qkv, heads):
        b, L, C3 = qkv.shape
        C = C3 // 3
        q, k, v = (t.reshape(b, L, heads, C // heads).transpose(1, 2) for t in self._c(qkv).split(C, dim=-1))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        return o.transpose(1, 2).reshape(b, L, C)

    def gelu_operand(self, x):
        return F.gelu(self._c(x))

    def token_embedding(self, tokens, table, pos):
        vocab = table.shape[0]
        if int(tokens.min()) < 0 or int(tokens.max()) >= vocab:
            raise ValueError(f"token_embedding: token ids must lie in [0, {vocab})")
        return self._c(table)[tokens] + self._c(pos)[:tokens.shape[1]]


class TextSplitOps(TorchSplitOps, TextRefOps):
    """split-bf16 operands [hi | lo | hi] (ParityOps) for the producers of GEMM operands."""

    def layernorm(self, x, gamma, beta, eps=1e-5, out_f32=False):
        y = TextRefOps.layernorm(self, x, gamma, beta, eps)
        return y if out_f32 else _enc(y)

    def attention_causal(self, qkv, heads):
        return _enc(TextRefOps.attention_causal(self, qkv, heads))

    def gelu_operand(self, x):
        return _enc(TextRefOps.gelu_operand(self, x))
