"""TEST INFRASTRUCTURE — a plain-torch op set with the same interface as panacea_b200.ops.NativeOps.

It exists so that the host-side orchestration (panacea_b200/engine.py: packing, layouts, epilogue fusion
bookkeeping, view/neighbour tables, caching) can be checked on CPU, without a GPU, against the oracle and the
reference's golden outputs. It is never imported by the package: the product path has no fallback.
Semantics follow include/panacea_b200.h literally (channels-last, fused epilogues).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from panacea_b200.ops import split3, split_encode

F32 = torch.float32


class TorchRefOps:
    """fp32 everywhere: operands are plain fp32 tensors, weights stay fp32. Results are allocated on the inputs' device
    and computed in `dtype`; with `pre_store` a method returns its value in `dtype` before the rounding to the output
    dtype the kernel stores (TorchRefOps64, the fp64 reference of the per-call replay check, tests/op_check.py)."""
    dtype = F32
    pre_store = False
    operand_mult = 1
    qkv_dtype = F32
    act_dtype = F32
    fused_operand_emit = False
    token_dtype = F32
    fold_layernorm = False

    def __init__(self):
        self.launches = 0

    def _c(self, t):
        return None if t is None else t.to(self.dtype)

    def _store(self, y, dtype):
        return y if self.pre_store else y.to(dtype)

    def pack_matrix(self, w, taps=1):
        return w.detach().to(F32).contiguous()

    def pack_small(self, w):
        return w.detach().to(F32).contiguous()

    def gemm(self, a, w, *, bias=None, rowvec=None, rows_per_group=0, n_groups=0, residual=None, residual2=None,
             geglu=False, out_dtype=F32, taps=(1, 1), out=None, ln=None, ln_stats_out=False):
        th, tw = taps
        C = a.shape[-1]
        N = w.shape[0]
        wf = self._c(w)
        if (th, tw) == (1, 1):
            lead = a.shape[:-1]
            y = self._c(a).reshape(-1, C) @ wf.t()
            if ln is not None:      # pn_gemm_args.ln_*: finish the folded LayerNorm from the producer's partial row sums
                st, colsum, eps = ln
                st, colsum = self._c(st), self._c(colsum)
                sm, sq = st[..., 0].sum(1), st[..., 1].sum(1)
                mu = sm / C
                rstd = torch.rsqrt((sq / C - mu * mu).clamp_min(0) + eps)
                y = rstd[:, None] * (y - mu[:, None] * colsum[None, :])
        else:
            NB, H, W, _ = a.shape
            lead = (NB, H, W)
            ap = F.pad(self._c(a), (0, 0, tw // 2, tw // 2, th // 2, th // 2))
            y = torch.zeros(NB * H * W, N, device=a.device, dtype=self.dtype)
            for i in range(th):
                for j in range(tw):
                    tap = i * tw + j
                    y += ap[:, i:i + H, j:j + W, :].reshape(-1, C) @ wf[:, tap * C:(tap + 1) * C].t()
        rows = y.shape[0]
        if bias is not None:
            y = y + self._c(bias)
        if rowvec is not None:
            grp = (torch.arange(rows, device=y.device) // rows_per_group) % n_groups
            y = y + self._c(rowvec)[grp]
        if geglu:
            y3 = y.reshape(rows, -1, 2, 16)          # packed layout: 16 value columns, then their 16 gate columns
            y = (y3[:, :, 0] * F.gelu(y3[:, :, 1])).reshape(rows, -1)
        if residual is not None:
            y = y + self._c(residual).reshape(rows, -1)
        if residual2 is not None:
            y = y + self._c(residual2).reshape(rows, -1)
        stats = None
        if ln_stats_out:
            # include/panacea_b200.h pn_gemm_args.ln_stats_out: part 2 * tile + h holds (sum, sum of squares) of the values
            # before the store rounding over columns [h * BN/2, (h + 1) * BN/2) of column tile `tile`, BN = 160 or 128
            n = y.shape[1]
            bn = 160 if n % 160 == 0 else 128
            parts = []
            for c0 in range(0, n, bn // 2):
                cols = y[:, c0:c0 + bn // 2]
                parts.append(torch.stack([cols.sum(1), (cols * cols).sum(1)], -1))
            stats = torch.stack(parts, 1).contiguous()
        y = self._store(y, out_dtype)
        if out is not None:
            out.reshape(rows, -1).copy_(y)
            res = out.reshape(*lead, y.shape[1])
        else:
            res = y.reshape(*lead, y.shape[1])
        return (res, stats) if ln_stats_out else res

    def groupnorm(self, x, gamma, beta, eps, silu, want_raw=False, out_f32=False):
        Fr, C = x.shape[0], x.shape[-1]
        x = self._c(x)
        z = x.reshape(Fr, -1, C).permute(0, 2, 1)
        y = F.group_norm(z, 32, self._c(gamma), self._c(beta), eps)
        if silu:
            y = F.silu(y)
        y = y.permute(0, 2, 1).reshape(x.shape).contiguous()
        return (y, x.clone()) if want_raw else y

    def groupnorm_pixel(self, x, gamma, beta, eps, silu):
        b, T, P, C = x.shape
        z = self._c(x).permute(0, 2, 3, 1).reshape(b * P, C, T)
        y = F.group_norm(z, 32, self._c(gamma), self._c(beta), eps)
        if silu:
            y = F.silu(y)
        return y.reshape(b, P, C, T).permute(0, 3, 1, 2).contiguous()

    def layernorm(self, x, gamma, beta, eps=1e-5, out_f32=False):
        return F.layer_norm(self._c(x), (x.shape[-1],), self._c(gamma), self._c(beta), eps)

    @staticmethod
    def _mha(q, k, v, heads):
        B, Nq, C = q.shape
        d = C // heads
        qh = q.reshape(B, Nq, heads, d).transpose(1, 2)
        kh = k.reshape(B, -1, heads, d).transpose(1, 2)
        vh = v.reshape(B, -1, heads, d).transpose(1, 2)
        s = (qh @ kh.transpose(-1, -2)) * (d ** -0.5)
        return (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, Nq, C)

    def attention_view(self, qkv, heads, cross, neighbours):
        Fr, H, V, w, C3 = qkv.shape
        C = C3 // 3
        q, k, v = self._c(qkv).split(C, dim=-1)
        out = torch.empty(Fr, H, V, w, C, device=qkv.device, dtype=self.dtype)
        for i in range(V):
            nb = neighbours[i] if cross else (i,)
            ki = torch.cat([k[:, :, j] for j in nb], dim=2).reshape(Fr, -1, C)
            vi = torch.cat([v[:, :, j] for j in nb], dim=2).reshape(Fr, -1, C)
            out[:, :, i] = self._mha(q[:, :, i].reshape(Fr, H * w, C), ki, vi, heads).reshape(Fr, H, w, C)
        return self._store(out, qkv.dtype)

    def attention_text(self, q, kv, heads):
        C = q.shape[-1]
        return self._store(self._mha(self._c(q), self._c(kv)[..., :C], self._c(kv)[..., C:], heads), q.dtype)

    def attention_temporal(self, qkv, heads):
        b, T, P, C3 = qkv.shape
        C = C3 // 3
        q, k, v = self._c(qkv).split(C, dim=-1)
        seq = lambda z: z.permute(0, 2, 1, 3).reshape(b * P, T, C)
        o = self._mha(seq(q), seq(k), seq(v), heads)
        return self._store(o.reshape(b, P, T, C).permute(0, 2, 1, 3).contiguous(), qkv.dtype)

    def attention_causal(self, qkv, heads):
        b, L, C3 = qkv.shape
        C = C3 // 3
        q, k, v = (t.reshape(b, L, heads, C // heads).transpose(1, 2) for t in self._c(qkv).split(C, dim=-1))
        o = F.scaled_dot_product_attention(q, k, v, is_causal=True)
        return o.transpose(1, 2).reshape(b, L, C)

    def gelu_operand(self, x):
        # through fp64: torch's fp32 CPU erf errs by several ulp near erf = -1, the kernel's erff by <= 2 ulp
        return F.gelu(x.double()).to(self.dtype)

    def token_embedding(self, tokens, table, pos):
        vocab = table.shape[0]
        if int(tokens.min()) < 0 or int(tokens.max()) >= vocab:
            raise ValueError(f"token_embedding: token ids must lie in [0, {vocab})")
        return self._c(table)[tokens] + self._c(pos)[:tokens.shape[1]]

    def conv3x3_direct(self, x, w_packed, bias, cout, *, stride=1, silu=False, addend=None, out_dtype=F32):
        cin = x.shape[-1]
        w = self._c(w_packed)[:, :cin, :cout].reshape(3, 3, cin, cout).permute(3, 2, 0, 1)
        y = F.conv2d(self._c(x).permute(0, 3, 1, 2), w, self._c(bias), stride=stride, padding=1)
        if silu:
            y = F.silu(y)
        y = y.permute(0, 2, 3, 1)
        if addend is not None:
            y = y + self._c(addend)
        return self._store(y.contiguous(), out_dtype)

    def im2col_s2(self, x, pad=1):
        Fr, H, W, C = x.shape
        if pad == 1:
            Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
            xp = F.pad(x, (0, 0, 1, 1, 1, 1))
        else:
            Ho, Wo = (H - 2) // 2 + 1, (W - 2) // 2 + 1
            xp = F.pad(x, (0, 0, 0, 2, 0, 2))
        cols = torch.stack([xp[:, i:i + 2 * Ho:2, j:j + 2 * Wo:2, :] for i in range(3) for j in range(3)], dim=3)
        return cols.reshape(Fr * Ho * Wo, 9 * C), (Fr, Ho, Wo)

    def upsample2x(self, x):
        return x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)

    def concat_add(self, h, skip, ctrl):
        return torch.cat([h, skip if ctrl is None else skip + ctrl], dim=-1)

    def add_(self, x, y):
        return x.add_(y)

    def cast_operand(self, x, weight_form=False):
        return x

    def softmax_rows(self, s, scale):
        return torch.softmax(self._c(s) * scale, dim=-1)

    def nchw_to_nhwc(self, x, out=None, ch_off=0):
        y = x.permute(0, 2, 3, 1)
        if out is None:
            return y.contiguous()
        out[..., ch_off:ch_off + x.shape[1]] = y
        return out

    def nhwc_to_nchw(self, x, channels=None):
        return (x if channels is None else x[..., :channels]).permute(0, 3, 1, 2).contiguous()

    def timestep_embedding(self, t, dim):
        half = dim // 2
        freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F32) / half).to(t.device)
        args = self._c(t[:, None].float() * freqs[None])       # the fp32 product, as the kernel forms it
        return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)

    def linear_small(self, x, w, bias, silu_in=False, silu_out=False):
        x = self._c(x)
        y = F.linear(F.silu(x) if silu_in else x, self._c(w), self._c(bias))
        return F.silu(y) if silu_out else y

    def cfg_euler_step(self, x, net2, x_in_next, sigma, sigma_next, scale, c_in_next, sigma_q=None, net_is_denoised=False):
        n = x.shape[0]
        sq = sigma if sigma_q is None else sigma_q
        den_u = net2[:n] if net_is_denoised else net2[:n] * (-sq) + x
        den_c = net2[n:] if net_is_denoised else net2[n:] * (-sq) + x
        den = den_u + scale * (den_c - den_u)
        x.copy_(x + (sigma_next - sigma) * ((x - den) / sigma))
        if x_in_next is not None:
            x_in_next.copy_(torch.cat([x, x]) * c_in_next)
        return x

    def scale_dup(self, x, s, copies):
        return torch.cat([x * s] * copies)


class TorchRefOps64(TorchRefOps):
    """The same semantics in fp64, results before the store rounding: the reference each kernel call is checked against.
    Convolutions stay one matmul per tap, so on a GPU they run as fp64 GEMMs."""
    dtype = torch.float64
    pre_store = True


class TorchFoldOps(TorchRefOps):
    """TorchRefOps with the LayerNorm fold switched on (the NativeOps fast-path orchestration: row statistics from the
    producers of the token stream, W diag(gamma) / column sums / W beta in the consumers), fp32 stream on CPU."""
    fold_layernorm = True
    LN_FOLD_MAX_C = 640


class TorchSplitOps(TorchRefOps):
    """CPU emulation of panacea_b200.ops.ParityOps: producers store split-bf16 operands [hi | lo | hi], weights are
    packed [W_hi | W_hi | W_lo] by the product's own split3(), and the GEMM multiplies the bf16 VALUES exactly as the
    tensor core does (bf16 x bf16 products are exact in fp32). Checks the engine's parity-mode packing/orchestration and
    the precision claim of the encoding without a GPU. The VAE mid-block attention's operands come in both split forms:
    the weight-form cast (pn_cast_operand mode 3) and the split3 row softmax (pn_softmax_rows_operand mode 1)."""
    operand_mult = 3

    def pack_matrix(self, w, taps=1):
        return split3(w, taps)

    def gemm(self, a, w, *, geglu=False, out_dtype=F32, **kw):
        y = super().gemm(a, w, geglu=geglu, out_dtype=F32, **kw)
        return split_encode(y) if geglu else y

    def groupnorm(self, x, gamma, beta, eps, silu, want_raw=False, out_f32=False):
        r = super().groupnorm(x, gamma, beta, eps, silu, want_raw)
        if out_f32:
            return r
        return (split_encode(r[0]), split_encode(r[1])) if want_raw else split_encode(r)

    def groupnorm_pixel(self, *a, **k):
        return split_encode(super().groupnorm_pixel(*a, **k))

    def layernorm(self, x, gamma, beta, eps=1e-5, out_f32=False):
        y = super().layernorm(x, gamma, beta, eps)
        return y if out_f32 else split_encode(y)

    def attention_view(self, *a, **k):
        return split_encode(super().attention_view(*a, **k))

    def attention_text(self, *a, **k):
        return split_encode(super().attention_text(*a, **k))

    def attention_temporal(self, *a, **k):
        return split_encode(super().attention_temporal(*a, **k))

    def attention_causal(self, *a, **k):
        return split_encode(super().attention_causal(*a, **k))

    def gelu_operand(self, x):
        return split_encode(super().gelu_operand(x))

    def im2col_s2(self, x, pad=1):
        cols, geo = super().im2col_s2(x, pad)
        C = x.shape[-1]
        return split_encode(cols.reshape(cols.shape[0], 9, C)).reshape(cols.shape[0], 27 * C), geo

    def upsample2x(self, x):
        return split_encode(super().upsample2x(x))

    def cast_operand(self, x, weight_form=False):
        return split_encode(x, weight_form)

    def softmax_rows(self, s, scale):
        return split_encode(super().softmax_rows(s, scale))
