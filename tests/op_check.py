"""TEST INFRASTRUCTURE — per-call replay check of an op set against an fp64 reference of the same call.

`checked(Base)` returns `Base` (NativeOps / ParityOps, or one of the torch emulations of tests/torch_ref_ops.py) with a
mixin in front. For every kernel method it snapshots the tensor arguments, runs the kernel, synchronises, recomputes the
call in fp64 on the snapshot (TorchRefOps64 semantics: the SAME operands the kernel read — bf16, or the split encodings
[hi | lo | hi] / [hi | hi | lo] whose products are exact in fp64) and asserts |got - ref| <= bound element by element.
The bounds are derived from the arithmetic of each kernel, next to its checker below; they are never fitted to data.

Also checked: every argument that is not an output is bitwise unchanged, and so is every part of an `out=` the op must
not write; the first call of each distinct signature is run once more on the snapshot into a fresh output and must
match bitwise (fixed reduction order); the first call of each distinct `gemm` signature is run once more into a
NaN-filled buffer with a wider row stride and an extra row, which must stay NaN outside the output.

Coverage: every public method of the op set either has a checker or is on EXCLUDED with a reason; calling any other
public method raises, so a kernel added later cannot escape the check.
"""
from __future__ import annotations

import inspect
import json
import math
import os
import sys
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

from panacea_b200.ops import split_encode
from torch_ref_ops import TorchRefOps64

F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
U_BF16, U_SPLIT, U_F32 = 2.0 ** -8, 2.0 ** -16, 2.0 ** -22   # store rounding, relative to |value|
TAU = 2.0 ** -14          # GEMM accumulation, relative to sum_k |a_k w_k| (see DESIGN.md section 5)
EPS_F32 = 2.0 ** -24      # fp32 unit roundoff: a serial sum of n terms errs by <= n * EPS_F32 * sum |terms|
TINY = 1e-38              # below the smallest normal fp32/bf16: an element whose ref and bound are 0 must be exactly 0

EXCLUDED = {
    "pack_matrix": "host-side weight packing",
    "pack_small": "host-side weight packing",
    "groupnorm_ctas_per_frame": "host-side launch geometry query",
    "sampler_step": "checked against fp64 in test_samplers_gpu.py",
    "cfg_euler_step": "checked against fp64 in test_samplers_gpu.py",
    "scale_dup": "checked against fp64 in test_samplers_gpu.py",
}
OP_CLASS = {"gemm": "gemm", "linear_small": "gemm", "groupnorm": "norm", "groupnorm_pixel": "norm", "layernorm": "norm",
            "attention_view": "attention", "attention_text": "attention", "attention_temporal": "attention",
            "attention_causal": "attention", "gelu_operand": "pointwise", "timestep_embedding": "pointwise",
            "softmax_rows": "pointwise", "conv3x3_direct": "pointwise", "token_embedding": "layout",
            "im2col_s2": "layout", "upsample2x": "layout", "concat_add": "layout", "add_": "layout",
            "cast_operand": "layout", "nchw_to_nhwc": "layout", "nhwc_to_nchw": "layout", "fingerprint": "layout"}


class OpCheckError(AssertionError):
    pass


# ------------------------------------------------------------------------------------------------ stored formats
def _fmt(got, width):
    """storage format of a kernel output whose logical last dimension is `width`"""
    if got.dtype == F32:
        return "f32"
    if got.dtype == BF16 and got.shape[-1] == 3 * width:
        return "split3"
    if got.dtype == BF16 and got.shape[-1] == width:
        return "bf16"
    raise OpCheckError(f"output {tuple(got.shape)} {got.dtype} is no format of width {width}")


def _decode(got, fmt):
    """fp64 value of a stored output; split3 [hi | lo | hi]: hi + lo, and both hi copies must be equal"""
    if fmt != "split3":
        return got.double()
    hi, lo, hi2 = got.split(got.shape[-1] // 3, dim=-1)
    if not torch.equal(hi.view(torch.int16), hi2.view(torch.int16)):
        raise OpCheckError("split3 output: the two hi copies differ")
    return hi.double() + lo.double()


def _unit(fmt):
    return {"f32": U_F32, "bf16": U_BF16, "split3": U_SPLIT}[fmt]


def _encode(x, fmt):
    """the exact stored form of a value that is representable in fp32 (layout / cast ops are bitwise)"""
    x = x.float()
    if fmt == "f32":
        return x
    if fmt == "bf16":
        return x.to(BF16)
    return split_encode(x, weight_form=fmt == "split3b")


def _bits(t):
    return t.contiguous().view(torch.uint8)


def _same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _clone(t):
    c = torch.empty_strided(t.size(), t.stride(), dtype=t.dtype, device=t.device)
    c.copy_(t)
    return c


def _span(t):
    lo = t.data_ptr()
    n = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride())) if t.numel() else 0
    return lo, lo + n * t.element_size()


def _overlaps(a, b):
    (a0, a1), (b0, b1) = _span(a), _span(b)
    return a.device == b.device and a0 < b1 and b0 < a1


# ------------------------------------------------------------------------------------------------ element bounds
def _abs_gemm(a, w, taps):
    """sum_k |a_k| |w_k| of every output element (fp64)"""
    return TorchRefOps64().gemm(a.abs(), w.abs(), taps=taps)


def _norm_bound(ref, xhat, ratio, gamma, silu, fmt):
    """normalisation kernels (fp32 statistics, one pass of sums): the mean and variance carry relative errors of a few
    2^-24 * (1 + mu^2/sigma^2) over at most 2^8 serial terms per thread plus the tree, i.e. <= 2^-16 (1 + mu^2/sigma^2) on
    x_hat; gamma carries it to the output, SiLU multiplies it by at most 1.1 and adds its own ex2/rcp.approx 2^-20."""
    e = 2.0 ** -16 * (1.0 + ratio) * gamma.abs() * (xhat.abs() + 1.0)
    if silu:
        e = 1.1 * e + 2.0 ** -20 * ref.abs()
    return e + _unit(fmt) * (ref.abs() + e)


class _Checks:
    """fp64 reference and element bound of one call: each method returns (ref, bound, extra) on the snapshot."""

    R = TorchRefOps64()

    # ---------------------------------------------------------------- gemm
    def gemm(self, got, a, w, *, bias=None, rowvec=None, rows_per_group=0, n_groups=0, residual=None, residual2=None,
             geglu=False, out_dtype=F32, taps=(1, 1), out=None, ln=None, ln_stats_out=False):
        """bound = TAU * (|A| |W|^T) + 2^-22 * (|bias| + |rowvec| + |residuals|) + store rounding.
        TAU = 2^-14: one 64-channel k-block carries ~sqrt(64) / (0.64 K taps) of sum |a w| (~2^-10 at K taps = 11,520),
        while the fp32 accumulation of K taps products errs by far less than 2^-16 of it."""
        R = self.R
        kw = dict(bias=bias, rowvec=rowvec, rows_per_group=rows_per_group, n_groups=n_groups, taps=taps)
        aw = _abs_gemm(a, w, taps).reshape(-1, w.shape[0])
        rows = aw.shape[0]
        add = torch.zeros_like(aw)
        if bias is not None:
            add += bias.double().abs()
        if rowvec is not None:
            add += rowvec.double().abs()[(torch.arange(rows, device=aw.device) // rows_per_group) % n_groups]
        extra = {}
        if ln is not None:
            # folded LayerNorm: out = rstd (A W'^T - mu s) + t, with mu/rstd from the stats the kernel was given. The
            # kernel forms var = E[y^2] - mu^2 in fp32: rstd carries <= 2^-21 (1 + mu^2/var) relative on top.
            st, colsum, eps = ln
            C = a.shape[-1]
            s64 = st.double()
            mu = s64[..., 0].sum(1) / C
            var = (s64[..., 1].sum(1) / C - mu * mu).clamp_min(0)
            rstd = 1.0 / torch.sqrt(var + eps)
            ratio = mu * mu / (var + eps)
            raw = R.gemm(a, w).reshape(rows, -1) - mu[:, None] * colsum.double()[None, :]
            e = TAU * rstd[:, None] * (aw + mu.abs()[:, None] * colsum.double().abs()[None, :]) \
                + 2.0 ** -21 * (1 + ratio[:, None]) * rstd[:, None] * raw.abs()
            extra["mu2_over_var"] = ratio.max().item()
        else:
            e = TAU * aw
        if geglu:
            # value * gelu(gate): |gelu| <= |g|, |gelu'| <= 1.13, the erfc fit errs by <= 1.1e-6 (ptx.cuh geglu_f32)
            y = R.gemm(a, w, **kw).reshape(rows, -1)
            e = e + U_F32 * (add + y.abs())
            y3, e3 = y.reshape(rows, -1, 2, 16), e.reshape(rows, -1, 2, 16)
            v, g, ev, eg = y3[:, :, 0], y3[:, :, 1], e3[:, :, 0], e3[:, :, 1]
            e = (g.abs() + eg) * ev + (v.abs() + ev) * (1.13 * eg + 1.1e-6 + U_F32 * g.abs())
            e = e.reshape(rows, -1)
            add = 0.0
        for r in (residual, residual2):
            if r is not None:
                add = add + r.double().abs().reshape(rows, -1)
        e = e + U_F32 * add
        res = R.gemm(a, w, **kw, geglu=geglu, residual=residual, residual2=residual2, ln=ln, ln_stats_out=ln_stats_out)
        ref, stats = res if ln_stats_out else (res, None)
        ref = ref.reshape(rows, -1)
        if stats is not None:
            # parts: sums of the pre-store values over their columns -> bounded by the sums of the element bounds (and the
            # fp32 sum of <= 80 terms: 2^-17 of sum |y|, 2^-17 of sum y^2)
            n = ref.shape[1]
            half = (160 if n % 160 == 0 else 128) // 2
            er = e.reshape(rows, -1, half)
            yr = ref.reshape(rows, -1, half).abs()
            es = er.sum(-1) + 2.0 ** -17 * yr.sum(-1)
            eq = (2 * yr * er + er * er).sum(-1) + 2.0 ** -17 * (yr * yr).sum(-1)
            extra["stats"] = (stats, torch.stack([es, eq], -1))
        fmt = _fmt(got[0] if ln_stats_out else got, ref.shape[-1])
        return ref, e + _unit(fmt) * (ref.abs() + e), extra

    # ---------------------------------------------------------------- norms
    def groupnorm(self, got, x, gamma, beta, eps, silu, want_raw=False, out_f32=False):
        Fr, C = x.shape[0], x.shape[-1]
        x64 = x.double().reshape(Fr, -1, 32, C // 32)
        mu = x64.mean((1, 3), keepdim=True)
        var = x64.var((1, 3), unbiased=False, keepdim=True)
        xhat = ((x64 - mu) / torch.sqrt(var + eps)).reshape(x.shape)
        ratio = (mu * mu / (var + eps)).max().item()
        y = got[0] if want_raw else got
        ref = self.R.groupnorm(x, gamma, beta, eps, silu)
        fmt = _fmt(y, C)
        g = gamma.double().repeat(1)
        return ref, _norm_bound(ref, xhat, ratio, g, silu, fmt), {"mu2_over_var": ratio, "raw": x if want_raw else None}

    def groupnorm_pixel(self, got, x, gamma, beta, eps, silu):
        b, T, P, C = x.shape
        x64 = x.double().reshape(b, T, P, 32, C // 32)
        mu = x64.mean((1, 4), keepdim=True)
        var = x64.var((1, 4), unbiased=False, keepdim=True)
        xhat = ((x64 - mu) / torch.sqrt(var + eps)).reshape(x.shape)
        ratio = (mu * mu / (var + eps)).max().item()
        ref = self.R.groupnorm_pixel(x, gamma, beta, eps, silu)
        return ref, _norm_bound(ref, xhat, ratio, gamma.double(), silu, _fmt(got, C)), {"mu2_over_var": ratio}

    def layernorm(self, got, x, gamma, beta, eps=1e-5, out_f32=False):
        x64 = x.double()
        mu = x64.mean(-1, keepdim=True)
        var = x64.var(-1, unbiased=False, keepdim=True)
        xhat = (x64 - mu) / torch.sqrt(var + eps)
        ratio = (mu * mu / (var + eps)).max().item()
        ref = self.R.layernorm(x, gamma, beta, eps)
        return ref, _norm_bound(ref, xhat, ratio, gamma.double(), False, _fmt(got, x.shape[-1])), {"mu2_over_var": ratio}

    # ---------------------------------------------------------------- attention
    @staticmethod
    def _attn_bound(ref, pv, q, k, heads, fmt, exact_p):
        """bf16 path: P is rounded to bf16 before PV (2^-8), the row sum is not -> 2^-7 (P |V|); fp32 path: 2^-16 (P |V|).
        Both: the fp32 scores err by <= d 2^-24 scale |q| |k| (Cauchy-Schwarz per head), exp turns that into a relative
        error of P, twice (numerator and row sum)."""
        d = q.shape[-1] // heads
        qn = q.double().reshape(*q.shape[:-1], heads, d).norm(dim=-1)
        kn = k.double().reshape(-1, heads, d).norm(dim=-1).amax(0)
        ds = d * EPS_F32 * d ** -0.5 * qn * kn
        ds = ds.repeat_interleave(d, dim=-1)
        c = U_SPLIT if exact_p else 2.0 ** -7
        e = (c + 2 * ds) * pv
        return e + _unit(fmt) * (ref.abs() + e)

    def _attn(self, got, name, qkv, heads, *args):
        C = qkv.shape[-1] // 3
        ref = getattr(self.R, name)(qkv, heads, *args)
        qkv_abs = torch.cat([qkv[..., :2 * C], qkv[..., 2 * C:].abs()], -1)
        pv = getattr(self.R, name)(qkv_abs, heads, *args)
        fmt = _fmt(got, C)
        return ref, self._attn_bound(ref, pv, qkv[..., :C], qkv[..., C:2 * C], heads, fmt, qkv.dtype == F32), {}

    def attention_view(self, got, qkv, heads, cross, neighbours):
        return self._attn(got, "attention_view", qkv, heads, cross, neighbours)

    def attention_temporal(self, got, qkv, heads):
        return self._attn(got, "attention_temporal", qkv, heads)

    def attention_causal(self, got, qkv, heads):
        return self._attn(got, "attention_causal", qkv, heads)

    def attention_text(self, got, q, kv, heads):
        C = q.shape[-1]
        ref = self.R.attention_text(q, kv, heads)
        pv = self.R.attention_text(q, torch.cat([kv[..., :C], kv[..., C:].abs()], -1), heads)
        return ref, self._attn_bound(ref, pv, q, kv[..., :C], heads, _fmt(got, C), q.dtype == F32), {}

    # ---------------------------------------------------------------- pointwise with approximations
    def gelu_operand(self, got, x):
        """erff: <= 2 ulp -> 2^-22 (|x| + |gelu|)"""
        ref = self.R.gelu_operand(x)
        e = U_F32 * (x.double().abs() + ref.abs())
        return ref, e + _unit(_fmt(got, x.shape[-1])) * (ref.abs() + e), {}

    def timestep_embedding(self, got, t, dim):
        """cosf / sinf of the same fp32 argument: <= 2 ulp of a value <= 1"""
        ref = self.R.timestep_embedding(t, dim)
        return ref, U_F32 * (1.0 + ref.abs()), {}

    def softmax_rows(self, got, s, scale):
        """per element: the fp32 exponent argument errs by 2^-23 (|s| + max|s|) scale log2(e), exp2f by 2 ulp, the row sum
        (N/256 serial terms per thread, 5 shuffle levels, 8 warps) by (N/256 + 13) 2^-24, 1/sum and the product 2 ulp"""
        ref = self.R.softmax_rows(s, scale)
        s64 = s.double().abs()
        m = s64.amax(-1, keepdim=True)
        lg = scale * 1.4426950408889634
        d_el = 2.0 ** -23 * (s64 + m) * lg * math.log(2) + 2.0 ** -22
        rel = d_el + d_el.amax(-1, keepdim=True) + (s.shape[-1] / 256 + 13) * EPS_F32 + 2.0 ** -22
        e = rel * ref
        return ref, e + _unit(_fmt(got, s.shape[-1])) * (ref + e), {}

    def conv3x3_direct(self, got, x, w_packed, bias, cout, *, stride=1, silu=False, addend=None, out_dtype=F32):
        """fp32 FMAs over 9 Cin products: (9 Cin + 1) 2^-24 of sum |x w|; SiLU as in the norms"""
        R = self.R
        ref = R.conv3x3_direct(x, w_packed, bias, cout, stride=stride, silu=silu, addend=addend)
        xw = R.conv3x3_direct(x.double().abs(), w_packed.abs(), None, cout, stride=stride)
        e = (9 * x.shape[-1] + 1) * EPS_F32 * xw + U_F32 * (bias.double().abs() if bias is not None else 0.0)
        if silu:
            e = 1.1 * e + 2.0 ** -20 * ref.abs()
        if addend is not None:
            e = e + U_F32 * addend.double().abs()
        return ref, e + _unit(_fmt(got, cout)) * (ref.abs() + e), {}

    def linear_small(self, got, x, w, bias, silu_in=False, silu_out=False):
        """fp32 dot products of K terms: (K + 1) 2^-24 of sum |x w| (plus SiLU's 2^-20 on the input and the output)"""
        R = self.R
        ref = R.linear_small(x, w, bias, silu_in, silu_out)
        xa = torch.nn.functional.silu(x.double()) if silu_in else x.double()
        xw = xa.abs() @ w.double().abs().t()
        e = (x.shape[1] + 1) * EPS_F32 * xw + U_F32 * (bias.double().abs() if bias is not None else 0.0)
        if silu_in:
            e = e + 2.0 ** -20 * (x.double().abs() @ w.double().abs().t())
        if silu_out:
            e = 1.1 * e + 2.0 ** -20 * ref.abs()
        return ref, e + U_F32 * ref.abs(), {}


# ------------------------------------------------------------------------------------------------ bitwise ops
def _bitwise_ref(name, got, args, kw, weight_form=False):
    """the exact output of a layout / cast / embedding op, in the output's stored form"""
    R = TorchRefOps64()
    if name == "token_embedding":
        return R.token_embedding(*args).float()
    if name == "concat_add":
        return R.concat_add(*(None if a is None else a.double() for a in args)).float()
    if name == "add_":
        return (args[0].double() + args[1].double()).float()
    if name == "nhwc_to_nchw":
        return R.nhwc_to_nchw(*args, **kw)
    if name == "im2col_s2":
        cols, geo = R.im2col_s2(*args, **kw)
        x = args[0]
        fmt = _fmt(got[0], 9 * x.shape[-1])
        return _encode(cols.reshape(cols.shape[0], 9, x.shape[-1]), fmt).reshape(got[0].shape), geo
    if name == "upsample2x":
        y = R.upsample2x(args[0])
        return _encode(y, _fmt(got, y.shape[-1]))
    if name == "cast_operand":
        x = args[0]
        fmt = _fmt(got, x.shape[-1])
        return _encode(x, "split3b" if fmt == "split3" and weight_form else fmt)
    raise KeyError(name)


def _fingerprint_ref(x):
    w = np.frombuffer(x.detach().cpu().contiguous().numpy().tobytes(), dtype=np.uint32).astype(np.uint64)
    i = np.arange(w.size, dtype=np.uint64)
    with np.errstate(over="ignore"):
        s1 = int(w.sum(dtype=np.uint64))
        s2 = int((w * (i * np.uint64(0x9E3779B97F4A7C15) + np.uint64(0xD1B54A32D192ED03))).sum(dtype=np.uint64))
    signed = lambda v: v - (1 << 64) if v >= 1 << 63 else v
    return (signed(s1), signed(s2), tuple(x.shape), x.dtype)


BITWISE = ("token_embedding", "concat_add", "add_", "nhwc_to_nchw", "im2col_s2", "upsample2x", "cast_operand",
           "nchw_to_nhwc", "fingerprint")
CHECKED = tuple(m for m in dir(_Checks) if not m.startswith("_") and m != "R") + BITWISE


# ------------------------------------------------------------------------------------------------ the mixin
def _site():
    """the innermost engine frame (panacea_b200/*.py, not ops.py) and the block key it works on"""
    fr = sys._getframe(2)
    while fr is not None:
        f = fr.f_code.co_filename.replace("\\", "/")
        if "/panacea_b200/" in f and not f.endswith("/ops.py"):
            loc = fr.f_locals
            key = next((loc[n] for n in ("t", "k", "key") if isinstance(loc.get(n), str)), None)
            if key is None and hasattr(loc.get("st"), "key"):
                key = loc["st"].key
            return f"{Path(f).name}:{fr.f_lineno} {fr.f_code.co_name}" + (f" [{key}]" if key else "")
        fr = fr.f_back
    return "<direct call>"


def _sig(name, args, kw):
    def one(v):
        if isinstance(v, torch.Tensor):
            return (tuple(v.shape), tuple(v.stride()), str(v.dtype))
        if isinstance(v, (tuple, list)):
            return tuple(one(u) for u in v)
        return v if isinstance(v, (int, float, bool, str, type(None))) else type(v).__name__
    return (name, tuple(one(a) for a in args), tuple(sorted((k, one(v)) for k, v in kw.items())))


def _tensors(args, kw):
    out = []
    for v in list(args) + list(kw.values()):
        if isinstance(v, torch.Tensor):
            out.append(v)
        elif isinstance(v, (tuple, list)):
            out.extend(u for u in v if isinstance(u, torch.Tensor))
    return out


class CheckMixin:
    """Goes in front of an op set (see `checked`). `first_only`: check only the first call of each distinct signature."""

    first_only = False

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.calls = 0
        self.seen = set()
        self.stats = defaultdict(lambda: {"calls": 0, "signatures": 0, "worst_ratio": 0.0, "worst_at": None})
        self.mu2 = {}                  # call site -> max mu^2/sigma^2 of a norm
        self.unchecked = []

    def _sync(self, t):
        if t.is_cuda:
            torch.cuda.synchronize(t.device)

    def _fail(self, name, idx, site, sig, what):
        raise OpCheckError(f"{name} call #{idx} at {site}: {what}\n  signature: {sig}")

    def _run(self, name, args, kw):
        fn = getattr(super(CheckMixin, self), name)
        tens = _tensors(args, kw)
        idx = self.calls
        self.calls += 1
        sig = _sig(name, args, kw)
        first = sig not in self.seen
        if self.first_only and not first:
            return fn(*args, **kw)
        self.seen.add(sig)
        site = _site()
        memo = {}

        def snap(v):
            if isinstance(v, torch.Tensor):
                key = (v.data_ptr(), tuple(v.shape), tuple(v.stride()), v.dtype)
                if key not in memo:
                    memo[key] = _clone(v)
                return memo[key]
            if isinstance(v, tuple) and any(isinstance(u, torch.Tensor) for u in v):
                return tuple(snap(u) for u in v)
            return v
        s_args = [snap(v) for v in args]
        s_kw = {k: snap(v) for k, v in kw.items()}
        got = fn(*args, **kw)
        self._sync(tens[0])
        # the outputs: the returned tensors plus `out=` / in-place targets
        outs = [got] if isinstance(got, torch.Tensor) else [g for g in (got if isinstance(got, tuple) else ()) if isinstance(g, torch.Tensor)]
        if name == "add_":
            outs.append(args[0])
        if kw.get("out") is not None:
            outs.append(kw["out"])
        for i, t in enumerate(tens):
            if any(_overlaps(t, o) for o in outs):
                continue
            if not _same_bits(t, snap(t)):
                self._fail(name, idx, site, sig, f"input tensor #{i} {tuple(t.shape)} was modified")
        st = self.stats[name]
        st["calls"] += 1
        st["signatures"] += int(first)
        ratio = self._check(name, idx, site, sig, got, args, kw, s_args, s_kw)
        if ratio > st["worst_ratio"] or st["worst_at"] is None:
            st["worst_ratio"], st["worst_at"] = ratio, f"call #{idx} {site}"
        if first and (name == "gemm" or (name not in ("fingerprint", "add_") and kw.get("out") is None)):
            self._replay(name, idx, site, sig, got, s_args, s_kw)
        return got

    # ---------------------------------------------------------------- value check
    def _check(self, name, idx, site, sig, got, args, kw, s_args, s_kw):
        if name == "fingerprint":
            if got != _fingerprint_ref(s_args[0]):
                self._fail(name, idx, site, sig, f"{got[:2]} != {_fingerprint_ref(s_args[0])[:2]}")
            return 0.0
        if name == "nchw_to_nhwc":
            x = s_args[0]
            out, ch_off = kw.get("out"), kw.get("ch_off", 0)
            want = x.permute(0, 2, 3, 1)
            if out is None:
                return self._bitwise(name, idx, site, sig, got, want.contiguous())
            before = _clone(s_kw["out"])
            before[..., ch_off:ch_off + x.shape[1]] = want
            return self._bitwise(name, idx, site, sig, got, before)
        if name in BITWISE:
            want = _bitwise_ref(name, got, s_args, s_kw, weight_form=s_kw.get("weight_form", False))
            if name == "im2col_s2":
                if tuple(got[1]) != tuple(want[1]):
                    self._fail(name, idx, site, sig, f"geometry {got[1]} != {want[1]}")
                return self._bitwise(name, idx, site, sig, got[0], want[0])
            return self._bitwise(name, idx, site, sig, got, want)
        ref, bound, extra = getattr(_Checks(), name)(got, *s_args, **s_kw)
        y = got
        if name == "gemm":
            y = got[0] if kw.get("ln_stats_out") else got
            y = y.reshape(-1, y.shape[-1]) if y.is_contiguous() else y
        if name == "groupnorm" and isinstance(got, tuple):
            y, raw = got
            self._bitwise(name + ".raw", idx, site, sig, raw, _encode(s_args[0], _fmt(raw, s_args[0].shape[-1])))
        if "mu2_over_var" in extra:
            self.mu2[site] = max(self.mu2.get(site, 0.0), extra["mu2_over_var"])
        ratio = self._compare(name, idx, site, sig, y, ref, bound)
        if "stats" in extra:
            (ref_st, b_st), got_st = extra["stats"], got[1]
            ratio = max(ratio, self._compare(name + ".ln_stats_out", idx, site, sig, got_st, ref_st, b_st, raw=True))
        return ratio

    def _bitwise(self, name, idx, site, sig, got, want):
        if not _same_bits(got, want):
            if got.shape != want.shape or got.dtype != want.dtype:
                self._fail(name, idx, site, sig, f"output {tuple(got.shape)} {got.dtype} != {tuple(want.shape)} {want.dtype}")
            bad = (_bits(got) != _bits(want)).reshape(-1).nonzero()
            self._fail(name, idx, site, sig, f"not bitwise: {bad.shape[0]} bytes differ, first at byte {bad[0].item()}")
        return 0.0

    def _compare(self, name, idx, site, sig, got, ref, bound, raw=False):
        width = ref.shape[-1]
        fmt = "f32" if raw else _fmt(got, width)
        g = _decode(got, fmt).reshape(ref.shape)
        d = (g - ref).abs()
        bad = ~(d <= bound)                          # NaN anywhere is a violation
        r = d / bound.clamp_min(TINY)
        ratio = float(r[~bad].max()) if (~bad).any() else 0.0
        if bad.any():
            i = int(torch.nonzero(bad.reshape(-1))[0].item()) if not bad.all() else 0
            k = torch.unravel_index(torch.tensor(i), ref.shape)
            where = tuple(int(v) for v in k)
            self._fail(name, idx, site, sig, f"{int(bad.sum())} of {ref.numel()} elements out of bound; worst ratio "
                       f"{float(r.max()):.3g}; first at {where}: got {g[where].item():.9g} ref {ref[where].item():.9g} "
                       f"bound {bound[where].item():.3g}")
        return ratio

    # ---------------------------------------------------------------- reproducibility / out-of-bounds writes
    def _replay(self, name, idx, site, sig, got, s_args, s_kw):
        fn = getattr(super(CheckMixin, self), name)
        memo = {}

        def fresh(v):
            if isinstance(v, torch.Tensor):
                key = id(v)
                if key not in memo:
                    memo[key] = _clone(v)
                return memo[key]
            if isinstance(v, tuple) and any(isinstance(u, torch.Tensor) for u in v):
                return tuple(fresh(u) for u in v)
            return v
        again = fn(*[fresh(v) for v in s_args], **{k: fresh(v) for k, v in s_kw.items()})
        self._sync(_tensors(s_args, s_kw)[0])
        pairs = list(zip(got, again)) if isinstance(got, tuple) else [(got, again)]
        for a, b in pairs:
            if isinstance(a, torch.Tensor) and not _same_bits(a, b):
                self._fail(name, idx, site, sig, "a second run on the same inputs is not bitwise the first")
        if name != "gemm" or not got_is_cuda(got):
            return
        y = got[0] if isinstance(got, tuple) else got
        if s_kw.get("geglu") and self.operand_mult == 3:
            return                                  # parity GEGLU takes no out=
        rows, n_out = y.numel() // y.shape[-1], y.shape[-1]
        canary = torch.full((rows + 1, n_out + 64), float("nan"), device=y.device, dtype=y.dtype)
        memo.clear()                                # the run above wrote into its clones of out / residual
        kw = {k: fresh(v) for k, v in s_kw.items()}
        out = s_kw.get("out")
        if out is not None and kw.get("residual") is not None and kw["residual"] is kw["out"]:
            kw["residual"] = _clone(kw["residual"])
        kw["out"] = canary[:rows, :n_out]
        res = fn(*[fresh(v) for v in s_args], **kw)
        self._sync(y)
        if not torch.isnan(canary[:rows, n_out:]).all() or not torch.isnan(canary[rows:]).all():
            self._fail(name, idx, site, sig, "wrote outside its output rows / columns")
        written = canary[:rows, :n_out]
        if torch.isnan(written).any():
            self._fail(name, idx, site, sig, "left output elements unwritten")
        yy = y.reshape(rows, n_out) if y.is_contiguous() else y
        if not _same_bits(written.contiguous(), yy.contiguous()):
            self._fail(name, idx, site, sig, "output at a wider row stride differs from the original run")
        del res

    # ---------------------------------------------------------------- reporting
    def records(self, run, precision):
        """one record per op class seen in this run"""
        by = defaultdict(lambda: {"calls": 0, "signatures": 0, "worst_ratio": 0.0, "worst_at": None, "ops": {}})
        for op, st in self.stats.items():
            c = by[OP_CLASS[op]]
            c["calls"] += st["calls"]
            c["signatures"] += st["signatures"]
            c["ops"][op] = round(st["worst_ratio"], 4)
            if st["worst_ratio"] >= c["worst_ratio"]:
                c["worst_ratio"], c["worst_at"] = st["worst_ratio"], f"{op} {st['worst_at']}"
        out = []
        for cls, c in sorted(by.items()):
            rec = {"run": run, "precision": precision, "op_class": cls, **c}
            if cls == "norm" and self.mu2:
                site = max(self.mu2, key=self.mu2.get)
                rec["max_mu2_over_var"], rec["max_mu2_over_var_at"] = self.mu2[site], site
            out.append(rec)
        return out


def got_is_cuda(got):
    t = got[0] if isinstance(got, tuple) else got
    return isinstance(t, torch.Tensor) and t.is_cuda


def _public(cls):
    return {n for n, v in inspect.getmembers(cls, callable) if not n.startswith("_")}


def checked(base):
    """`base` with the checking mixin in front; public methods that are neither checked nor excluded raise."""
    ns = {}
    for name in _public(base):
        if name in EXCLUDED:
            continue
        if name in CHECKED:
            ns[name] = (lambda n: lambda self, *a, **k: self._run(n, a, k))(name)
        else:
            def refuse(self, *a, _n=name, **k):
                self.unchecked.append(_n)
                raise OpCheckError(f"{_n}: public op without a checker and not excluded")
            ns[name] = refuse
    return type("Checked" + base.__name__, (CheckMixin, base), ns)


def log_records(records):
    """print one OP_REPLAY line per record; also append them to the JSON-lines file PN_OP_REPLAY_LOG names, if set"""
    for rec in records:
        print("OP_REPLAY " + json.dumps(rec))
    if not os.environ.get("PN_OP_REPLAY_LOG"):
        return
    out = Path(os.environ["PN_OP_REPLAY_LOG"])
    try:
        out.parent.mkdir(parents=True, exist_ok=True)
        with out.open("a") as f:
            for rec in records:
                f.write(json.dumps(rec) + "\n")
    except OSError:
        pass
