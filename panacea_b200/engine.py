"""Denoising engine: executes the network plan on channels-last buffers through an op set.

One fp32 residual stream `[frames, H, Wtot, C]` (frames = b*T with t fastest, Wtot = 6 views side by side) flows
through the whole network; every GEMM/conv operand is a bf16 tensor produced by the norm/activation kernel in
front of it, and every residual add, bias, time-embedding add, positional-embedding add and GEGLU is a GEMM
epilogue. None of the reference's ~100 rearrange/contiguous copies per SpatialTemporalTransformer exist: the
"(b t)(h w) c -> (b h w) t c" and per-view slicings are index arithmetic inside the kernels.

Step-invariant work is hoisted into `prepare_condition`: the BEV hint stem (controlmodel.py:118) and all 69 text
K/V projections (attention.py:248-250), which the reference recomputes at every step — including 26.8 TFLOP of
per-pixel repeated text K/V in the temporal blocks (attention.py:1122-1125) that simply never happens here.

`ops` is `panacea_b200.ops.NativeOps` in production (hand-written sm_90a kernels). Tests inject a torch
reference op set with the same interface to check this orchestration on CPU; the package itself has no fallback.
"""
from __future__ import annotations

import math

import torch

from .ops import geglu_pack
from .netplan import (CROSS_VIEW_NEIGHBOURS, HINT_STRIDES, STT_BRANCHES, NetConfig, Plan, Stage, make_plan)

F32 = torch.float32


def temporal_pos_table(T: int, dim: int) -> torch.Tensor:
    """Reference-faithful positional table (attention.py:1140-1159): the frequency vector is truncated to int64
    (:1148), so every frequency but the first is 0 and pe[t] = [sin t, cos t, 0, 1, 0, 1, ...]."""
    pe = torch.zeros(T, dim, dtype=F32)
    t = torch.arange(T, dtype=F32)
    pe[:, 0] = torch.sin(t)
    pe[:, 1] = torch.cos(t)
    pe[:, 3::2] = 1.0
    return pe


class PackedWeights(dict):
    """key -> packed device tensor (MMA-operand dtype for matrices, fp32 for biases / norm affine).
    `tag` ("unet" / "controlnet") names the network in the text-K/V cache."""
    tag = ""


STEM_CPAD = 64       # input channels of the stem conv padded to one 64-channel swizzle atom
OUT_NPAD = 8         # output channels of the out-head conv padded to the GEMM's minimum N


def _conv3_matrix(w):      # [Cout, Cin, 3, 3] -> fp32 [Cout, (ky, kx, ci)]
    return w.detach().to(F32).permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def _conv1d_matrix(w):     # [Cout, Cin, 3] -> fp32 [Cout, (k, ci)]
    return w.detach().to(F32).permute(0, 2, 1).reshape(w.shape[0], -1)


def _pack_direct(w, cin_pad=None):   # [Cout, Cin, 3, 3] -> fp32 [9, Cin_pad, Cout_pad16]
    cout, cin = w.shape[0], w.shape[1]
    cin_p = cin_pad or (cin + 3) // 4 * 4
    cout_p = (cout + 15) // 16 * 16
    out = torch.zeros(9, cin_p, cout_p, dtype=F32, device=w.device)
    out[:, :cin, :cout] = w.permute(2, 3, 1, 0).reshape(9, cin, cout).float()
    return out


class Engine:
    """`ops` decides the precision mode: NativeOps (bf16 operands) or ParityOps (split-bf16 operands = fp32-class
    products, fp32 attention). The engine only asks it how to pack a weight matrix (`pack_matrix`, `pack_small`), which
    dtype attention inputs (`qkv_dtype`) and CUDA-core intermediates (`act_dtype`) have, and whether a GEMM epilogue can
    emit the next operand directly (`fused_operand_emit`)."""

    def __init__(self, cfg: NetConfig, ops):
        self.cfg = cfg
        self.ops = ops
        self.plan_unet: Plan = make_plan(cfg, decoder=True)
        self.plan_cn: Plan = make_plan(cfg, decoder=False)
        self.wu: PackedWeights | None = None
        self.wc: PackedWeights | None = None
        self.generation = 0
        self.cond = {"guided": None, "kv": {}, "b": None}     # step-invariant state (prepare_hint / prepare_text)
        self._xin = {}
        self.two_streams = True         # ControlNet || UNet encoder (see eps); False gives the single-stream launch order
        self._side = None

    # ------------------------------------------------------------------------------------------ packing
    def _pack_trunk(self, P: dict, plan: Plan) -> PackedWeights:
        f = lambda t: t.detach().to(F32).contiguous()
        mat, small = self.ops.pack_matrix, self.ops.pack_small
        W = PackedWeights()
        W["te0.w"] = small(P["time_embed.0.weight"]); W["te0.b"] = f(P["time_embed.0.bias"])
        W["te2.w"] = small(P["time_embed.2.weight"]); W["te2.b"] = f(P["time_embed.2.bias"])
        emb_w, emb_b, off = [], [], 0
        for st in plan.stages():
            k = st.key
            if st.kind == "stem":
                # the 8 -> 320 input conv runs on the tensor-core conv kernel with its input channels zero-padded to one
                # 64-channel atom (the CUDA-core direct conv took 660 us per network at level 0; this is ~70 us)
                w_in = P[k + ".weight"].detach().to(F32)
                if w_in.shape[1] > STEM_CPAD:
                    raise NotImplementedError(f"input conv with {w_in.shape[1]} > {STEM_CPAD} channels")
                w_in = torch.nn.functional.pad(w_in, (0, 0, 0, 0, 0, STEM_CPAD - w_in.shape[1]))
                W[k + ".w"] = mat(_conv3_matrix(w_in), 9); W[k + ".b"] = f(P[k + ".bias"])
            elif st.kind == "res":
                for nm in ("in_layers.0", "in_layers_temporal.0", "out_layers.0", "out_layers_temporal.0"):
                    W[f"{k}.{nm}.g"] = f(P[f"{k}.{nm}.weight"]); W[f"{k}.{nm}.b"] = f(P[f"{k}.{nm}.bias"])
                W[k + ".in.w"] = mat(_conv3_matrix(P[k + ".in_layers.2.weight"]), 9); W[k + ".in.b"] = f(P[k + ".in_layers.2.bias"])
                W[k + ".out.w"] = mat(_conv3_matrix(P[k + ".out_layers.3.weight"]), 9); W[k + ".out.b"] = f(P[k + ".out_layers.3.bias"])
                W[k + ".int.w"] = mat(_conv1d_matrix(P[k + ".in_layers_temporal.2.weight"]), 3)
                W[k + ".int.b"] = f(P[k + ".in_layers_temporal.2.bias"])
                W[k + ".outt.w"] = mat(_conv1d_matrix(P[k + ".out_layers_temporal.3.weight"]), 3)
                W[k + ".outt.b"] = f(P[k + ".out_layers_temporal.3.bias"])
                if st.cin != st.cout:
                    W[k + ".skip.w"] = mat(P[k + ".skip_connection.weight"].detach().reshape(st.cout, st.cin))
                    W[k + ".skip.b"] = f(P[k + ".skip_connection.bias"])
                emb_w.append(P[k + ".emb_layers.1.weight"].detach()); emb_b.append(P[k + ".emb_layers.1.bias"].detach())
                W[k + ".emb_off"] = off
                off += st.cout
            elif st.kind == "stt":
                c = st.cin
                for br in STT_BRANCHES:
                    W[f"{k}.norm{br}.g"] = f(P[f"{k}.norm{br}.weight"]); W[f"{k}.norm{br}.b"] = f(P[f"{k}.norm{br}.bias"])
                    for pj in ("proj_in", "proj_out"):
                        W[f"{k}.{pj}{br}.w"] = mat(P[f"{k}.{pj}{br}.weight"])
                        W[f"{k}.{pj}{br}.b"] = f(P[f"{k}.{pj}{br}.bias"])
                    t = f"{k}.transformer_blocks{br}.0"
                    for nm in ("norm1", "norm2", "norm3"):
                        W[f"{t}.{nm}.g"] = f(P[f"{t}.{nm}.weight"]); W[f"{t}.{nm}.b"] = f(P[f"{t}.{nm}.bias"])
                    fold = self._fold_ln(c)
                    W[t + ".fold"] = fold
                    wqkv = torch.cat([P[f"{t}.attn1.to_{n}.weight"].detach() for n in "qkv"], 0)
                    if fold:   # LayerNorm folded into the consumer GEMM: W' = W diag(gamma), s = rowsum(bf16 W'), t = W beta
                        W[t + ".qkv.w"], W[t + ".qkv.s"], W[t + ".qkv.t"] = self._ln_fold_pack(wqkv, None, W[t + ".norm1.g"], W[t + ".norm1.b"])
                        W[t + ".q2.w"], W[t + ".q2.s"], W[t + ".q2.t"] = self._ln_fold_pack(
                            P[t + ".attn2.to_q.weight"].detach(), None, W[t + ".norm2.g"], W[t + ".norm2.b"])
                    else:
                        W[t + ".qkv.w"] = mat(wqkv)
                        W[t + ".q2.w"] = mat(P[t + ".attn2.to_q.weight"])
                    W[t + ".kv2.w"] = mat(torch.cat([P[t + ".attn2.to_k.weight"].detach(), P[t + ".attn2.to_v.weight"].detach()], 0))
                    for a in ("attn1", "attn2"):
                        W[f"{t}.{a}.o.w"] = mat(P[f"{t}.{a}.to_out.0.weight"])
                        W[f"{t}.{a}.o.b"] = f(P[f"{t}.{a}.to_out.0.bias"])
                    # GEGLU: 16 value rows then their 16 gate rows, so one accumulator chunk holds both halves
                    w1, b1 = P[t + ".ff.net.0.proj.weight"].detach(), P[t + ".ff.net.0.proj.bias"].detach()
                    W[t + ".ff1.w"] = mat(geglu_pack(w1))
                    W[t + ".ff1.b"] = geglu_pack(b1).to(F32).contiguous()
                    W[t + ".ff2.w"] = mat(P[t + ".ff.net.2.weight"]); W[t + ".ff2.b"] = f(P[t + ".ff.net.2.bias"])
            elif st.kind == "down":
                W[k + ".w"] = mat(_conv3_matrix(P[k + ".op.weight"]), 9); W[k + ".b"] = f(P[k + ".op.bias"])
            elif st.kind == "up":
                W[k + ".w"] = mat(_conv3_matrix(P[k + ".conv.weight"]), 9); W[k + ".b"] = f(P[k + ".conv.bias"])
        W["emb.w"] = small(torch.cat(emb_w, 0))
        W["emb.b"] = torch.cat(emb_b, 0).to(F32).contiguous()
        return W

    def _fold_ln(self, c: int) -> bool:
        ops = self.ops
        return bool(getattr(ops, "fold_layernorm", False)) and c <= ops.LN_FOLD_MAX_C and (c % 160 == 0 or c % 128 == 0)

    @staticmethod
    def _ln_fold_pack(w, bias, gamma, beta, pack=None):
        """nn.LayerNorm(C) followed by nn.Linear W (attention.py:699-701, 732-747) as ONE GEMM on the un-normalised rows:
        LN(y) W^T = rstd (y W'^T - mean s) + t with W' = W diag(gamma), s_n = sum_k W'[n,k] (of the bf16-rounded W' the MMA
        multiplies), t_n = sum_k beta_k W[n,k] (+ bias_n). Returns (bf16 W', fp32 s, fp32 t), optionally row-permuted."""
        w = w.detach().to(F32)
        wp = (w * gamma.to(w.device)[None, :]).to(torch.bfloat16)
        s = wp.to(F32).sum(1)
        t = w @ beta.to(w.device)
        if bias is not None:
            t = t + bias.detach().to(F32)
        if pack is not None:
            wp, s, t = pack(wp), pack(s), pack(t)
        return wp.contiguous(), s.contiguous(), t.contiguous()

    def pack(self, unet_params: dict | None, cn_params: dict | None) -> None:
        """(Re)build packed weights from fp32 parameters keyed by the reference's state-dict names
        (ControlledUNetModel3D's own keys / ControlNet3D's keys, without prefixes). Either may be None."""
        cfg = self.cfg
        f = lambda t: t.detach().to(F32).contiguous()
        self.wu = self.wc = None
        self.generation = getattr(self, "generation", 0) + 1      # monotonically increasing: cache / graph signatures key on it
        if unet_params is not None:
            wu = self._pack_trunk(unet_params, self.plan_unet)
            wu.tag = "unet"
            wu["out.g"] = f(unet_params["out.0.weight"]); wu["out.bn"] = f(unet_params["out.0.bias"])
            # the 320 -> 4 output conv as a GEMM whose N is zero-padded to 8 (the narrowest the epilogue stores)
            w_out = unet_params["out.2.weight"].detach().to(F32)
            if w_out.shape[0] > OUT_NPAD:
                raise NotImplementedError(f"output conv with {w_out.shape[0]} > {OUT_NPAD} channels")
            n_pad = OUT_NPAD - w_out.shape[0]
            wu["out.w"] = self.ops.pack_matrix(_conv3_matrix(torch.nn.functional.pad(w_out, (0, 0, 0, 0, 0, 0, 0, n_pad))), 9)
            wu["out.b"] = torch.nn.functional.pad(f(unet_params["out.2.bias"]), (0, n_pad)).contiguous()
            self.wu = wu
        if cn_params is not None:
            wc = self._pack_trunk(cn_params, self.plan_cn)
            wc.tag = "controlnet"
            for i in range(len(HINT_STRIDES)):
                w = cn_params[f"input_hint_block.{2 * i}.weight"].detach()
                wc[f"hint{i}.w"] = _pack_direct(w, cin_pad=(w.shape[1] + 3) // 4 * 4)
                wc[f"hint{i}.b"] = f(cn_params[f"input_hint_block.{2 * i}.bias"])
            s = float(cfg.control_scales)
            names = [f"zero_convs.{i}.0" for i in range(len(self.plan_cn.skip_channels))] + ["middle_block_out.0"]
            for i, nm in enumerate(names):
                w = cn_params[nm + ".weight"].detach()
                wc[f"zc{i}.w"] = self.ops.pack_matrix(w.reshape(w.shape[0], w.shape[1]).to(F32) * s)
                wc[f"zc{i}.b"] = (cn_params[nm + ".bias"].detach().to(F32) * s).contiguous()
            self.wc = wc
        self.cond = {"guided": None, "kv": {}, "b": None}

    # ------------------------------------------------------------------------------------------ step-invariant
    def prepare_hint(self, hint_nchw: torch.Tensor, hint_repeat: int = 1) -> None:
        """BEV hint stem, once per sample (controlmodel.py:43-59,118). hint_nchw fp32
        [frames/hint_repeat, hint_channels, 8H, 8W]; under CFG both halves share the hint (hint_repeat=2)."""
        ops, wc = self.ops, self.wc
        dt = ops.act_dtype
        assert wc is not None, "pack() the ControlNet parameters first"
        Fh, Ch, Hh, Wh = hint_nchw.shape
        cin_pad = wc["hint0.w"].shape[1]
        h = torch.zeros((Fh, Hh, Wh, cin_pad), device=hint_nchw.device, dtype=F32)
        ops.nchw_to_nhwc(hint_nchw.to(F32).contiguous(), out=h, ch_off=0)
        n = len(HINT_STRIDES)
        for i, s in enumerate(HINT_STRIDES):
            cout = wc[f"hint{i}.b"].numel()
            last = i == n - 1
            h = ops.conv3x3_direct(h, wc[f"hint{i}.w"], wc[f"hint{i}.b"], cout, stride=s, silu=not last,
                                   out_dtype=F32 if last else dt)
        if hint_repeat > 1:
            h = h.repeat(hint_repeat, 1, 1, 1)
        old = self.cond["guided"]
        if old is not None and old.shape == h.shape and old.device == h.device:
            old.copy_(h)          # keep the buffer address stable: a captured CUDA graph stays valid across samples
        else:
            self.cond["guided"] = h

    def prepare_text(self, context: torch.Tensor) -> None:
        """K/V projections of the text context for every attn2 (attention.py:248-250), once per sample.
        context fp32 [b, L<=128, context_dim]."""
        ops = self.ops
        dt = ops.qkv_dtype
        b, L, D = context.shape
        ctx = self._to_operand(context.to(F32).contiguous().reshape(b * L, D))
        kv = self.cond["kv"]
        for W, plan in ((self.wu, self.plan_unet), (self.wc, self.plan_cn)):
            if W is None:
                continue
            for st in plan.stages():
                if st.kind != "stt":
                    continue
                for br in STT_BRANCHES:
                    t = f"{st.key}.transformer_blocks{br}.0"
                    old = kv.get((W.tag, t))
                    if old is not None and old.shape == (b, L, 2 * st.cin):
                        ops.gemm(ctx, W[t + ".kv2.w"], out_dtype=dt, out=old.view(b * L, 2 * st.cin))   # same address
                    else:
                        kv[(W.tag, t)] = ops.gemm(ctx, W[t + ".kv2.w"], out_dtype=dt).reshape(b, L, 2 * st.cin)
        self.cond["b"] = b

    def prepare_condition(self, hint_nchw: torch.Tensor, context: torch.Tensor, hint_repeat: int = 1) -> None:
        self.prepare_hint(hint_nchw, hint_repeat)
        self.prepare_text(context)

    # ------------------------------------------------------------------------------------------ blocks
    def _emb_vectors(self, W, t):
        """[frames, sum(Cout)] = Linear_i(SiLU(time_embed(t))) for every ResBlock i of the network, one launch
        (openaimodel.py:936-943 then :439-445, 520-523)."""
        ops = self.ops
        te = ops.timestep_embedding(t, self.cfg.model_channels)
        e = ops.linear_small(te, W["te0.w"], W["te0.b"], silu_out=True)
        # every consumer of `emb` is Sequential(SiLU, Linear) (openaimodel.py:439-445): the SiLU is applied ONCE, in the
        # epilogue of time_embed's second Linear — as `silu_in` of the big [sum(Cout), 1280] projection each of its 5,000
        # warps recomputed it for all 16 x 1280 inputs (2 MUFU each): 1.0 ms per step for two GEMVs
        e = ops.linear_small(e, W["te2.w"], W["te2.b"], silu_out=True)
        return ops.linear_small(e, W["emb.w"], W["emb.b"])

    def _res(self, W, st: Stage, x, embv):
        """ResBlock3D._forward (openaimodel.py:499-542)."""
        ops, k, T = self.ops, st.key, self.cfg.num_frames
        Fr, H, Wd, _ = x.shape
        b, P, C = Fr // T, H * Wd, st.cout
        need_skip = st.cin != st.cout
        a = ops.groupnorm(x, W[k + ".in_layers.0.g"], W[k + ".in_layers.0.b"], 1e-5, True, want_raw=need_skip)
        a, raw = a if need_skip else (a, None)
        h = ops.gemm(a, W[k + ".in.w"], bias=W[k + ".in.b"], taps=(3, 3))                     # [Fr,H,Wd,C] fp32
        tn = ops.groupnorm_pixel(h.view(b, T, P, C), W[k + ".in_layers_temporal.0.g"], W[k + ".in_layers_temporal.0.b"], 1e-5, True)
        off = W[k + ".emb_off"]
        # h = h + conv1d_T(...) + emb  (identity add :515 and timestep add :531 in one epilogue)
        h = ops.gemm(tn, W[k + ".int.w"], bias=W[k + ".int.b"], taps=(3, 1), residual=h, out=h,
                     rowvec=embv[:, off:off + C], rows_per_group=P, n_groups=Fr).view(Fr, H, Wd, C)
        a2 = ops.groupnorm(h, W[k + ".out_layers.0.g"], W[k + ".out_layers.0.b"], 1e-5, True)
        h2 = ops.gemm(a2, W[k + ".out.w"], bias=W[k + ".out.b"], taps=(3, 3))
        tn2 = ops.groupnorm_pixel(h2.view(b, T, P, C), W[k + ".out_layers_temporal.0.g"], W[k + ".out_layers_temporal.0.b"], 1e-5, True)
        if need_skip:
            h2 = ops.gemm(tn2, W[k + ".outt.w"], bias=W[k + ".outt.b"], taps=(3, 1), residual=h2, out=h2).view(Fr, H, Wd, C)
            return ops.gemm(raw, W[k + ".skip.w"], bias=W[k + ".skip.b"], residual=h2, out=h2).view(Fr, H, Wd, C)
        return ops.gemm(tn2, W[k + ".outt.w"], bias=W[k + ".outt.b"], taps=(3, 1), residual=h2, residual2=x, out=h2).view(Fr, H, Wd, C)

    def _transformer(self, W, t: str, y, heads, mode, geom, kv):
        """BasicTransformerBlock._forward (attention.py:726-747) on the token stream y [tokens, C] (ops.token_dtype).

        A folded block (W[t + ".fold"]) takes y = (stream, its row statistics from proj_in) and folds norm1 and norm2 into
        the GEMMs around the bf16 token stream: every GEMM that writes the stream also emits the per-row (sum, sum of
        squares) of what it stored, and the GEMM that consumes LN(stream) multiplies the un-normalised stream by
        W diag(gamma) and finishes the normalisation in its epilogue. No LayerNorm kernel, no normalised copy of the
        stream. norm3 stays a kernel: the GEGLU epilogue is the long pole of ff1 at level 0, a rank-1 correction there
        would lengthen it."""
        ops, dt = self.ops, self.ops.qkv_dtype
        Fr, H, Wd, C, b, T = geom
        fold = W[t + ".fold"]
        y, st = y if fold else (y, None)
        stats_out = {"ln_stats_out": True} if fold else {}

        def ln_gemm(stream, stats, norm, proj):
            """LN_norm(stream) W_proj^T: folded into the GEMM, or a LayerNorm kernel and then the GEMM"""
            if fold:
                return ops.gemm(stream, W[f"{t}.{proj}.w"], bias=W[f"{t}.{proj}.t"], out_dtype=dt, ln=(stats, W[f"{t}.{proj}.s"], 1e-5))
            return ops.gemm(ops.layernorm(stream, W[f"{t}.{norm}.g"], W[f"{t}.{norm}.b"]), W[f"{t}.{proj}.w"], out_dtype=dt)

        qkv = ln_gemm(y, st, "norm1", "qkv")
        if mode == "temporal":
            o = ops.attention_temporal(qkv.view(b, T, H * Wd, 3 * C), heads)
        else:
            V = self.cfg.num_views
            o = ops.attention_view(qkv.view(Fr, H, V, Wd // V, 3 * C), heads, mode == "cross", CROSS_VIEW_NEIGHBOURS)
        r = ops.gemm(o.view(-1, o.shape[-1]), W[t + ".attn1.o.w"], bias=W[t + ".attn1.o.b"], residual=y, out=y, out_dtype=y.dtype,
                     **stats_out)
        y, st = r if fold else (r, None)
        q = ln_gemm(y, st, "norm2", "q2")
        o = ops.attention_text(q.view(b, T * H * Wd, C), kv, heads)
        y = ops.gemm(o.view(-1, o.shape[-1]), W[t + ".attn2.o.w"], bias=W[t + ".attn2.o.b"], residual=y, out=y, out_dtype=y.dtype)
        n3 = ops.layernorm(y, W[t + ".norm3.g"], W[t + ".norm3.b"])
        ff = ops.gemm(n3, W[t + ".ff1.w"], bias=W[t + ".ff1.b"], geglu=True, out_dtype=ops.act_dtype)
        # the block's output is only ever consumed as the bf16 operand of proj_out: emit it in that form directly
        # (saves the fp32 write, the cast kernel's fp32 read and one launch per transformer block)
        if fold or ops.fused_operand_emit:
            return ops.gemm(ff, W[t + ".ff2.w"], bias=W[t + ".ff2.b"], residual=y, out_dtype=torch.bfloat16)
        return ops.gemm(ff, W[t + ".ff2.w"], bias=W[t + ".ff2.b"], residual=y, out=y, out_dtype=y.dtype)

    def _stt(self, W, st: Stage, x):
        """SpatialTemporalTransformer.forward (attention.py:1064-1134): intra-view, cross-view, temporal."""
        ops, k, T = self.ops, st.key, self.cfg.num_frames
        Fr, H, Wd, C = x.shape
        b = Fr // T
        geom = (Fr, H, Wd, C, b, T)
        for br, mode in zip(STT_BRANCHES, ("intra", "cross", "temporal")):
            a = ops.groupnorm(x, W[f"{k}.norm{br}.g"], W[f"{k}.norm{br}.b"], 1e-6, False)
            t = f"{k}.transformer_blocks{br}.0"
            fold = {"ln_stats_out": True} if W[t + ".fold"] else {}
            if mode == "temporal":
                pe = self._pos_table(T, C, x.device)
                y = ops.gemm(a.view(-1, a.shape[-1]), W[f"{k}.proj_in{br}.w"], bias=W[f"{k}.proj_in{br}.b"], rowvec=pe,
                             rows_per_group=H * Wd, n_groups=T, out_dtype=ops.token_dtype, **fold)
            else:
                y = ops.gemm(a.view(-1, a.shape[-1]), W[f"{k}.proj_in{br}.w"], bias=W[f"{k}.proj_in{br}.b"],
                             out_dtype=ops.token_dtype, **fold)
            y = self._transformer(W, t, y, st.heads, mode, geom, self.cond["kv"][(W.tag, t)])
            yb = self._to_operand(y) if y.dtype == F32 else y
            x = ops.gemm(yb, W[f"{k}.proj_out{br}.w"], bias=W[f"{k}.proj_out{br}.b"], residual=x, out=x).view(Fr, H, Wd, C)
        return x

    def _to_operand(self, y):
        return self.ops.cast_operand(y)

    def _pos_table(self, T, C, device):
        key = (T, C, str(device))
        cache = self.__dict__.setdefault("_pe_cache", {})
        if key not in cache:
            cache[key] = temporal_pos_table(T, C).to(device)
        return cache[key]

    def _run_block(self, W, blk, h, embv, guided=None):
        ops = self.ops
        for st in blk:
            if st.kind == "stem":
                h = ops.gemm(h, W[st.key + ".w"], bias=W[st.key + ".b"], taps=(3, 3), residual=guided)      # h: stem operand
            elif st.kind == "res":
                h = self._res(W, st, h, embv)
            elif st.kind == "stt":
                h = self._stt(W, st, h)
            elif st.kind == "down":
                cols, (Fr, Ho, Wo) = ops.im2col_s2(h)
                h = ops.gemm(cols, W[st.key + ".w"], bias=W[st.key + ".b"]).view(Fr, Ho, Wo, st.cout)
            elif st.kind == "up":
                u = ops.upsample2x(h)
                h = ops.gemm(u, W[st.key + ".w"], bias=W[st.key + ".b"], taps=(3, 3))
            else:
                raise ValueError(st.kind)
        return h

    # ------------------------------------------------------------------------------------------ networks
    def controlnet(self, x, t):
        """ControlNet3D.forward (controlmodel.py:86-142) on channels-last x [frames,H,W,in_channels] -> 13 residuals."""
        W, ops = self.wc, self.ops
        embv = self._emb_vectors(W, t)
        outs = []
        h = self.stem_operand(x)
        for i, blk in enumerate(self.plan_cn.encoder):
            h = self._run_block(W, blk, h, embv, guided=self.cond["guided"] if i == 0 else None)
            outs.append(ops.gemm(self._to_operand(h), W[f"zc{i}.w"], bias=W[f"zc{i}.b"]))
        h = self._run_block(W, self.plan_cn.middle, h, embv)
        i = len(self.plan_cn.encoder)
        outs.append(ops.gemm(self._to_operand(h), W[f"zc{i}.w"], bias=W[f"zc{i}.b"]))
        return outs

    def unet_encode(self, x, t):
        """Input blocks + middle block of ControlledUNetModel3D.forward (controlmodel.py:160-187): everything that does not
        need the ControlNet residuals. Returns (h, skips, emb vectors)."""
        W = self.wu
        embv = self._emb_vectors(W, t)
        hs = []
        h = self.stem_operand(x)
        for blk in self.plan_unet.encoder:
            h = self._run_block(W, blk, h, embv)
            hs.append(h)
        h = self._run_block(W, self.plan_unet.middle, h, embv)
        return h, hs, embv

    def unet_decode(self, enc, control):
        """`h += control.pop()`, the output blocks on cat([h, hs.pop() + control.pop()]) and the out head
        (controlmodel.py:188-202)."""
        W, ops = self.wu, self.ops
        h, hs, embv = enc
        control = list(control)
        h = ops.add_(h, control.pop().view(h.shape))
        for blk in self.plan_unet.decoder:
            skip = hs.pop()
            h = ops.concat_add(h, skip, control.pop().view(skip.shape))
            h = self._run_block(W, blk, h, embv)
        a = ops.groupnorm(h, W["out.g"], W["out.bn"], 1e-5, True)
        return ops.gemm(a, W["out.w"], bias=W["out.b"], taps=(3, 3))      # [frames,H,W,OUT_NPAD]: channels >= out_channels are 0

    def unet(self, x, t, control):
        """ControlledUNetModel3D.forward (controlmodel.py:160-202), channels-last x [frames,H,W,in_channels] (or the stem
        operand); returns eps [frames,H,W,OUT_NPAD] whose first out_channels channels are the prediction."""
        return self.unet_decode(self.unet_encode(x, t), control)

    def stem_operand(self, x):
        """fp32 channels-last network input [frames,H,W,in_channels] -> the MMA operand of the input conv: channels
        zero-padded to STEM_CPAD. A tensor that already has STEM_CPAD channels (the buffer eps() fills) is only cast."""
        if x.dtype != F32:
            return x                                     # already an operand
        if x.shape[-1] != STEM_CPAD:
            xp = torch.zeros((*x.shape[:-1], STEM_CPAD), device=x.device, dtype=F32)      # module-level entry points only
            xp[..., :x.shape[-1]] = x
            x = xp
        return self.ops.cast_operand(x)

    def eps(self, x_nchw, concat_nchw, t):
        """OpenAIWrapperControlLDM3D.forward (wrappers.py:37-70) with the step-invariant parts precomputed."""
        ops = self.ops
        assert self.cond is not None and self.cond["guided"] is not None and self.cond["kv"], "call prepare_condition() first"
        Fr, Cx, H, Wd = x_nchw.shape
        key = (Fr, H, Wd, str(x_nchw.device))
        if key not in self._xin:
            # channels in_channels..STEM_CPAD-1 stay zero for the life of the buffer. One buffer per input geometry, never
            # freed: a CUDA graph captured for an earlier geometry keeps replaying into ITS buffer
            self._xin[key] = torch.zeros((Fr, H, Wd, STEM_CPAD), device=x_nchw.device, dtype=F32)
        xin = self._xin[key]
        ops.nchw_to_nhwc(x_nchw, out=xin, ch_off=0)
        if concat_nchw is not None:
            ops.nchw_to_nhwc(concat_nchw, out=xin, ch_off=Cx)
        xin = ops.cast_operand(xin)                     # one operand for both input convs (ControlNet and UNet)
        if self.two_streams and xin.is_cuda:
            # The ControlNet and the UNet's own encoder + middle block only meet at the first skip join (controlmodel.py:
            # 176-195): they run on two streams (a fork / join pair of events, captured into the step's CUDA graph like
            # everything else). The big level-0/1 launches have many waves of tiles and fill all SMs either way; what
            # overlaps is the under-filled tail — level-2/3/mid GEMMs and attentions with fewer tiles than SMs, small
            # norms — and, since the GEMM kernel fits two CTAs per SM, a GEMM tile of one branch can share an SM with a
            # tile of the other.
            cur = torch.cuda.current_stream(xin.device)
            if self._side is None or self._side.device != xin.device:
                self._side = torch.cuda.Stream(device=xin.device)
            self._side.wait_stream(cur)
            with torch.cuda.stream(self._side):
                control = self.controlnet(xin, t)
            enc = self.unet_encode(xin, t)
            cur.wait_stream(self._side)
            e = self.unet_decode(enc, control)
        else:
            control = self.controlnet(xin, t)
            e = self.unet(xin, t, control)
        return ops.nhwc_to_nchw(e, channels=self.cfg.out_channels)
