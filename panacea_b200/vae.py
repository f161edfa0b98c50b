"""VAE decoder and encoder on the hot path's own kernels (SURVEY.md section 8f, row N2): the steps right after / before
the denoising loop.

Executes the reference's `AutoencoderKL.decode` = `Decoder(post_quant_conv(z))`
(sgm/models/autoencoder.py:362-365; sgm/modules/diffusionmodules/model.py:882-1030: conv_in, mid = ResnetBlock /
AttnBlock / ResnetBlock, then per level 3 ResnetBlocks (+ nearest-2x Upsample + conv), GroupNorm(32, eps 1e-6) + swish
+ conv_out) on channels-last buffers over the 6-view panorama, with the kernels of the UNet path: `pn_gemm` for every
3x3 / 1x1 convolution (residual and shortcut adds in the epilogue), `pn_groupnorm_silu`, `pn_upsample2x`,
`pn_conv3x3_direct` for the 4-channel input and 3-channel output convs, and — for the single-head attention of the mid
block whose head_dim is the full channel count (512) — two GEMMs around `pn_softmax_rows_operand` per frame:
S = q k^T, P = softmax(S / sqrt(C)), O = P v (the value bias is added after the product: rows of P sum to one).
The op set decides the precision, as on the UNet: NativeOps gives bf16 operands with fp32 accumulation and residual
stream; ParityOps gives split-bf16 operands (fp32-class products), the reference's fp32 VAE to rtol 1e-3 / atol 1e-4.
Parameters are addressed by the reference's state-dict names (`decoder.*`, `post_quant_conv.*`), so SD-VAE checkpoints
load unchanged."""
from __future__ import annotations

import torch

from .engine import _conv3_matrix, _pack_direct

F32 = torch.float32


def decoder_param_spec(dd: dict, embed_dim: int = 4) -> dict:
    """Keys/shapes of `post_quant_conv` + `decoder.*` for a ddconfig (model.py:882-985)."""
    ch, ch_mult, nrb, zc, out_ch = dd["ch"], tuple(dd["ch_mult"]), dd["num_res_blocks"], dd["z_channels"], dd["out_ch"]
    if dd.get("attn_resolutions"):
        raise NotImplementedError("attn_resolutions must be empty (the SD-2.1 VAE of the reference config)")
    spec = {"post_quant_conv.weight": (zc, embed_dim, 1, 1), "post_quant_conv.bias": (zc,)}

    def conv(k, co, ci, ks):
        spec[k + ".weight"] = (co, ci, ks, ks)
        spec[k + ".bias"] = (co,)

    def norm(k, c):
        spec[k + ".weight"] = (c,)
        spec[k + ".bias"] = (c,)

    def res(k, ci, co):
        norm(k + ".norm1", ci); conv(k + ".conv1", co, ci, 3); norm(k + ".norm2", co); conv(k + ".conv2", co, co, 3)
        if ci != co:
            conv(k + ".nin_shortcut", co, ci, 1)

    block_in = ch * ch_mult[-1]
    conv("decoder.conv_in", block_in, zc, 3)
    res("decoder.mid.block_1", block_in, block_in)
    norm("decoder.mid.attn_1.norm", block_in)
    for n in ("q", "k", "v", "proj_out"):
        conv(f"decoder.mid.attn_1.{n}", block_in, block_in, 1)
    res("decoder.mid.block_2", block_in, block_in)
    for lvl in reversed(range(len(ch_mult))):
        block_out = ch * ch_mult[lvl]
        for i in range(nrb + 1):
            res(f"decoder.up.{lvl}.block.{i}", block_in, block_out)
            block_in = block_out
        if lvl != 0:
            conv(f"decoder.up.{lvl}.upsample.conv", block_in, block_in, 3)
    norm("decoder.norm_out", block_in)
    conv("decoder.conv_out", out_ch, block_in, 3)
    return spec


def encoder_param_spec(dd: dict, embed_dim: int = 4) -> dict:
    """Keys/shapes of `encoder.*` + `quant_conv` (model.py:763-853; autoencoder.py:352-353)."""
    ch, ch_mult, nrb, zc, cin = dd["ch"], tuple(dd["ch_mult"]), dd["num_res_blocks"], dd["z_channels"], dd["in_channels"]
    if dd.get("attn_resolutions") or not dd.get("double_z", True):
        raise NotImplementedError("attn_resolutions must be empty and double_z true (the SD-2.1 VAE of the reference config)")
    spec = {"quant_conv.weight": (2 * embed_dim, 2 * zc, 1, 1), "quant_conv.bias": (2 * embed_dim,)}

    def conv(k, co, ci, ks):
        spec[k + ".weight"] = (co, ci, ks, ks)
        spec[k + ".bias"] = (co,)

    def norm(k, c):
        spec[k + ".weight"] = (c,)
        spec[k + ".bias"] = (c,)

    def res(k, ci, co):
        norm(k + ".norm1", ci); conv(k + ".conv1", co, ci, 3); norm(k + ".norm2", co); conv(k + ".conv2", co, co, 3)
        if ci != co:
            conv(k + ".nin_shortcut", co, ci, 1)

    conv("encoder.conv_in", ch, cin, 3)
    in_mult = (1,) + ch_mult
    block_in = ch
    for lvl in range(len(ch_mult)):
        block_in, block_out = ch * in_mult[lvl], ch * ch_mult[lvl]
        for i in range(nrb):
            res(f"encoder.down.{lvl}.block.{i}", block_in, block_out)
            block_in = block_out
        if lvl != len(ch_mult) - 1:
            conv(f"encoder.down.{lvl}.downsample.conv", block_in, block_in, 3)
    res("encoder.mid.block_1", block_in, block_in)
    norm("encoder.mid.attn_1.norm", block_in)
    for n in ("q", "k", "v", "proj_out"):
        conv(f"encoder.mid.attn_1.{n}", block_in, block_in, 1)
    res("encoder.mid.block_2", block_in, block_in)
    norm("encoder.norm_out", block_in)
    conv("encoder.conv_out", 2 * zc, block_in, 3)
    return spec


class _VAEBlocks:
    """ResnetBlock / AttnBlock / packing shared by the decoder and encoder engines."""

    def _pack_common(self, P: dict, direct: tuple) -> dict:
        f = lambda t: t.detach().to(F32).contiguous()
        mat = self.ops.pack_matrix
        W = {}
        for k in self.spec:
            if k.endswith(".weight") and ".norm" in k:
                W[k[:-7] + ".g"], W[k[:-7] + ".b"] = f(P[k]), f(P[k[:-6] + "bias"])
        for k, shape in self.spec.items():
            if not k.endswith(".weight") or len(shape) != 4 or k in direct:
                continue
            base = k[:-7]
            W[base + ".w"] = mat(_conv3_matrix(P[k]), 9) if shape[2] == 3 else mat(P[k].detach().reshape(shape[0], shape[1]))
            W[base + ".b"] = f(P[base + ".bias"])
        return W

    @staticmethod
    def _pack_1x1_direct(w):
        """a 1x1 conv on few channels as the centre tap of the CUDA-core direct 3x3 conv"""
        w = w.detach().to(F32)
        w3 = torch.zeros(w.shape[0], w.shape[1], 3, 3, device=w.device)
        w3[:, :, 1, 1] = w[:, :, 0, 0]
        return _pack_direct(w3)

    def frame_chunks(self, frames: int, hw: tuple, max_frames: int) -> list:
        """Split `frames` into calls of at most `max_frames` frames that give bitwise the output of one call over all
        of them, or [frames] if there is no such split. Every op of the network is per frame: pn_gemm has no split-K
        and sums each row in the same order whatever the row count, the convs pad at frame edges, the attention loops
        over frames. The one exception is GroupNorm: pn_groupnorm_silu reduces each frame over `cpf` pixel ranges, and
        `cpf` depends on how many frames the call holds. A chunk size is allowed when it gives the same `cpf` as all
        frames for every (pixels, channels) the network normalises."""
        if frames <= max_frames:
            return [frames]
        shapes = self._gn_shapes(hw)
        cpf = self.ops.groupnorm_ctas_per_frame
        want = [cpf(frames, P, C) for P, C in shapes]
        ok = [c for c in range(max_frames, 0, -1) if all(cpf(c, P, C) == w for (P, C), w in zip(shapes, want))]
        best = {0: []}                                  # fewest calls that add up to n frames, allowed sizes only
        for n in range(1, frames + 1):
            cands = [best[n - c] + [c] for c in ok if c <= n and n - c in best]
            if cands:
                best[n] = min(cands, key=len)
        return best.get(frames, [frames])


class VAEDecoderEngine(_VAEBlocks):
    def __init__(self, ddconfig: dict, ops, embed_dim: int = 4):
        self.dd, self.ops, self.embed_dim = dict(ddconfig), ops, embed_dim
        self.spec = decoder_param_spec(self.dd, embed_dim)
        self.W = None

    # ------------------------------------------------------------------------------------------ packing
    def pack(self, P: dict) -> None:
        f = lambda t: t.detach().to(F32).contiguous()
        W = self._pack_common(P, ("post_quant_conv.weight", "decoder.conv_in.weight", "decoder.conv_out.weight"))
        W["pq.w"], W["pq.b"] = self._pack_1x1_direct(P["post_quant_conv.weight"]), f(P["post_quant_conv.bias"])
        W["in.w"], W["in.b"] = _pack_direct(P["decoder.conv_in.weight"].detach()), f(P["decoder.conv_in.bias"])
        W["out.w"], W["out.b"] = _pack_direct(P["decoder.conv_out.weight"].detach()), f(P["decoder.conv_out.bias"])
        self.W = W

    # ------------------------------------------------------------------------------------------ blocks
    def _res(self, k, x):
        """ResnetBlock.forward (model.py:175-196), temb = None, dropout 0."""
        ops, W = self.ops, self.W
        cin, cout = x.shape[-1], W[k + ".conv1.b"].numel()
        a = ops.groupnorm(x, W[k + ".norm1.g"], W[k + ".norm1.b"], 1e-6, True, want_raw=cin != cout)
        a, raw = a if cin != cout else (a, None)
        h = ops.gemm(a, W[k + ".conv1.w"], bias=W[k + ".conv1.b"], taps=(3, 3))
        a2 = ops.groupnorm(h, W[k + ".norm2.g"], W[k + ".norm2.b"], 1e-6, True)
        if cin != cout:
            x = ops.gemm(raw, W[k + ".nin_shortcut.w"], bias=W[k + ".nin_shortcut.b"]).view(*x.shape[:-1], cout)
        return ops.gemm(a2, W[k + ".conv2.w"], bias=W[k + ".conv2.b"], taps=(3, 3), residual=x).view(*x.shape[:-1], cout)

    def _attn(self, k, x):
        """AttnBlock.forward (model.py:395-414): single head over all H*W tokens of a frame, head_dim = C."""
        ops, W = self.ops, self.W
        Fr, H, Wd, C = x.shape
        P = H * Wd
        if P % 64 or C % 64:
            raise NotImplementedError("VAE mid attention needs H*W and C to be multiples of 64")
        if ops.operand_mult == 3:
            return self._attn_split3(k, x)
        a = ops.groupnorm(x, W[k + ".norm.g"], W[k + ".norm.b"], 1e-6, False).view(Fr, P, C)
        out = torch.empty_like(x)
        dt = a.dtype
        for f in range(Fr):
            af = a[f]
            q = ops.gemm(af, W[k + ".q.w"], bias=W[k + ".q.b"], out_dtype=dt)
            kk = ops.gemm(af, W[k + ".k.w"], bias=W[k + ".k.b"], out_dtype=dt)
            vT = ops.gemm(W[k + ".v.w"], af, out_dtype=dt)                     # [C, P] = W_v a^T (value bias added below)
            s = ops.gemm(q, kk)                                                # [P, P] fp32 scores
            p = ops.softmax_rows(s, C ** -0.5).to(dt)
            o = ops.gemm(p, vT, bias=W[k + ".v.b"], out_dtype=dt)              # rows of p sum to 1: + b_v after the product
            ops.gemm(o, W[k + ".proj_out.w"], bias=W[k + ".proj_out.b"], residual=x[f].reshape(P, C), out=out[f].view(P, C))
        return out

    def _attn_split3(self, k, x):
        """AttnBlock.forward in parity mode (split-bf16 operands, fp32-class products). Both factors of S = q k^T and of
        O = P v are activations, so one of each pair is cast to the weight form [hi | hi | lo] on the device; the
        other is in the A form [hi | lo | hi] that every producer writes."""
        ops, W = self.ops, self.W
        Fr, H, Wd, C = x.shape
        P = H * Wd
        a = ops.groupnorm(x, W[k + ".norm.g"], W[k + ".norm.b"], 1e-6, False).view(Fr, P, -1)
        out = torch.empty_like(x)
        for f in range(Fr):
            af = a[f]
            q = ops.gemm(af, W[k + ".q.w"], bias=W[k + ".q.b"])                  # fp32 [P, C]
            kk = ops.gemm(af, W[k + ".k.w"], bias=W[k + ".k.b"])
            v = ops.gemm(af, W[k + ".v.w"])                                     # value bias added after the product
            s = ops.gemm(ops.cast_operand(q), ops.cast_operand(kk, weight_form=True))      # [P, P] fp32 scores
            del q, kk
            p = ops.softmax_rows(s, C ** -0.5)                                  # split3 [P, 3P]
            del s
            vT = ops.nhwc_to_nchw(v.view(1, 1, P, C)).view(C, P)                # [C, P]
            o = ops.gemm(p, ops.cast_operand(vT, weight_form=True), bias=W[k + ".v.b"])     # rows of p sum to 1
            del p
            ops.gemm(ops.cast_operand(o), W[k + ".proj_out.w"], bias=W[k + ".proj_out.b"], residual=x[f].reshape(P, C),
                     out=out[f].view(P, C))
        return out

    def _gn_shapes(self, hw):
        """(pixels per frame, channels) of every GroupNorm of a decode from a latent of `hw` (decode() below)"""
        (h, w), ch, ch_mult, nrb = hw, self.dd["ch"], tuple(self.dd["ch_mult"]), self.dd["num_res_blocks"]
        block_in = ch * ch_mult[-1]
        shapes = {(h * w, block_in)}                                         # mid block
        for i, lvl in enumerate(reversed(range(len(ch_mult)))):
            P, block_out = (h << i) * (w << i), ch * ch_mult[lvl]
            shapes |= {(P, block_in), (P, block_out)}                        # norm1 of the first block, every other norm
            block_in = block_out
        return sorted(shapes)                                                # norm_out: (last P, ch * ch_mult[0]) is in it

    # ------------------------------------------------------------------------------------------ network
    @torch.no_grad()
    def decode(self, z_nchw: torch.Tensor) -> torch.Tensor:
        """z [F, z_channels, h, W] (already divided by scale_factor) -> image [F, out_ch, 8h, 8W]."""
        ops, W, dd = self.ops, self.W, self.dd
        assert W is not None, "pack() the decoder parameters first"
        ch_mult, nrb = tuple(dd["ch_mult"]), dd["num_res_blocks"]
        z = ops.nchw_to_nhwc(z_nchw.float().contiguous())
        z = ops.conv3x3_direct(z, W["pq.w"], W["pq.b"], dd["z_channels"])
        h = ops.conv3x3_direct(z, W["in.w"], W["in.b"], W["in.b"].numel())
        h = self._res("decoder.mid.block_1", h)
        h = self._attn("decoder.mid.attn_1", h)
        h = self._res("decoder.mid.block_2", h)
        for lvl in reversed(range(len(ch_mult))):
            for i in range(nrb + 1):
                h = self._res(f"decoder.up.{lvl}.block.{i}", h)
            if lvl != 0:
                u = ops.upsample2x(h)
                h = ops.gemm(u, W[f"decoder.up.{lvl}.upsample.conv.w"], bias=W[f"decoder.up.{lvl}.upsample.conv.b"], taps=(3, 3))
        a = ops.groupnorm(h, W["decoder.norm_out.g"], W["decoder.norm_out.b"], 1e-6, True, out_f32=ops.act_dtype == F32)
        img = ops.conv3x3_direct(a, W["out.w"], W["out.b"], dd["out_ch"])
        return ops.nhwc_to_nchw(img)


class VAEEncoderEngine(_VAEBlocks):
    """`quant_conv(Encoder(x))` (autoencoder.py:352-357; model.py:763-880): conv_in, per level 2 ResnetBlocks (+ Downsample
    = zero row/column appended at the far edges, then a stride-2 3x3 conv without padding), mid block, GroupNorm + swish +
    conv_out -> the posterior's moments [F, 2 z_channels, h/8, w/8]; sampling the posterior is the caller's one-liner."""
    _res = VAEDecoderEngine._res
    _attn = VAEDecoderEngine._attn
    _attn_split3 = VAEDecoderEngine._attn_split3

    def __init__(self, ddconfig: dict, ops, embed_dim: int = 4):
        self.dd, self.ops, self.embed_dim = dict(ddconfig), ops, embed_dim
        self.spec = encoder_param_spec(self.dd, embed_dim)
        self.W = None

    def pack(self, P: dict) -> None:
        f = lambda t: t.detach().to(F32).contiguous()
        W = self._pack_common(P, ("quant_conv.weight", "encoder.conv_in.weight"))
        cin = self.dd["in_channels"]
        W["in.w"], W["in.b"] = _pack_direct(P["encoder.conv_in.weight"].detach(), cin_pad=(cin + 3) // 4 * 4), f(P["encoder.conv_in.bias"])
        W["q.w"], W["q.b"] = self._pack_1x1_direct(P["quant_conv.weight"]), f(P["quant_conv.bias"])
        self.W = W

    def _gn_shapes(self, hw):
        """(pixels per frame, channels) of every GroupNorm of an encode of an image of `hw` (encode_moments() below;
        Downsample: (n - 2) // 2 + 1)"""
        (h, w), ch, ch_mult = hw, self.dd["ch"], tuple(self.dd["ch_mult"])
        shapes, block_in = set(), ch
        for lvl in range(len(ch_mult)):
            block_out = ch * ch_mult[lvl]
            shapes |= {(h * w, block_in), (h * w, block_out)}                # norm1 of the first block, every other norm
            block_in = block_out
            if lvl != len(ch_mult) - 1:
                h, w = (h - 2) // 2 + 1, (w - 2) // 2 + 1
        return sorted(shapes)                                                # mid block and norm_out: (last P, block_in)

    @torch.no_grad()
    def encode_moments(self, x_nchw: torch.Tensor) -> torch.Tensor:
        ops, W, dd = self.ops, self.W, self.dd
        assert W is not None, "pack() the encoder parameters first"
        ch_mult, nrb = tuple(dd["ch_mult"]), dd["num_res_blocks"]
        Fr, cin, H, Wd = x_nchw.shape
        xin = torch.zeros((Fr, H, Wd, W["in.w"].shape[1]), device=x_nchw.device, dtype=F32)     # channels padded to a multiple of 4
        ops.nchw_to_nhwc(x_nchw.float().contiguous(), out=xin, ch_off=0)
        h = ops.conv3x3_direct(xin, W["in.w"], W["in.b"], W["in.b"].numel())
        for lvl in range(len(ch_mult)):
            for i in range(nrb):
                h = self._res(f"encoder.down.{lvl}.block.{i}", h)
            if lvl != len(ch_mult) - 1:
                k = f"encoder.down.{lvl}.downsample.conv"
                cols, (f_, Ho, Wo) = ops.im2col_s2(h, pad=0)
                h = ops.gemm(cols, W[k + ".w"], bias=W[k + ".b"]).view(f_, Ho, Wo, -1)
        h = self._res("encoder.mid.block_1", h)
        h = self._attn("encoder.mid.attn_1", h)
        h = self._res("encoder.mid.block_2", h)
        a = ops.groupnorm(h, W["encoder.norm_out.g"], W["encoder.norm_out.b"], 1e-6, True)
        m = ops.gemm(a, W["encoder.conv_out.w"], bias=W["encoder.conv_out.b"], taps=(3, 3))
        m = ops.conv3x3_direct(m.view(*h.shape[:-1], -1), W["q.w"], W["q.b"], W["q.b"].numel())
        return ops.nhwc_to_nchw(m)
