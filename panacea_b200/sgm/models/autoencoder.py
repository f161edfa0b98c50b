"""First stage behind the reference's interface (sgm/models/autoencoder.py:333-373, `AutoencoderKLInferenceWrapper`).

* `decode(z)` — the KL autoencoder's DECODER (SURVEY.md section 8f, row N2) runs natively on the hot path's kernels
  (`panacea_b200.vae.VAEDecoderEngine`); parameters live under the reference's state-dict names (`decoder.*`,
  `post_quant_conv.*`), so an SD-2.1 VAE checkpoint loads unchanged (`load_state_dict(strict=False)`).
* `encode(x)` — the ENCODER (`quant_conv(Encoder(x))`, model.py:763-880) runs natively too
  (`panacea_b200.vae.VAEEncoderEngine`, `encoder.*` / `quant_conv.*` keys); the posterior is sampled like the reference
  (distributions.py:24-41: mean + exp(0.5 clamp(logvar, -30, 20)) * randn drawn on the CPU generator).
* `precision` ("bf16" | "parity", default env PN_PRECISION, else "bf16") selects the op set of both engines, as on the
  UNet: "parity" reproduces the reference's fp32 VAE (its config runs the first stage with autocast disabled).
* `frames_per_call` bounds how many frames one engine call holds (default: 2 in parity mode, all in bf16 mode). A
  full-size parity decode of 8 frames needs 50.7 GB at once, too much next to a parity UNet on an 80 GB card; split
  into calls of 2 frames it needs a quarter of that. The split is chosen so that the result is bitwise the unsplit one
  (`VAEDecoderEngine.frame_chunks`).
Without a checkpoint the parameters are random-init (BASELINE.json configs[3]: "random-init VAE/CLIP stubs")."""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ...vae import VAEDecoderEngine, VAEEncoderEngine, decoder_param_spec, encoder_param_spec


class AutoencoderKLInferenceWrapper(nn.Module):
    PARITY_FRAMES_PER_CALL = 2

    def __init__(self, embed_dim=4, ddconfig=None, lossconfig=None, monitor=None, seed: int = 1234, precision=None,
                 frames_per_call=None, **kwargs):
        super().__init__()
        dd = dict(ddconfig or {})
        dd.setdefault("ch", 128); dd.setdefault("ch_mult", [1, 2, 4, 4]); dd.setdefault("num_res_blocks", 2)
        dd.setdefault("z_channels", embed_dim); dd.setdefault("out_ch", 3); dd.setdefault("in_channels", 3)
        self.ddconfig, self.embed_dim = dd, embed_dim
        self.factor = 2 ** (len(dd["ch_mult"]) - 1)
        g = torch.Generator().manual_seed(seed)
        self._spec = {**decoder_param_spec(dd, embed_dim), **encoder_param_spec(dd, embed_dim)}
        self._attr = {k: "p__" + k.replace(".", "__") for k in self._spec}
        for k, shape in self._spec.items():
            p = torch.empty(shape)
            if k.endswith(".bias"):
                p.zero_()
            elif len(shape) == 1:
                p.fill_(1.0)
            else:
                p.copy_(torch.randn(shape, generator=g) * (1.0 / math.sqrt(math.prod(shape[1:]))))
            self.register_parameter(self._attr[k], nn.Parameter(p, requires_grad=False))
        self._version = 0
        self.frames_per_call = frames_per_call
        self.set_precision(precision)
        self.sample_posterior = True

    def set_precision(self, precision) -> None:
        """"bf16" or "parity" (None: env PN_PRECISION, else "bf16"); both engines are rebuilt and repacked on their next
        call (parity weights are packed split3)."""
        from ..modules.diffusionmodules.controlmodel import _resolve_precision
        self.precision = _resolve_precision(precision)
        self._engine = None
        self._enc_engine = None
        self._packed, self._enc_packed = -1, -1

    # --- reference key names
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        for k, a in self._attr.items():
            p = getattr(self, a)
            destination[prefix + k] = p if keep_vars else p.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        for k, a in self._attr.items():
            if prefix + k in state_dict:
                with torch.no_grad():
                    getattr(self, a).copy_(state_dict[prefix + k])
            else:
                missing_keys.append(prefix + k)
        self._version += 1

    def _apply(self, fn, recurse=True):
        r = super()._apply(fn, recurse)
        self._version += 1
        return r

    @property
    def post_quant_conv(self):                  # the reference reads `.post_quant_conv.weight.dtype` (diffusion.py:140)
        return type("PQ", (), {"weight": getattr(self, self._attr["post_quant_conv.weight"])})()

    def decoder_parameters(self) -> dict:
        return {k: getattr(self, a) for k, a in self._attr.items()}

    def _by_frames(self, eng, run, x):
        """run(x) over frame chunks of at most frames_per_call frames, bitwise equal to one call (eng.frame_chunks)."""
        limit = self.frames_per_call or (self.PARITY_FRAMES_PER_CALL if self.precision == "parity" else x.shape[0])
        chunks = eng.frame_chunks(x.shape[0], tuple(x.shape[2:]), limit)
        if len(chunks) == 1:
            return run(x)
        outs, i = [], 0
        for n in chunks:
            outs.append(run(x[i:i + n]))
            i += n
        return torch.cat(outs)

    @torch.no_grad()
    def encode_moments(self, x):
        if not x.is_cuda:
            raise RuntimeError("panacea_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        if self._enc_engine is None:
            from ..modules.diffusionmodules.controlmodel import _native_ops
            self._enc_engine = VAEEncoderEngine(self.ddconfig, _native_ops(self.precision), self.embed_dim)
        if self._enc_packed != self._version:
            self._enc_engine.pack(self.decoder_parameters())
            self._enc_packed = self._version
        return self._by_frames(self._enc_engine, self._enc_engine.encode_moments, x)

    @torch.no_grad()
    def encode(self, x):
        """autoencoder.py:352-357 + :366-368: a sample of the posterior N(mean, exp(logvar)) (distributions.py:24-41)."""
        mean, logvar = torch.chunk(self.encode_moments(x), 2, dim=1)
        if not self.sample_posterior:
            return mean.contiguous()
        std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
        return mean + std * torch.randn(mean.shape).to(mean.device)      # CPU generator draw, like the reference

    @torch.no_grad()
    def decode(self, z):
        """autoencoder.py:362-365 on the sm_90a kernels (no CPU path)."""
        if not z.is_cuda:
            raise RuntimeError("panacea_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        if self._engine is None:
            from ..modules.diffusionmodules.controlmodel import _native_ops
            self._engine = VAEDecoderEngine(self.ddconfig, _native_ops(self.precision), self.embed_dim)
        if self._packed != self._version:
            self._engine.pack(self.decoder_parameters())
            self._packed = self._version
        return self._by_frames(self._engine, self._engine.decode, z)
