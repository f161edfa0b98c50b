"""First stage behind the reference's interface (sgm/models/autoencoder.py:333-373, `AutoencoderKLInferenceWrapper`).

* `decode(z)` — the KL autoencoder's DECODER (SURVEY.md section 8f, row N2) runs natively on the hot path's kernels
  (`panacea_b200.vae.VAEDecoderEngine`); parameters live under the reference's state-dict names (`decoder.*`,
  `post_quant_conv.*`), so an SD-2.1 VAE checkpoint loads unchanged (`load_state_dict(strict=False)`).
* `encode(x)` — the ENCODER (`quant_conv(Encoder(x))`, model.py:763-880) runs natively too
  (`panacea_b200.vae.VAEEncoderEngine`, `encoder.*` / `quant_conv.*` keys); the posterior is sampled like the reference
  (distributions.py:24-41: mean + exp(0.5 clamp(logvar, -30, 20)) * randn drawn on the CPU generator).
Without a checkpoint the parameters are random-init (BASELINE.json configs[3]: "random-init VAE/CLIP stubs")."""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ...vae import VAEDecoderEngine, VAEEncoderEngine, decoder_param_spec, encoder_param_spec


class AutoencoderKLInferenceWrapper(nn.Module):
    def __init__(self, embed_dim=4, ddconfig=None, lossconfig=None, monitor=None, seed: int = 1234, **kwargs):
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
        self._engine = None
        self._enc_engine = None
        self._version, self._packed, self._enc_packed = 0, -1, -1
        self.sample_posterior = True

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

    @torch.no_grad()
    def encode_moments(self, x):
        if not x.is_cuda:
            raise RuntimeError("panacea_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        if self._enc_engine is None:
            from ...ops import NativeOps
            self._enc_engine = VAEEncoderEngine(self.ddconfig, NativeOps(), self.embed_dim)
        if self._enc_packed != self._version:
            self._enc_engine.pack(self.decoder_parameters())
            self._enc_packed = self._version
        return self._enc_engine.encode_moments(x)

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
            from ...ops import NativeOps
            self._engine = VAEDecoderEngine(self.ddconfig, NativeOps(), self.embed_dim)
        if self._packed != self._version:
            self._engine.pack(self.decoder_parameters())
            self._packed = self._version
        return self._engine.decode(z)
