"""Conditioner glue around the hot path (SURVEY.md section 8f, row N1): `GeneralConditioner`
(reference sgm/modules/encoders/modules.py:95-220) with the three embedders configs/inference_nuscenes.yaml:73-93 names.

The conditioner runs ONCE per sample, before the denoising loop; it only routes tensors (rearrange, cat, zeros for the
unconditional branch) and is therefore plain host/torch code, like the reference's. `FrozenOpenCLIPEmbedder` runs the
OpenCLIP ViT-H/14 text tower on the sm_90a kernels (panacea_b200.text_encoder) once text-tower weights are loaded;
without them it stays a deterministic stand-in that maps each prompt string to a reproducible [77, context_dim] tensor.
`VAEEmbedder` delegates to whatever first-stage model the engine hands it (the native VAE).
"""
from __future__ import annotations

import hashlib
from contextlib import nullcontext
from pathlib import Path

import torch
import torch.nn as nn

from ...util import instantiate_from_config


class AbstractEmbModel(nn.Module):
    """modules.py:51-92: carries is_trainable / ucg_rate / input_key."""

    def __init__(self):
        super().__init__()
        self.is_trainable = False
        self.ucg_rate = 0.0
        self.input_key = None
        self.legacy_ucg_val = None


class IdentityEncoder(AbstractEmbModel):
    """modules.py:244-249: the BEV control maps pass through unchanged (they become c["cond_feat"])."""

    def encode(self, x):
        return x

    def forward(self, x):
        return x


class FrozenOpenCLIPEmbedder(AbstractEmbModel):
    """modules.py:559-632: the OpenCLIP ViT-H/14 text tower, [b, 77, 1024] from the penultimate (or last) block.

    With text-tower weights the tower runs natively (`panacea_b200.text_encoder.TextEncoderEngine`, sm_90a kernels, no
    CPU path). Weights come from `version=<local open_clip file>` (.bin / .pt / .safetensors; `visual.*` ignored; a
    pretrained tag such as the default loads nothing) or from a state dict with `<prefix>model.*` keys, e.g. an engine
    checkpoint's `conditioner.embedders.0.model.*`. They appear in `state_dict()` under the same names. `forward` takes
    prompt strings (tokenized with the CLIP BPE vocabulary from `bpe_path=`, else open_clip's bundled copy) or an int64
    [b, 77] token tensor. `precision` ("bf16" | "parity", default env PN_PRECISION) selects the op set, as on the UNet.

    Without weights it is a deterministic stand-in: each prompt string maps to a reproducible randn [77, context_dim],
    so the conditional and unconditional ("") branches differ reproducibly on every rank."""
    LAYERS = ("last", "penultimate")
    FILE_SUFFIXES = (".bin", ".pt", ".pth", ".safetensors")

    def __init__(self, arch="ViT-H-14", version="laion2b_s32b_b79k", device="cuda", max_length=77, freeze=True,
                 layer="penultimate", always_return_pooled=False, legacy=True, context_dim=1024, bpe_path=None,
                 precision=None):
        super().__init__()
        if layer not in self.LAYERS:
            raise ValueError(f"layer must be one of {self.LAYERS}, got {layer!r}")
        self.max_length, self.context_dim = max_length, context_dim
        self.layer_idx = 1 if layer == "penultimate" else 0
        self.bpe_path = bpe_path
        self.register_buffer("_dev", torch.zeros(1), persistent=False)
        self._tower_keys = []                  # open_clip names of the loaded tower tensors (buffers "t__<name>")
        self._tokenizer = None
        self._engine = None
        self._version, self._packed = 0, -1
        self.set_precision(precision)
        if isinstance(version, str) and version.endswith(self.FILE_SUFFIXES):
            self._set_tower(_read_open_clip_file(version), source=version)

    # --- weights
    def set_precision(self, precision) -> None:
        """"bf16" or "parity"; the tower is repacked on the next call."""
        from ..diffusionmodules.controlmodel import _resolve_precision
        self.precision = _resolve_precision(precision)
        self._engine = None

    @property
    def has_tower(self) -> bool:
        return bool(self._tower_keys)

    def _tower_errors(self, sd: dict) -> list:
        from ....text_encoder import text_config_from_params, text_param_spec
        if "token_embedding.weight" not in sd or "positional_embedding" not in sd:
            return ["missing " + ", ".join(k for k in ("token_embedding.weight", "positional_embedding") if k not in sd)]
        cfg = text_config_from_params(sd)
        spec = text_param_spec(**cfg)
        missing = [k for k in spec if k not in sd]
        if missing:
            return [f"missing {len(missing)} keys: {', '.join(missing[:12])}{' ...' if len(missing) > 12 else ''}"]
        bad = [k for k, s in spec.items() if tuple(sd[k].shape) != s]
        if bad:
            return [f"misshaped: {', '.join(f'{k} {tuple(sd[k].shape)}' for k in bad[:6])}"]
        errs = []
        if cfg["width"] != self.context_dim:
            errs.append(f"tower width {cfg['width']} != context_dim {self.context_dim}")
        if cfg["ctx"] != self.max_length:
            errs.append(f"positional_embedding has {cfg['ctx']} positions, max_length is {self.max_length}")
        if cfg["width"] % 64:
            errs.append(f"tower width {cfg['width']} is not a multiple of head_dim 64")
        if cfg["layers"] <= self.layer_idx:
            errs.append(f"{cfg['layers']} blocks cannot serve layer_idx {self.layer_idx}")
        return errs

    def _set_tower(self, sd: dict, source: str) -> None:
        sd = {k: v for k, v in sd.items() if not k.startswith("visual.")}
        errs = self._tower_errors(sd)
        if errs:
            raise ValueError(f"FrozenOpenCLIPEmbedder: text tower from {source}: " + "; ".join(errs))
        for k in self._tower_keys:
            delattr(self, "t__" + k.replace(".", "__"))
        self._tower_keys = sorted(sd)
        for k in self._tower_keys:
            self.register_buffer("t__" + k.replace(".", "__"), sd[k].detach().clone().to(self._dev.device), persistent=False)
        self._version += 1

    def tower_parameters(self) -> dict:
        return {k: getattr(self, "t__" + k.replace(".", "__")) for k in self._tower_keys}

    def _save_to_state_dict(self, destination, prefix, keep_vars):
        for k, v in self.tower_parameters().items():
            destination[prefix + "model." + k] = v

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        p = prefix + "model."
        sd = {k[len(p):]: v for k, v in state_dict.items() if k.startswith(p)}
        if not sd:
            return                              # no tower in this state dict: the embedder keeps what it has
        sd = {k: v for k, v in sd.items() if not k.startswith("visual.")}
        errs = self._tower_errors(sd)
        if errs:
            error_msgs.append(f"text tower under {p}*: " + "; ".join(errs))
            return
        self._set_tower(sd, source=p + "*")

    def _apply(self, fn, recurse=True):
        r = super()._apply(fn, recurse)
        self._version += 1
        return r

    # --- forward
    def tokenize(self, text) -> torch.Tensor:
        if self._tokenizer is None:
            from ....clip_tokenizer import ClipTokenizer
            self._tokenizer = ClipTokenizer(self.bpe_path)
        return self._tokenizer.tokenize(list(text), self.max_length)

    def engine(self):
        from ....text_encoder import TextEncoderEngine
        if self._engine is None:
            from ..diffusionmodules.controlmodel import _native_ops
            self._engine = TextEncoderEngine(_native_ops(self.precision))
            self._packed = -1
        if self._packed != self._version:
            self._engine.pack(self.tower_parameters())
            self._packed = self._version
        return self._engine

    def encode(self, text):
        return self(text)

    @torch.no_grad()
    def forward(self, text):
        if not self.has_tower:
            return self._stand_in(text)
        dev = self._dev.device
        if dev.type != "cuda":
            raise RuntimeError("panacea_b200 runs on CUDA (sm_90a) only; the text tower has no CPU path (call .cuda())")
        if isinstance(text, torch.Tensor):
            if text.dtype != torch.int64 or text.dim() != 2 or text.shape[1] != self.max_length:
                raise ValueError(f"token tensor must be int64 [b, {self.max_length}], got {text.dtype} {tuple(text.shape)}")
            tokens = text
        else:
            tokens = self.tokenize(text)
        return self.engine().encode(tokens.to(dev), self.layer_idx)

    def _stand_in(self, text):
        outs = []
        for s in text:
            seed = int.from_bytes(hashlib.sha256(str(s).encode()).digest()[:8], "little") % (2 ** 63)
            g = torch.Generator().manual_seed(seed)
            outs.append(torch.randn(self.max_length, self.context_dim, generator=g))
        return torch.stack(outs).to(self._dev.device)


def _read_open_clip_file(path: str) -> dict:
    """A stock open_clip weights file (the reference's commented-out local-file alternative, modules.py:580-583)."""
    if not Path(path).is_file():
        raise FileNotFoundError(f"FrozenOpenCLIPEmbedder: version={path!r} names a weights file that does not exist")
    if path.endswith(".safetensors"):
        from safetensors.torch import load_file
        sd = load_file(path)
    else:
        sd = torch.load(path, map_location="cpu", weights_only=True)
        sd = sd.get("state_dict", sd)
    return {k[len("module."):] if k.startswith("module.") else k: v for k, v in sd.items()}


class VAEEmbedder(AbstractEmbModel):
    """modules.py:1000-1055: encodes the image-condition frames with the engine's first stage and scales the latent
    (the engine injects first_stage_model / scale_factor / disable_first_stage_autocast, diffusion.py:111-122)."""

    def __init__(self, down_blur_factor: int = 1):
        super().__init__()
        if down_blur_factor != 1:
            raise NotImplementedError("down_blur_factor > 1 is not used by the reference config")
        self.first_stage_model = None
        self.scale_factor = None

    def freeze(self):
        return self

    def encode(self, x):
        return self(x)

    @torch.no_grad()
    def forward(self, x):
        assert self.first_stage_model is not None and self.scale_factor is not None, "first_stage_model / scale_factor not set"
        return self.scale_factor * self.first_stage_model.encode(x)


class GeneralConditioner(nn.Module):
    """modules.py:95-220, same routing rules: output key by tensor rank (2 vector, 3 crossattn, 4/5 concat), the
    `cond_img` embedder feeds "cond_feat", [b t c h w] inputs are flattened to (b t), equal keys are concatenated,
    `force_zero_embeddings` zeroes an embedder's output for the unconditional branch."""
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1}

    def __init__(self, emb_models):
        super().__init__()
        embedders = []
        for embconfig in emb_models:
            embedder = instantiate_from_config(embconfig)
            assert isinstance(embedder, AbstractEmbModel), f"{type(embedder).__name__} has to inherit from AbstractEmbModel"
            embedder.is_trainable = embconfig.get("is_trainable", False)
            embedder.ucg_rate = embconfig.get("ucg_rate", 0.0)
            if "input_key" in embconfig:
                embedder.input_key = embconfig["input_key"]
            elif "input_keys" in embconfig:
                embedder.input_keys = embconfig["input_keys"]
            else:
                raise KeyError(f"need either 'input_key' or 'input_keys' for embedder {type(embedder).__name__}")
            embedder.legacy_ucg_val = embconfig.get("legacy_ucg_value", None)
            if embedder.legacy_ucg_val is not None:
                raise NotImplementedError("legacy_ucg_value (training-time dropout) is not part of the inference path")
            embedders.append(embedder.eval())
        self.embedders = nn.ModuleList(embedders)

    def forward(self, batch: dict, force_zero_embeddings=None) -> dict:
        output = {}
        force_zero_embeddings = force_zero_embeddings or []
        for embedder in self.embedders:
            with (nullcontext() if embedder.is_trainable else torch.no_grad()):
                if getattr(embedder, "input_key", None) is not None:
                    x = batch[embedder.input_key]
                    if embedder.input_key in ("final_cond_zero", "cond_img"):      # modules.py:157-166
                        x = x.reshape(-1, *x.shape[2:]).contiguous()               # "b t c h w -> (b t) c h w"
                    emb_out = embedder(x)
                else:
                    emb_out = embedder(*[batch[k] for k in embedder.input_keys])
            if not isinstance(emb_out, (list, tuple)):
                emb_out = [emb_out]
            for emb in emb_out:
                out_key = "cond_feat" if getattr(embedder, "input_key", None) == "cond_img" else self.OUTPUT_DIM2KEYS[emb.dim()]
                if embedder.ucg_rate > 0.0:                                         # modules.py:184-195 (training-time dropout)
                    keep = torch.bernoulli((1.0 - embedder.ucg_rate) * torch.ones(emb.shape[0], device=emb.device))
                    emb = keep.reshape(-1, *([1] * (emb.dim() - 1))) * emb
                if getattr(embedder, "input_key", None) in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                if out_key in output:
                    output[out_key] = torch.cat((output[out_key], emb), self.KEY2CATDIM[out_key])
                else:
                    output[out_key] = emb
        return output

    def get_unconditional_conditioning(self, batch_c, batch_uc=None, force_uc_zero_embeddings=None):
        """modules.py:204-219: ucg dropout disabled for both passes."""
        rates = [e.ucg_rate for e in self.embedders]
        for e in self.embedders:
            e.ucg_rate = 0.0
        c = self(batch_c)
        uc = self(batch_c if batch_uc is None else batch_uc, force_uc_zero_embeddings or [])
        for e, r in zip(self.embedders, rates):
            e.ucg_rate = r
        return c, uc
