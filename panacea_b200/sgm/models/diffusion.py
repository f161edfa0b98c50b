"""`DiffusionEngine3D` — the engine glue of the reference (sgm/models/diffusion.py:30-377) without Lightning: builds
network + wrapper, denoiser, sampler, conditioner and first stage from the `model.params` block of
configs/inference_nuscenes.yaml and runs the inference control flow `log_images -> sample -> decode_first_stage`
(SURVEY.md section 8f, row N1). Training, EMA, optimisers and logging of text images are not part of the inference
path and are not mirrored. The denoising loop inside `sample` is the hot path of this repository (sm_90a kernels)."""
from __future__ import annotations

import torch
import torch.nn as nn

from ..modules.diffusionmodules.sampling import BoundDenoiser
from ..modules.diffusionmodules.wrappers import OpenAIWrapperControlLDM3D
from ..modules.encoders.modules import FrozenOpenCLIPEmbedder, VAEEmbedder
from ..util import default, instantiate_from_config

UNCONDITIONAL_CONFIG = {"target": "sgm.modules.GeneralConditioner", "params": {"emb_models": []}}


def _params(cfg):
    return cfg.get("params", {}) if isinstance(cfg, dict) else cfg.params


class DiffusionEngine3D(nn.Module):
    def __init__(self, network_config, denoiser_config, first_stage_config, first_stage_config_2d=None, conditioner_config=None,
                 sampler_config=None, optimizer_config=None, scheduler_config=None, loss_fn_config=None, network_wrapper=None,
                 ckpt_path=None, vae_path=None, use_ema=False, ema_decay_rate=0.9999, scale_factor=1.0,
                 disable_first_stage_autocast=False, input_key="jpg", log_keys=None, no_cond_log=False, compile_model=False,
                 freeze_type="none", lr_rate=1.0, wrapper_type="OPENAIUNETWRAPPERCONTROLLDM3D", share_noise_level=0.0,
                 use_cuda_graph=True, precision=None):
        super().__init__()
        if use_ema:
            raise NotImplementedError("EMA weights are a training feature; the inference config sets use_ema: False")
        if wrapper_type != "OPENAIUNETWRAPPERCONTROLLDM3D" or network_wrapper is not None:
            raise NotImplementedError("only OpenAIWrapperControlLDM3D (the reference inference config) is implemented")
        self.share_noise_level = float(share_noise_level)
        self.alpha = _params(network_config).get("alpha", 1)                       # diffusion.py:65
        self.num_frames = _params(network_config)["num_frames"]                    # diffusion.py:79
        self.log_keys, self.input_key = log_keys, input_key
        model = instantiate_from_config(network_config)                            # diffusion.py:71
        if precision is not None:
            model.set_precision(precision)
        self.model = OpenAIWrapperControlLDM3D(model, compile_model=compile_model, use_cuda_graph=use_cuda_graph)
        self.denoiser = instantiate_from_config(denoiser_config)
        self.sampler = instantiate_from_config(sampler_config) if sampler_config is not None else None
        self.conditioner = instantiate_from_config(default(conditioner_config, UNCONDITIONAL_CONFIG))
        self.first_stage_model = instantiate_from_config(first_stage_config).eval()      # diffusion.py:124-130
        for p in self.first_stage_model.parameters():
            p.requires_grad = False
        if precision is not None:
            self.first_stage_model.set_precision(precision)                       # VAEEmbedder shares this model
        self.scale_factor = scale_factor
        self.disable_first_stage_autocast = disable_first_stage_autocast
        for emb in self.conditioner.embedders:                                     # diffusion.py:111-122 setup_vaeembedder
            if precision is not None and isinstance(emb, FrozenOpenCLIPEmbedder):
                emb.set_precision(precision)
            if isinstance(emb, VAEEmbedder):
                emb.first_stage_model = self.first_stage_model
                emb.disable_first_stage_autocast = disable_first_stage_autocast
                emb.scale_factor = scale_factor

    @property
    def device(self):
        return next(self.first_stage_model.parameters()).device

    def get_input(self, batch):
        return batch[self.input_key]

    @torch.no_grad()
    def decode_first_stage(self, z):
        return self.first_stage_model.decode(1.0 / self.scale_factor * z)          # diffusion.py:137-143

    @torch.no_grad()
    def encode_first_stage(self, x):
        return self.scale_factor * self.first_stage_model.encode(x)                # diffusion.py:145-150

    @torch.no_grad()
    def sample(self, cond, uc=None, batch_size=16, shape=None, randn=None, **kwargs):
        """diffusion.py:233-255. `randn` (optional) replaces the CPU-generator draw for tests."""
        if randn is None:
            randn = torch.randn(batch_size, *shape)                                 # CPU generator, like the reference (:242)
        randn = randn.to(self.device)
        if self.share_noise_level > 0.0:
            last = cond["concat"].to(self.device)[-1]
            randn = randn + last.unsqueeze(0).expand(self.num_frames, *last.shape).repeat(randn.shape[0] // self.num_frames, 1, 1, 1) \
                * self.share_noise_level
        return self.sampler(BoundDenoiser(self.denoiser, self.model), randn, cond, uc=uc)

    @torch.no_grad()
    def log_images(self, batch, N=8, sample=True, ucg_keys=None, **kwargs):
        """diffusion.py:300-377 for the SD-2.1 branch the config takes (unconditional prompt = ""), without the text/cond
        renderings (log_conditionings draws strings with PIL fonts — not part of the data path)."""
        log = {}
        x = self.get_input(batch)
        if "cond_img" in batch:
            log["cond_img"] = batch["cond_img"].reshape(-1, *batch["cond_img"].shape[2:]).contiguous()
        batch_uc = dict(batch)
        batch_uc["txt"] = ["" for _ in batch["txt"]]                                # diffusion.py:329-331
        c, uc = self.conditioner.get_unconditional_conditioning(batch, batch_uc=batch_uc, force_uc_zero_embeddings=[])
        N = min(x.shape[0], N)
        x = x.to(self.device)[:N]
        x = x.reshape(-1, *x.shape[2:]).contiguous()                                 # "b t c h w -> (b t) c h w"
        log["inputs"] = x
        z = self.encode_first_stage(x)
        log["reconstructions"] = self.decode_first_stage(z)
        if "cond_feat" in c:
            log["control"] = c["cond_feat"] * 2.0 - 1.0
        for k in c:                                                                  # diffusion.py:356-364
            if isinstance(c[k], torch.Tensor):
                if k in ("concat", "cond_bev_feat"):
                    c[k], uc[k] = (y[k][:N * self.num_frames].to(self.device) for y in (c, uc))
                elif k == "cond_feat":
                    c[k], uc[k] = (y[k][:N * self.num_frames * 4].to(self.device) for y in (c, uc))
                else:
                    c[k], uc[k] = (y[k][:N].to(self.device) for y in (c, uc))
        if sample:
            samples = self.sample(c, shape=z.shape[1:], uc=uc, batch_size=N * self.num_frames)
            log["samples"] = self.decode_first_stage(samples)
            log["sample_latents"] = samples
        return log
