"""`DiffusionEngine3D` — the engine glue of the reference (sgm/models/diffusion.py:30-377) without Lightning: builds
network + wrapper, denoiser, sampler, conditioner and first stage from the `model.params` block of
configs/inference_nuscenes.yaml and runs the inference control flow `log_images -> sample -> decode_first_stage`
(SURVEY.md section 8f, row N1); every clip, generated, edited or outpainted, goes through `_sample_clip`. Training, EMA,
optimisers and logging of text images are not part of the inference path and are not mirrored. The denoising loop
inside the sampler call is the hot path of this repository (sm_90a kernels)."""
from __future__ import annotations

import torch
import torch.nn as nn

from ...composite import composite_frames
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

    def _initial_noise(self, cond, batch_size, shape):
        randn = torch.randn(batch_size, *shape).to(self.device)                    # CPU generator, like the reference (:242)
        if self.share_noise_level > 0.0:
            last = cond["concat"].to(self.device)[-1]
            randn = randn + last.unsqueeze(0).expand(self.num_frames, *last.shape).repeat(randn.shape[0] // self.num_frames, 1, 1, 1) \
                * self.share_noise_level
        return randn

    @torch.no_grad()
    def log_images(self, batch, N=8, sample=True, ucg_keys=None, **kwargs):
        """diffusion.py:300-377 for the SD-2.1 branch the config takes (unconditional prompt = ""), without the text/cond
        renderings (log_conditionings draws strings with PIL fonts — not part of the data path)."""
        if not sample:
            return self._log_inputs(batch, N)[0]
        return self._sample_clip(batch, N)

    def _sample_clip(self, batch, N, strength=1.0, known=None, mask=None, edit_sigma=None):
        """The path of every clip: _log_inputs, the start latent, one sampler call (diffusion.py:233-255 `sample`),
        decode. The start latent is the initial noise eps, or with `edit_sigma` = sigma the encoded clip z0 noised to
        sigma and scaled for the sampler's first launch, (z0 + sigma eps) / sqrt(1 + sigma^2); an edit's `mask` is then
        reshaped to [N T, h, w] and keeps `known` = z0 where it is 0. Returns the log with "samples" and
        "sample_latents", and for an edit "edit_mask" (all ones without a mask)."""
        log, c, uc, N, latent_shape, z = self._log_inputs(batch, N)
        x = self._initial_noise(c, N * self.num_frames, latent_shape)
        if edit_sigma is not None:
            x = (z + edit_sigma * x) / (1.0 + edit_sigma ** 2) ** 0.5
            if mask is not None:
                known, mask = z, mask.to(self.device, torch.float32).reshape(z.shape[0], *z.shape[2:])
        samples = self.sampler(BoundDenoiser(self.denoiser, self.model), x, c, uc=uc, strength=strength, known=known, mask=mask)
        log["samples"] = self.decode_first_stage(samples)
        log["sample_latents"] = samples
        if edit_sigma is not None:
            log["edit_mask"] = torch.ones(z.shape[0], *z.shape[2:], device=z.device) if mask is None else mask
        return log

    def _log_inputs(self, batch, N):
        """log_images up to the sampler: (log, c, uc, N, latent shape, z = the encoded ground truth or None)."""
        log, z = {}, None
        if "cond_img" in batch:
            log["cond_img"] = batch["cond_img"].reshape(-1, *batch["cond_img"].shape[2:]).contiguous()
        batch_uc = dict(batch)
        batch_uc["txt"] = ["" for _ in batch["txt"]]                                # diffusion.py:329-331
        c, uc = self.conditioner.get_unconditional_conditioning(batch, batch_uc=batch_uc, force_uc_zero_embeddings=[])
        if self.input_key in batch:
            x = self.get_input(batch)
            N = min(x.shape[0], N)
            x = x.to(self.device)[:N]
            x = x.reshape(-1, *x.shape[2:]).contiguous()                             # "b t c h w -> (b t) c h w"
            log["inputs"] = x
            z = self.encode_first_stage(x)
            log["reconstructions"] = self.decode_first_stage(z)
            latent_shape = z.shape[1:]
        else:
            # no ground truth (the clips k > 0 of a scene): the latent shape comes from the image condition
            if "concat" not in c:
                raise KeyError(f"batch has no {self.input_key!r} and the conditioner produces no 'concat' to take the latent shape from")
            N = min(c["concat"].shape[0] // self.num_frames, N)
            latent_shape = c["concat"].shape[1:]
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
        return log, c, uc, N, latent_shape, z

    @torch.no_grad()
    def edit_images(self, batch, strength, mask=None, N=8, composite=None):
        """log_images for a recorded clip (DESIGN.md section 13): the sampler starts from the clip's own latent z0 =
        encode(batch["jpg"]) noised to the first sigma of the strength's schedule, z0 + sigma_start eps (eps drawn as
        `sample` draws it), handed over as (z0 + sigma_start eps) / sqrt(1 + sigma_start^2) since the sampler's first
        launch scales by sqrt(1 + sigma_0^2) (upstream's do_img2img). `mask` [N T, h, w] in [0, 1] (None: no blending)
        regenerates only where it is > 0: elsewhere every step's result is the known latent z0 noised to its level, and
        the final latent is z0 where mask = 0. Returns the log_images keys plus "edit_mask".

        `composite` = F pastes the recorded pixels back outside the regenerated cells with a feather of F pixels
        (panacea_b200/composite.py): "samples" becomes the composite, "decoded_samples" the plain decode and
        "composite_alpha" [N T, H, 6w] the weight of the decode. It draws nothing from any generator, and needs a mask."""
        if self.input_key not in batch:
            raise KeyError(f"edit_images needs the recorded frames in batch[{self.input_key!r}]")
        if composite is not None and mask is None:
            raise ValueError("composite pastes the recorded pixels back outside a mask: an edit without one regenerates "
                             "every cell, so there is nothing to paste")
        sigma = float(self.sampler.sigmas(strength=strength)[0])                  # rejects a bad strength first
        log = self._sample_clip(batch, N, strength, mask=mask, edit_sigma=sigma)
        if composite is not None:
            log["decoded_samples"] = log["samples"]
            log["samples"], log["composite_alpha"] = composite_frames(log["decoded_samples"], log["inputs"], log["edit_mask"],
                                                                      composite)
        return log

    def _image_condition_key(self) -> str:
        keys = [e.input_key for e in self.conditioner.embedders if isinstance(e, VAEEmbedder)]
        if len(keys) != 1:
            raise ValueError(f"a scene needs exactly one VAEEmbedder image condition in the conditioner, found {len(keys)}")
        return keys[0]

    @torch.no_grad()
    def outpaint_images(self, batch, known, mask, N=8, **kwargs):
        """log_images with part of the clip given (DESIGN.md section 11): the conditioning, the initial noise and the
        full-strength schedule of `log_images`, with `known` [N T, 4, h, w] kept where `mask` [N T, h, w] is 0 (the
        sampler blends every step's result toward known + sigma xi there, so the final latent is `known` exactly) and
        generated where it is 1. The known region's Philox seed is drawn from the CPU generator after the churn seed.
        Other `log_images` keywords are accepted and ignored, as `log_images` ignores its own."""
        return self._sample_clip(batch, N, known=known, mask=mask)

    @torch.no_grad()
    def sample_scene(self, batches, use_last_frame=True, overlap=None, **kwargs):
        """A scene of K = len(batches) clips chained through their boundary frame, or through `overlap` = m shared
        frames (panacea_b200/scene.py).

        `batches[k]` is clip k's layout batch as `MyDataset.__getitem__` + the DataLoader give it (one sequence):
        `cond_img`, `txt`, `filenames`; clip 0 also carries the ground truth and its real image condition. Tensors may
        stay on the host: each clip's are moved to the device when that clip runs. Clip k > 0 is
        conditioned on the frame of clip k-1 that lands on its conditioning index a (a = T-1 with `use_last_frame`,
        else 0; `scene.handoff_index`), quantised like the writers and read back like the dataset, in a
        `final_cond_zero` that is zero elsewhere; it goes through the conditioner and the VAE embedder unchanged.

        `overlap` None: each clip is one `log_images` call, in clip order, so the CPU generator is drawn as K successive
        calls draw it, and K = 1 is exactly `log_images`; clip k > 0 regenerates the boundary frame and the scene keeps
        clip k-1's copy. `overlap` m in 1 .. T-1: clip 0 is one `log_images` call and clip k > 0 one `outpaint_images`
        call, which keeps clip k-1's final latents of the m shared frames (`scene.known_region`) and generates the other
        T-m; the shared latents, and so their decoded frames, come out equal to clip k-1's. Per carrying clip the CPU
        generator gives the initial noise, then the churn seed (noisy samplers only), then the known region's seed, as
        `edit_images` draws them; so the draws of clips k > 1 differ from the same scene with `overlap` None.

        The wrapper replays the one CUDA graph of clip 0 (the conditioning is re-prepared into the same buffers). A
        clip's decoded frames and latent move to the host before the next clip starts, and the latent comes back to
        the device only as the next clip's known region, so the device peak of a scene is that of one clip.

        Returns a dict (all tensors on the host): "samples" the scene [K(T-m)+m, 3, H, W] in chronological order (m = 1
        for `overlap` None), "sample_latents" the K per-clip latents [T, 4, h, w], "handoff_frames" the K-1 dequantised
        frames [3, H, W] that conditioned clips 1..K-1, "clip_samples" the K decoded clips [T, 3, H, W], "overlap", and
        "filenames" in scene order when the batches carry them."""
        from ... import scene as S
        T = self.num_frames
        S.check_overlap(overlap, T)
        key = self._image_condition_key() if len(batches) > 1 else None
        clips, latents, handoffs = [], [], []
        for k, batch in enumerate(batches):
            batch = {n: v.to(self.device) if isinstance(v, torch.Tensor) else v for n, v in batch.items()}   # one clip at a time
            if k > 0:
                cond = S.condition_from_frame(handoffs[-1], T, use_last_frame)
                batch = {n: v for n, v in batch.items() if n != self.input_key}
                batch[key] = cond.unsqueeze(0).to(self.device)
            if k > 0 and overlap is not None:
                known, mask = S.known_region(latents[-1].to(self.device), use_last_frame, overlap)
                log = self.outpaint_images(batch, known, mask, **kwargs)
                del known, mask
            else:
                log = self.log_images(batch, **kwargs)
            if log["samples"].shape[0] != T:
                raise ValueError(f"a scene clip is one sequence of {T} frames; clip {k} decoded {log['samples'].shape[0]}")
            clips.append(log["samples"].cpu())
            latents.append(log["sample_latents"].cpu())
            del log                                                         # the clip's device tensors go before the next clip
            if k + 1 < len(batches):
                handoffs.append(S.quantize_frame(clips[-1][S.handoff_index(T, use_last_frame, overlap)]))
        out = {"samples": S.scene_order(clips, use_last_frame, overlap), "sample_latents": latents,
               "handoff_frames": handoffs, "clip_samples": clips, "overlap": overlap}
        if all("filenames" in b for b in batches):
            out["filenames"] = S.scene_order([b["filenames"] for b in batches], use_last_frame, overlap)
        return out
