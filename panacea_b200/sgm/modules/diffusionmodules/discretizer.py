"""discretizer.py:11-69 LegacyDDPMDiscretization, restated with numpy on the host (float64 schedule, fp32 sigmas)."""
from __future__ import annotations

import numpy as np
import torch


def generate_roughly_equally_spaced_steps(num_substeps: int, max_step: int) -> np.ndarray:
    return np.linspace(max_step - 1, 0, num_substeps, endpoint=False).astype(int)[::-1]


def img2img_sigmas(sigmas: torch.Tensor, strength: float) -> torch.Tensor:
    """The tail a denoise from `strength` runs over (upstream sgm.inference.helpers.Img2ImgDiscretizationWrapper): of
    the n + 1 sigmas, trailing 0 included, the last k = int(strength (n + 1)). strength 1 keeps them all."""
    strength = float(strength)
    if not 0.0 < strength <= 1.0:
        raise ValueError(f"strength must lie in (0, 1], got {strength}")
    k = int(strength * len(sigmas))
    if k < 2:
        raise ValueError(f"strength {strength} keeps {k} of {len(sigmas)} sigmas; a denoise needs at least one step (2)")
    return sigmas[len(sigmas) - k:]


class LegacyDDPMDiscretization:
    def __init__(self, linear_start=0.00085, linear_end=0.0120, num_timesteps=1000):
        self.num_timesteps = num_timesteps
        betas = np.linspace(linear_start ** 0.5, linear_end ** 0.5, num_timesteps, dtype=np.float64) ** 2
        self.alphas_cumprod = np.cumprod(1.0 - betas, axis=0)

    def get_sigmas(self, n, device="cpu"):
        if n < self.num_timesteps:
            ac = self.alphas_cumprod[generate_roughly_equally_spaced_steps(n, self.num_timesteps)]
        elif n == self.num_timesteps:
            ac = self.alphas_cumprod
        else:
            raise ValueError(n)
        sig = torch.tensor((1 - ac) / ac, dtype=torch.float32, device=device) ** 0.5
        return torch.flip(sig, (0,))

    def __call__(self, n, do_append_zero=True, device="cpu", flip=False):
        sig = self.get_sigmas(n, device=device)
        if do_append_zero:
            sig = torch.cat([sig, sig.new_zeros([1])])
        return sig if not flip else torch.flip(sig, (0,))
