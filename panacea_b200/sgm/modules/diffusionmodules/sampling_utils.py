"""sampling_utils.py:7-48: the guidance combine and the solver helpers, restated for the host.

The samplers evaluate these once per schedule, before the loop, on fp32 CPU tensors with the reference's own
expressions (so the scalars they hand to pn_sampler_step are the values the reference's tensors hold); the per-element
arithmetic (to_d, the guidance combine) lives in pn_sampler_step."""
from __future__ import annotations

import torch


class NoDynamicThresholding:
    def __call__(self, uncond, cond, scale):
        return uncond + scale * (cond - uncond)


def linear_multistep_coeff(order, t, i, j, epsrel=1e-4):
    """sampling_utils.py:12-24: integral over [t_i, t_{i+1}] of the Lagrange basis polynomial of node i - j."""
    from scipy import integrate          # only LinearMultistepSampler needs scipy

    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")

    def fn(tau):
        prod = 1.0
        for k in range(order):
            if j == k:
                continue
            prod *= (tau - t[i - k]) / (t[i - j] - t[i - k])
        return prod

    return integrate.quad(fn, t[i], t[i + 1], epsrel=epsrel)[0]


def get_ancestral_step(sigma_from, sigma_to, eta=1.0):
    """sampling_utils.py:27-36 -> (sigma_down, sigma_up)."""
    if not eta:
        return sigma_to, 0.0
    sigma_up = torch.minimum(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


def to_d(x, sigma, denoised):
    """sampling_utils.py:39-40 (sigma a scalar or a tensor broadcastable against x)."""
    return (x - denoised) / sigma


def to_neg_log_sigma(sigma):
    return sigma.log().neg()


def to_sigma(neg_log_sigma):
    return neg_log_sigma.neg().exp()
