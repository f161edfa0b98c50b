"""TEST INFRASTRUCTURE — pn_sampler_step (include/panacea_b200.h) restated in plain torch on top of the CPU op set
tests/torch_ref_ops.TorchRefOps, so the mirror samplers' host logic (per-evaluation scalars, buffer choreography,
noise draws) runs on the CPU; and the fp32 reference the GPU kernel tests compare with."""
from __future__ import annotations

import torch

from panacea_b200.ops import SAMPLER_DPM, SAMPLER_DPM_2M, SAMPLER_EULER, SAMPLER_HEUN, SAMPLER_LMS, SAMPLER_SCALE
from philox_ref import philox_normal
from torch_ref_ops import TorchRefOps

F32 = torch.float32


def sampler_step_torch(mode, x, net=None, *, x_eval=None, out=None, hist=None, noise=None, x_in_next=None, halves=2,
                       net_is_denoised=False, sigma_q=0.0, cfg_scale=1.0, sigma=0.0, dt=0.0, coef=(), hist_read=(),
                       hist_write=-1, noise_scale=1.0, noise_amp=0.0, seed=0, draw=0, c_in_next=0.0):
    """Same arguments and semantics as panacea_b200.ops.NativeOps.sampler_step, fp32 torch ops on x's device.
    Scalars are rounded to fp32 first, as the C struct does."""
    f = lambda v: torch.tensor(float(v), dtype=F32, device=x.device)
    n = x.numel()
    shape = x.shape
    xs = x.reshape(-1)
    c = [f(v) for v in coef] + [f(0.0)] * (4 - len(coef))
    slot = lambda s: hist.reshape(-1)[s * n:(s + 1) * n]
    if mode == SAMPLER_SCALE:
        o = xs * c[0]
    else:
        xe = xs if x_eval is None else x_eval.reshape(-1)
        nf = net.reshape(-1).float()
        den = nf[:n] if net_is_denoised else nf[:n] * (-f(sigma_q)) + xe
        if halves == 2:
            den_c = nf[n:] if net_is_denoised else nf[n:] * (-f(sigma_q)) + xe
            den = den + f(cfg_scale) * (den_c - den)
        if mode == SAMPLER_EULER:
            d = (xe - den) / f(sigma)
            o = xe + f(dt) * d
            new_hist = d
        elif mode == SAMPLER_HEUN:
            d_new = (xe - den) / f(sigma)
            o = xs + ((slot(hist_read[0]) + d_new) / 2.0) * f(dt)
            new_hist = None
        elif mode == SAMPLER_LMS:
            d = (xe - den) / f(sigma)
            acc = c[0] * d
            for j, r in enumerate(list(hist_read)[:3]):
                if r >= 0:
                    acc = acc + c[j + 1] * slot(r)
            o = xs + acc
            new_hist = d
        elif mode == SAMPLER_DPM:
            o = c[0] * xs - c[1] * den
            new_hist = den
        elif mode == SAMPLER_DPM_2M:
            den_d = c[2] * den - c[3] * slot(hist_read[0])
            o = c[0] * xs - c[1] * den_d
            new_hist = den
        else:
            raise ValueError(mode)
        if hist_write >= 0 and new_hist is not None:
            slot(hist_write).copy_(new_hist)
    if noise_amp != 0.0:
        xi = noise.reshape(-1) if noise is not None else torch.from_numpy(philox_normal(seed, draw, n)).to(x.device)
        o = o + xi * f(noise_scale) * f(noise_amp)
    dst = x if out is None else out
    dst.reshape(-1).copy_(o)
    if x_in_next is not None:
        v = o * f(c_in_next)
        x_in_next.reshape(-1).copy_(torch.cat([v] * halves))
    return dst.reshape(shape) if out is None else dst


class TorchSamplerRefOps(TorchRefOps):
    """TorchRefOps plus sampler_step."""

    @staticmethod
    def sampler_step(*args, **kwargs):
        return sampler_step_torch(*args, **kwargs)

