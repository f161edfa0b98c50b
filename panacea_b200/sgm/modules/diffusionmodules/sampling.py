"""sampling.py:24-365: the reference's samplers — EulerEDMSampler / EDMSampler (with stochastic churn), HeunEDMSampler,
EulerAncestralSampler, DPMPP2SAncestralSampler, DPMPP2MSampler and LinearMultistepSampler — around the DiscreteDenoiser
and VanillaCFG / IdentityGuider. The reference config uses EulerEDMSampler with s_churn = 0 and VanillaCFG ("DDIM
(eta=0)", configs/inference_nuscenes.yaml:115-126); the others are one `sampler_config.target` away.

Every scalar of the loop — sigma, quantised sigma, timestep index and c_in of every network evaluation (second stages
at off-schedule sigmas included), the churn amplitudes, get_ancestral_step, the DPM++ multipliers, the LMS coefficients
— is computed on the host before the loop, with the reference's own fp32 tensor expressions. Per evaluation the device
then executes one network evaluation (ControlNet + UNet, optionally one CUDA graph replay) and ONE pn_sampler_step launch
that applies the denoiser scalings, the guidance combine, the solver update, the noise and the next network input's
scaling + batch doubling. The reference's per-step torch.cat / dict rebuild (guiders.py:31-40) happens once per sample.

Noise (churn, ancestral): by default a counter-based Philox4x32-10 stream generated inside pn_sampler_step, keyed by a
seed drawn once per sample from torch's default CPU generator (so `torch.manual_seed` makes a run reproducible). It has
the distribution of the reference's `torch.randn_like`, not its stream. A caller who sets `noise_sampler` (the
reference's attribute of AncestralSampler; here on every sampler, the EDM churn included) gets one call per draw,
`noise_sampler(x) -> tensor like x`, and that tensor is used instead.

Editing (DESIGN.md section 13): `strength` < 1 runs the tail of the schedule (discretizer.img2img_sigmas), and a
`known` latent with a `mask` [N, h, W] blends every launch that leaves a sampler step's result in x (the initial scaling
and each `_Eval.end` launch) toward known + s xi, s the noise level of that result, in the same launch
(pn_sampler_step_known). The known region's noise is a second Philox stream, its seed drawn once per sample after the
churn / ancestral seed, one draw index per blended launch."""
from __future__ import annotations

import math

import numpy as np
import torch

from ...util import default, instantiate_from_config
from .discretizer import img2img_sigmas
from .sampling_utils import get_ancestral_step, linear_multistep_coeff, to_neg_log_sigma, to_sigma

DEFAULT_GUIDER = {"target": "sgm.modules.diffusionmodules.guiders.IdentityGuider"}
F32 = torch.float32
# include/panacea_b200.h pn_sampler_mode (restated so the host logic imports without the native library)
EULER, HEUN, LMS, DPM, DPM_2M, SCALE = range(6)


class BoundDenoiser:
    """What `DiffusionEngine3D.sample` passes to the sampler in the reference is a lambda closing over
    (denoiser, model) (diffusion.py:251-254); this object is the same callable with the two parts visible, so the
    sampler can fuse the denoiser scalings, the guidance and the solver update into one kernel per evaluation."""

    def __init__(self, denoiser, network):
        self.denoiser = denoiser
        self.network = network

    def __call__(self, x, sigma, cond):
        return self.denoiser(self.network, x, sigma, cond)


class _Eval:
    """One network evaluation of the loop and the pn_sampler_step launch that follows it."""
    __slots__ = ("sigma", "step", "mode", "at_stage", "out_stage", "end", "kw")

    def __init__(self, eval_sigma, step, mode, *, at_stage=False, out_stage=False, end=False, **kw):
        self.sigma = float(eval_sigma)  # what the reference passes to the denoiser at this evaluation
        self.step = step
        self.mode = mode
        self.at_stage = at_stage        # evaluated at the stage buffer (Heun predictor, DPM++ 2S midpoint), not at x
        self.out_stage = out_stage      # the update goes to the stage buffer; x is left as it is
        self.end = end                  # x holds the result of sampler step `step` after this launch
        self.kw = kw                    # sigma, dt, coef, hist_read, hist_write, noise_amp, noise_scale


class BaseDiffusionSampler:
    def __init__(self, discretization_config, num_steps=None, guider_config=None, verbose=False, device="cuda"):
        self.num_steps = num_steps
        self.discretization = instantiate_from_config(discretization_config)
        self.guider = instantiate_from_config(default(guider_config, DEFAULT_GUIDER))
        self.verbose = verbose
        self.device = device
        self.last_timestep_indices = []     # timestep index of every network evaluation, in order (fused path)
        self.step_callback = None           # optional: called as step_callback(i, x) after every sampler step (tests)
        self.noise_sampler = None           # optional: noise_sampler(x) -> N(0,1) tensor like x, one call per draw
        self.ops = None                     # op set (default panacea_b200.ops.NativeOps)
        self.host_scalars = {}              # the solver scalars of the last schedule (get_ancestral_step, mults, LMS)

    def sigmas(self, num_steps=None, strength=1.0):
        """The schedule one sample runs over: the discretization's n + 1 sigmas, cut to the tail of `strength`."""
        return img2img_sigmas(self.discretization(self.num_steps if num_steps is None else num_steps, device="cpu"), strength)

    # ------------------------------------------------------------------ host plan
    def plan(self, num_steps=None, strength=1.0):
        """(init, evals) for one sample: `init` the keyword scalars of the launch that applies prepare_sampling_loop's
        x *= sqrt(1 + sigma_0^2) (sampling.py:50), `evals` one _Eval per network evaluation."""
        sig = self.sigmas(num_steps, strength).to(F32)
        self.host_scalars = {"ancestral": [], "mult": [], "lms": []}
        init = {"coef": (math.sqrt(1.0 + float(sig[0]) ** 2.0),)}
        return init, self._plan(sig, init)

    def _plan(self, sigmas, init):
        raise NotImplementedError

    def hist_slots(self):
        return 0

    # ------------------------------------------------------------------ loop
    @torch.no_grad()
    def __call__(self, denoiser, x, cond, uc=None, num_steps=None, *, strength=1.0, known=None, mask=None):
        """x [N,4,H,W] initial noise (unit variance); cond / uc dicts as produced by the conditioner. `denoiser` is any
        callable (x, sigma, cond) -> denoised, like the reference's lambda (diffusion.py:251-254); a `BoundDenoiser`
        takes the fused path. Returns the final latent, like the reference.

        `strength` in (0, 1] runs the last int(strength (n + 1)) sigmas only (x is then the scaled noisy latent of
        upstream's do_img2img); `known` [N,4,H,W] with `mask` [N,H,W] in [0, 1] keeps known + sigma xi where mask = 0."""
        if self.ops is None:
            from ....ops import NativeOps
            self.ops = NativeOps()
        uc = default(uc, cond)
        init, evals = self.plan(num_steps, strength)
        blend = self._blend_source(x, known, mask, evals)
        if not isinstance(denoiser, BoundDenoiser):
            return self._generic_loop(denoiser, x, cond, uc, init, evals, blend)
        net = denoiser.network
        cc = self.guider.prepare_cond(cond, uc)                   # once per sample
        if hasattr(net, "prepare"):
            net.prepare(cc)                                       # step-invariant conditioning work, once per sample
        return self._fused_loop(denoiser.denoiser, net, x, cc, init, evals, blend)

    def _halves(self):
        return 1 if type(self.guider).__name__.startswith("Identity") else 2

    def _buffers(self, x, evals):
        x0 = x.float().contiguous()
        stage = torch.empty_like(x0) if any(e.at_stage or e.out_stage for e in evals) else None
        slots = self.hist_slots()
        hist = torch.empty((slots, *x0.shape), dtype=F32, device=x0.device) if slots else None
        return x0, torch.empty_like(x0), stage, hist

    def _noise_source(self, init, evals):
        """-> draw(x, kw) adding the noise arguments of one launch: the caller's noise_sampler, or the in-kernel Philox
        stream with one seed per sample (torch's default CPU generator) and one draw index per noisy launch."""
        noisy = bool(init.get("noise_amp")) or any(e.kw.get("noise_amp") for e in evals)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if noisy and self.noise_sampler is None else 0
        count = [0]

        def draw(x, kw):
            if not kw.get("noise_amp"):
                return kw
            kw = dict(kw)
            if self.noise_sampler is not None:
                kw["noise"] = self.noise_sampler(x).to(device=x.device, dtype=F32).contiguous()
            else:
                kw["seed"], kw["draw"] = seed, count[0]
            count[0] += 1
            return kw
        return draw

    def _blend_source(self, x, known, mask, evals):
        """-> blend(k, kw) adding the known-latent arguments of a launch: k = -1 the initial scaling, else the index of
        the evaluation the launch follows. Only launches that leave a step's result in x blend; s is the sigma the
        next step's first evaluation sees (its sigma_hat under EDM churn), 0 after the last step."""
        if known is None and mask is None:
            return lambda k, kw: kw
        if known is None or mask is None:
            raise ValueError("known and mask go together")
        want = (x.shape[0], *x.shape[2:])
        if known.shape != x.shape or mask.shape != want:
            raise ValueError(f"known must be shaped like x {tuple(x.shape)} and mask {want}; got {tuple(known.shape)}, {tuple(mask.shape)}")
        known = known.to(device=x.device, dtype=F32).contiguous()
        mask = mask.to(device=x.device, dtype=F32).contiguous()
        if not (torch.isfinite(mask).all() and ((mask >= 0) & (mask <= 1)).all() and torch.isfinite(known).all()):
            raise ValueError("mask must be finite and in [0, 1], known finite")
        level = [e.sigma for e in evals] + [0.0]                   # level[k + 1]: what the launch after eval k leaves
        state = {"draw": 0}

        def blend(k, kw):
            if k >= 0 and not evals[k].end:
                return kw
            if "seed" not in state:                                # drawn at the first launch, after the churn seed
                state["seed"] = int(torch.randint(0, 2 ** 62, (1,)).item())
            kw = dict(kw, known=known, mask=mask, known_seed=state["seed"], known_draw=state["draw"], known_sigma=level[k + 1])
            state["draw"] += 1
            return kw
        return blend

    def _fused_loop(self, den, net, x, cc, init, evals, blend=lambda k, kw: kw):
        ops, halves = self.ops, self._halves()
        n = x.shape[0]
        scal = [den.step_scalars(e.sigma) for e in evals]           # (timestep index, quantised sigma, c_in)
        self.last_timestep_indices = [s[0] for s in scal]
        t_host = torch.tensor([[s[0]] * (halves * n) for s in scal], dtype=torch.int64)
        t_all = t_host.pin_memory().to(x.device, non_blocking=True) if x.is_cuda else t_host
        x0, xs, stage, hist = self._buffers(x, evals)
        x_in = torch.empty((halves * n, *x0.shape[1:]), dtype=F32, device=x0.device)
        draw = self._noise_source(init, evals)
        scale = float(getattr(self.guider, "scale", 1.0)) if halves == 2 else 1.0
        ops.sampler_step(SCALE, x0, out=xs, halves=halves, x_in_next=x_in, c_in_next=scal[0][2], **blend(-1, draw(x0, init)))
        x = xs
        static = hasattr(net, "static_io")
        for k, e in enumerate(evals):
            eps = net(x_in, t_all[k], cc, return_static=True) if static else net(x_in, t_all[k], cc)
            last = k + 1 == len(evals)
            ops.sampler_step(e.mode, x, eps.float().contiguous(), x_eval=stage if e.at_stage else None,
                             out=stage if e.out_stage else None, hist=hist, x_in_next=None if last else x_in,
                             halves=halves, sigma_q=scal[k][1], cfg_scale=scale, c_in_next=0.0 if last else scal[k + 1][2],
                             **blend(k, draw(x, e.kw)))
            if e.end and self.step_callback is not None:
                self.step_callback(e.step, x)
        return x

    def _generic_loop(self, denoiser, x, cond, uc, init, evals, blend=lambda k, kw: kw):
        """The reference's call contract: an opaque `denoiser(x2, sigma2, cond2) -> denoised2` per evaluation with the
        guider's inputs; guidance combine + solver update in one kernel (net_is_denoised)."""
        ops, halves = self.ops, self._halves()
        n = x.shape[0]
        self.last_timestep_indices = []
        x0, xs, stage, hist = self._buffers(x, evals)
        draw = self._noise_source(init, evals)
        scale = float(getattr(self.guider, "scale", 1.0)) if halves == 2 else 1.0
        ops.sampler_step(SCALE, x0, out=xs, halves=halves, **blend(-1, draw(x0, init)))
        x = xs
        for k, e in enumerate(evals):
            s_in = torch.full((n,), e.sigma, dtype=F32, device=x.device)
            x2, s2, c2 = self.guider.prepare_inputs(stage if e.at_stage else x, s_in, cond, uc)
            den2 = denoiser(x2, s2, c2).float().contiguous()
            ops.sampler_step(e.mode, x, den2, x_eval=stage if e.at_stage else None, out=stage if e.out_stage else None,
                             hist=hist, halves=halves, net_is_denoised=True, cfg_scale=scale, **blend(k, draw(x, e.kw)))
            if e.end and self.step_callback is not None:
                self.step_callback(e.step, x)
        return x


class SingleStepDiffusionSampler(BaseDiffusionSampler):
    pass


class EDMSampler(SingleStepDiffusionSampler):
    """sampling.py:85-133: sigma_hat = sigma (1 + gamma), gamma = min(s_churn / (num_sigmas - 1), sqrt 2 - 1) inside
    [s_tmin, s_tmax]; the churn noise s_noise sqrt(sigma_hat^2 - sigma^2) xi enters x before the evaluation at
    sigma_hat — emitted by the launch that ends the previous step (step 0: by the initial scaling)."""

    def __init__(self, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.s_churn = s_churn
        self.s_tmin = s_tmin
        self.s_tmax = s_tmax
        self.s_noise = s_noise

    def _plan(self, sigmas, init):
        num_sigmas = len(sigmas)
        hats, amps = [], []
        for i in range(num_sigmas - 1):
            gamma = min(self.s_churn / (num_sigmas - 1), 2 ** 0.5 - 1) if self.s_tmin <= sigmas[i] <= self.s_tmax else 0.0
            hat = sigmas[i] * (gamma + 1.0)
            hats.append(hat)
            amps.append(float((hat ** 2 - sigmas[i] ** 2) ** 0.5) if gamma > 0 else 0.0)
        churn = lambda i: {"noise_amp": amps[i], "noise_scale": self.s_noise} if i < len(amps) and amps[i] else {}
        init.update(churn(0))
        evals = []
        for i in range(num_sigmas - 1):
            dt = float(sigmas[i + 1] - hats[i])
            evals += self._edm_step(i, float(hats[i]), float(sigmas[i + 1]), dt, churn(i + 1))
        return evals

    def _edm_step(self, i, sigma_hat, next_sigma, dt, noise):
        return [_Eval(sigma_hat, i, EULER, end=True, sigma=sigma_hat, dt=dt, **noise)]


class EulerEDMSampler(EDMSampler):
    """sampling.py:214-218: d = (x - D) / sigma_hat, x += (sigma_next - sigma_hat) d."""


class HeunEDMSampler(EDMSampler):
    """sampling.py:221-237: predictor x_e = x + dt d (stage buffer, d kept in the history slot), corrector at
    (x_e, sigma_next): x += dt (d + d') / 2. One evaluation on the last step (sigma_next = 0)."""

    def hist_slots(self):
        return 1

    def _edm_step(self, i, sigma_hat, next_sigma, dt, noise):
        if next_sigma < 1e-14:
            return super()._edm_step(i, sigma_hat, next_sigma, dt, noise)
        return [_Eval(sigma_hat, i, EULER, out_stage=True, sigma=sigma_hat, dt=dt, hist_write=0),
                _Eval(next_sigma, i, HEUN, at_stage=True, end=True, sigma=next_sigma, dt=dt, hist_read=(0,), **noise)]


class AncestralSampler(SingleStepDiffusionSampler):
    """sampling.py:136-173: (sigma_down, sigma_up) = get_ancestral_step; after the update x += s_noise sigma_up xi when
    sigma_next > 0."""

    def __init__(self, eta=1.0, s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.eta = eta
        self.s_noise = s_noise

    def _plan(self, sigmas, init):
        evals = []
        for i in range(len(sigmas) - 1):
            sigma, next_sigma = sigmas[i], sigmas[i + 1]
            sigma_down, sigma_up = get_ancestral_step(sigma, next_sigma, eta=self.eta)
            self.host_scalars["ancestral"].append((float(sigma_down), float(sigma_up)))
            noise = {"noise_amp": float(sigma_up), "noise_scale": self.s_noise} if next_sigma > 0.0 else {}
            evals += self._ancestral_step(i, sigma, next_sigma, sigma_down, noise)
        return evals

    def _euler(self, i, sigma, sigma_down, noise):
        return [_Eval(sigma, i, EULER, end=True, sigma=float(sigma), dt=float(sigma_down - sigma), **noise)]


class EulerAncestralSampler(AncestralSampler):
    """sampling.py:240-247: x += (sigma_down - sigma) d, then the ancestral noise."""

    def _ancestral_step(self, i, sigma, next_sigma, sigma_down, noise):
        return self._euler(i, sigma, sigma_down, noise)


class DPMPP2SAncestralSampler(AncestralSampler):
    """sampling.py:250-287: midpoint x2 = (sigma_s / sigma) x - expm1(-h/2) D (stage buffer) evaluated at sigma_s,
    then x = (sigma_down / sigma) x - expm1(-h) D2, then the ancestral noise. Euler when sigma_down = 0."""

    def get_variables(self, sigma, sigma_down):
        t, t_next = [to_neg_log_sigma(s) for s in (sigma, sigma_down)]
        h = t_next - t
        s = t + 0.5 * h
        return h, s, t, t_next

    def get_mult(self, h, s, t, t_next):
        mult1 = to_sigma(s) / to_sigma(t)
        mult2 = (-0.5 * h).expm1()
        mult3 = to_sigma(t_next) / to_sigma(t)
        mult4 = (-h).expm1()
        return mult1, mult2, mult3, mult4

    def _ancestral_step(self, i, sigma, next_sigma, sigma_down, noise):
        if sigma_down < 1e-14:
            return self._euler(i, sigma, sigma_down, noise)
        h, s, t, t_next = self.get_variables(sigma, sigma_down)
        m = [float(v) for v in self.get_mult(h, s, t, t_next)]
        self.host_scalars["mult"].append(m)
        return [_Eval(sigma, i, DPM, out_stage=True, coef=m[:2]),
                _Eval(to_sigma(s), i, DPM, at_stage=True, end=True, coef=m[2:], **noise)]


class DPMPP2MSampler(BaseDiffusionSampler):
    """sampling.py:290-365: x = (sigma_next / sigma) x - expm1(-h) D_d, D_d = (1 + 1/2r) D - (1/2r) D_old; x_standard
    (D_d = D) on the first step and when sigma_next = 0 — chosen here on the host, where the reference computes
    -log 0 = inf and selects with torch.where. D goes to the one history slot."""

    def hist_slots(self):
        return 1

    def get_variables(self, sigma, next_sigma, previous_sigma=None):
        t, t_next = [to_neg_log_sigma(s) for s in (sigma, next_sigma)]
        h = t_next - t
        if previous_sigma is not None:
            h_last = t - to_neg_log_sigma(previous_sigma)
            r = h_last / h
            return h, r, t, t_next
        return h, None, t, t_next

    def get_mult(self, h, r, t, t_next, previous_sigma):
        mult1 = to_sigma(t_next) / to_sigma(t)
        mult2 = (-h).expm1()
        if previous_sigma is not None:
            mult3 = 1 + 1 / (2 * r)
            mult4 = 1 / (2 * r)
            return mult1, mult2, mult3, mult4
        return mult1, mult2

    def _plan(self, sigmas, init):
        evals = []
        for i in range(len(sigmas) - 1):
            previous = None if i == 0 else sigmas[i - 1]
            h, r, t, t_next = self.get_variables(sigmas[i], sigmas[i + 1], previous)
            m = [float(v) for v in self.get_mult(h, r, t, t_next, previous)]
            self.host_scalars["mult"].append(m)
            if previous is None or sigmas[i + 1] < 1e-14:
                evals.append(_Eval(sigmas[i], i, DPM, end=True, coef=m[:2], hist_write=0))
            else:
                evals.append(_Eval(sigmas[i], i, DPM_2M, end=True, coef=m, hist_read=(0,), hist_write=0))
        return evals


class LinearMultistepSampler(BaseDiffusionSampler):
    """sampling.py:176-211: x += sum_j c_j d_{i-j} over the last min(i + 1, order) derivatives (a ring of `order`
    history slots); the coefficients come from linear_multistep_coeff (scipy quad) once per schedule."""

    def __init__(self, order=4, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if not 1 <= order <= 4:
            raise NotImplementedError("pn_sampler_step takes up to 4 LMS coefficients (order <= 4; the reference default is 4)")
        self.order = order

    def hist_slots(self):
        return self.order

    def _plan(self, sigmas, init):
        sigmas_cpu = sigmas.numpy().astype(np.float32)
        evals = []
        for i in range(len(sigmas) - 1):
            cur_order = min(i + 1, self.order)
            coeffs = [linear_multistep_coeff(cur_order, sigmas_cpu, i, j) for j in range(cur_order)]
            self.host_scalars["lms"] += [(cur_order, i, j, float(c)) for j, c in enumerate(coeffs)]
            reads = tuple((i - j) % self.order for j in range(1, cur_order))
            evals.append(_Eval(sigmas[i], i, LMS, end=True, sigma=float(sigmas[i]), coef=coeffs, hist_read=reads,
                               hist_write=i % self.order))
        return evals
