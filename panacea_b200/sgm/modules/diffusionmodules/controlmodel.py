"""Drop-in replacements for `sgm.modules.diffusionmodules.controlmodel.{ControlNet3D, ControlledUNetModel3D}`
(reference controlmodel.py:19-202; topology from UNetModel3D.__init__, openaimodel.py:804-1261).

Same constructor keywords, same `forward` signatures, same state-dict keys — but no nn.Module tree and no
torch compute: parameters live in one flat table keyed by the reference's names, and `forward` runs the
hand-written sm_90a kernels through `panacea_b200.engine.Engine`. Without the native library (or without a
CUDA device) `forward` raises; there is no eager fallback.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from ....engine import Engine
from ....netplan import (NetConfig, config_from_kwargs, controlnet_param_spec, is_zero_init, unet_param_spec)
from ...util import instantiate_from_config


class _FlatParams(nn.Module):
    """Holds parameters under the reference's dotted key names (state_dict()/load_state_dict() compatible)."""

    def __init__(self, spec: dict):
        super().__init__()
        self._spec = dict(spec)
        self._attr = {k: "p__" + k.replace(".", "__") for k in spec}
        for k, shape in spec.items():
            self.register_parameter(self._attr[k], nn.Parameter(torch.empty(shape), requires_grad=False))
        self._pack_version = 0
        self.reset_parameters()

    @torch.no_grad()
    def reset_parameters(self) -> None:
        """Reference default init: nn.Conv*/nn.Linear kaiming-uniform(a=sqrt 5) + uniform bias, norms (1, 0), and
        the reference's zero_module()'d layers zeroed (so a fresh model predicts eps == 0, like the reference)."""
        for k in self._spec:
            p = getattr(self, self._attr[k])
            if is_zero_init(k):
                p.zero_()
            elif p.ndim == 1 and k.endswith(".weight"):
                p.fill_(1.0)
            elif k.endswith(".weight"):
                nn.init.kaiming_uniform_(p, a=math.sqrt(5))
            else:  # bias
                wkey = k[: -len("bias")] + "weight"
                w = self._spec.get(wkey)
                if w is not None and len(w) > 1:
                    bound = 1.0 / math.sqrt(math.prod(w[1:]))
                    p.uniform_(-bound, bound)
                else:
                    p.zero_()
        self._pack_version += 1

    @torch.no_grad()
    def randomize_zero_init(self, seed: int = 0, std: float = 0.02) -> None:
        """Re-draw the zero-initialised tensors ~ N(0, std^2) (synthetic benchmarks / parity tests need a
        network whose output is not identically zero). Drawn on the parameter's own device."""
        gens = {}
        for k in sorted(self._spec):
            if is_zero_init(k):
                p = getattr(self, self._attr[k])
                g = gens.get(p.device)
                if g is None:
                    g = gens[p.device] = torch.Generator(device=p.device).manual_seed(seed)
                p.copy_(torch.randn(p.shape, generator=g, device=p.device) * std)
        self._pack_version += 1

    def reference_parameters(self) -> dict:
        return {k: getattr(self, a) for k, a in self._attr.items()}

    def _apply(self, fn, recurse=True):
        """.to() / .cuda() / .float() replace or rewrite the parameters: the packed operands are stale afterwards."""
        r = super()._apply(fn, recurse)
        self._pack_version += 1
        return r

    def mark_parameters_changed(self) -> None:
        """Call after editing parameters in place (p.copy_(), p.mul_() ...): forces a repack on the next forward."""
        self._pack_version += 1

    # --- state-dict plumbing with the reference's key names
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        for k, a in self._attr.items():
            p = getattr(self, a)
            destination[prefix + k] = p if keep_vars else p.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        for k, a in self._attr.items():
            full = prefix + k
            if full not in state_dict:
                missing_keys.append(full)
                continue
            src = state_dict[full]
            p = getattr(self, a)
            if tuple(src.shape) != tuple(p.shape):
                error_msgs.append(f"size mismatch for {full}: checkpoint {tuple(src.shape)} vs model {tuple(p.shape)}")
                continue
            with torch.no_grad():
                p.copy_(src)
        if strict:
            children = set(self._modules)
            for full in state_dict:
                if full.startswith(prefix):
                    rest = full[len(prefix):]
                    if rest not in self._attr and rest.split(".", 1)[0] not in children:
                        unexpected_keys.append(full)
        self._pack_version += 1


PRECISIONS = ("bf16", "parity")


def _resolve_precision(precision):
    """Precision mode of the engine: "bf16" (default; bf16 tensor-core operands, fp32 accumulation / softmax / norms /
    residual stream) or "parity" (split-bf16 operands = fp32-class products, fp32 attention: matches the reference's
    fp32 math to rtol 1e-3 / atol 1e-4 at 3-4x the cost). Constructor kwarg `precision=`, else env PN_PRECISION."""
    import os
    p = precision if precision is not None else os.environ.get("PN_PRECISION", "bf16")
    if p not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {p!r}")
    return p


def _native_ops(precision: str = "bf16"):
    from ....ops import NativeOps, ParityOps
    return ParityOps() if precision == "parity" else NativeOps()


class ControlNet3D(_FlatParams):
    """controlmodel.py:19-142. Encoder copy + BEV hint stem + 13 zero convolutions."""

    def __init__(self, hint_channels, control_scales, dims=2, disable_temporal=False, *args, precision=None, **kwargs):
        if args:
            raise TypeError("ControlNet3D takes keyword arguments only (as instantiate_from_config passes them)")
        if dims != 2 or disable_temporal:
            raise NotImplementedError("panacea_b200: dims=2 and disable_temporal=False only")
        kwargs = dict(kwargs)
        kwargs["out_channels"] = kwargs["in_channels"]            # controlmodel.py:29
        cfg = config_from_kwargs(kwargs, hint_channels=hint_channels, control_scales=float(control_scales))
        if hint_channels > 19:
            raise NotImplementedError("hint_channels > 19 (multi-map hints, controlmodel.py:108-117) is not supported")
        super().__init__(controlnet_param_spec(cfg))
        self.precision = _resolve_precision(precision)
        self.cfg: NetConfig = cfg
        self.control_scales = control_scales
        self.hint_channels = hint_channels
        self.num_frames = self.cfg.num_frames
        self.num_classes = None
        self.model_channels = self.cfg.model_channels
        self._engine: Engine | None = None
        self._engine_version = -1

    def _standalone_engine(self) -> Engine:
        if self._engine is None:
            self._engine = Engine(self.cfg, _native_ops(self.precision))
        if self._engine_version != self._pack_version:
            self._engine.pack(None, self.reference_parameters())
            self._engine_version = self._pack_version
        return self._engine

    @torch.no_grad()
    def forward(self, x, hint, timesteps=None, context=None, y=None, **kwargs):
        """x [N,C,H,W] fp32, hint [N,19,8H,8W], timesteps int64 [N], context [b,77,D] -> list of 13 NCHW tensors."""
        assert y is None, "must specify y if and only if the model is class-conditional"
        eng = self._standalone_engine()
        ops = eng.ops
        eng.prepare_hint(hint.float())
        eng.prepare_text(context.float())
        outs = eng.controlnet(ops.nchw_to_nhwc(x.float().contiguous()), timesteps.to(torch.int64).contiguous())
        res = []
        for o, st_shape in zip(outs, self._out_shapes(x)):
            res.append(ops.nhwc_to_nchw(o.view(*st_shape)))
        return res

    def _out_shapes(self, x):
        N, _, H, W = x.shape
        shapes, h, w = [], H, W
        for blk in self._standalone_engine().plan_cn.encoder:
            if blk[0].kind == "down":
                h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            shapes.append((N, h, w, blk[-1].cout))
        shapes.append((N, h, w, shapes[-1][3]))
        return shapes


class ControlledUNetModel3D(_FlatParams):
    """controlmodel.py:146-202. UNet whose decoder consumes the ControlNet residuals; owns `.controlnet`."""

    def __init__(self, controlnet_config=None, only_add_on_center_frame=False, *args, precision=None, **kwargs):
        if args:
            raise TypeError("ControlledUNetModel3D takes keyword arguments only")
        cfg = config_from_kwargs(dict(kwargs))
        super().__init__(unet_param_spec(cfg))
        self.precision = _resolve_precision(precision)
        self.cfg: NetConfig = cfg
        self.num_frames = self.cfg.num_frames
        self.num_classes = None
        self.model_channels = self.cfg.model_channels
        self.in_channels = self.cfg.in_channels
        self.out_channels = self.cfg.out_channels
        self._engine: Engine | None = None
        self._engine_version = None
        if controlnet_config is not None:
            self.controlnet = instantiate_from_config(controlnet_config)
            cn = self.controlnet.cfg
            assert (cn.model_channels, cn.channel_mult, cn.num_frames) == (self.cfg.model_channels, self.cfg.channel_mult, self.cfg.num_frames), \
                "ControlNet and UNet configurations must agree"
            self.cfg.hint_channels = cn.hint_channels
            self.cfg.control_scales = cn.control_scales

    def set_precision(self, precision: str) -> None:
        """Switch between "bf16" and "parity"; the engine (packed weights, caches) is rebuilt on the next call."""
        self.precision = _resolve_precision(precision)
        self._engine = None
        self._engine_version = None
        self._pack_version += 1           # wrappers key their caches / captured graph on the pack generation

    def engine(self) -> Engine:
        """Lazily builds the engine and (re)packs the MMA operands whenever parameters changed."""
        if self._engine is None:
            self._engine = Engine(self.cfg, _native_ops(self.precision))
        cn = getattr(self, "controlnet", None)
        dev = getattr(self, next(iter(self._attr.values()))).device
        ver = (self._pack_version, cn._pack_version if cn is not None else -1, str(dev))
        if self._engine_version != ver:
            self._engine.pack(self.reference_parameters(), cn.reference_parameters() if cn is not None else None)
            self._engine_version = ver
        return self._engine

    @torch.no_grad()
    def forward(self, x, timesteps=None, context=None, y=None, control=None, **kwargs):
        """x [N,C,H,W], timesteps int64 [N], context [b,77,D], control: list of 13 NCHW residuals (consumed)."""
        assert y is None, "must specify y if and only if the model is class-conditional"
        eng = self.engine()
        ops = eng.ops
        eng.prepare_text(context.float())
        ctrl = [ops.nchw_to_nhwc(c.float().contiguous()) for c in control]
        del control[:]                                            # the reference pops every entry (controlmodel.py:192-195)
        e = eng.unet(ops.nchw_to_nhwc(x.float().contiguous()), timesteps.to(torch.int64).contiguous(), ctrl)
        return ops.nhwc_to_nchw(e, channels=self.cfg.out_channels)
