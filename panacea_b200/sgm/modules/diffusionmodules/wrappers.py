"""Drop-in for `sgm.modules.diffusionmodules.wrappers.OpenAIWrapperControlLDM3D` (reference wrappers.py:37-70):
`forward(x, t, c) -> eps` with c = {concat, cond_feat, crossattn}. This is the operator boundary the denoiser
calls once per Euler step (denoiser.py:28)."""
from __future__ import annotations

import torch
import torch.nn as nn

OPENAIUNETWRAPPERCONTROLLDM3D = "sgm.modules.diffusionmodules.wrappers.OpenAIWrapperControlLDM3D"


class IdentityWrapper(nn.Module):
    def __init__(self, diffusion_model, compile_model: bool = False):
        super().__init__()
        if compile_model:
            raise NotImplementedError("compile_model=True: torch.compile is not part of this implementation")
        self.diffusion_model = diffusion_model

    def forward(self, *args, **kwargs):
        return self.diffusion_model(*args, **kwargs)


class OpenAIWrapperControlLDM3D(IdentityWrapper):
    """ControlNet -> UNet on the channel-concatenated latent. Step-invariant work (BEV hint stem, the 69 text K/V
    projections) is cached across calls, keyed on the CONTENT of `c["cond_feat"]` / `c["crossattn"]`:

      * same tensor objects as last call (held by strong reference, `_version` unchanged) -> reuse, no device work;
      * different objects (the reference's VanillaCFG.prepare_inputs torch.cat-s a fresh dict every step,
        guiders.py:31-40) -> a 64-bit content fingerprint (pn_fingerprint, ~0.2 ms) decides; equal -> reuse;
      * otherwise the conditioning is recomputed.

    Addresses are never trusted (the caching allocator recycles them between samples). `prepare(c)` recomputes
    unconditionally — the samplers of this package call it once per sample. The per-step network runs as one CUDA graph
    when `use_cuda_graph` is set (static shapes, no allocation inside the graph's replay)."""

    def __init__(self, diffusion_model, compile_model: bool = False, use_cuda_graph: bool = False, hint_repeat: int = 1):
        super().__init__(diffusion_model, compile_model)
        self.use_cuda_graph = use_cuda_graph
        self.hint_repeat = hint_repeat        # 2 when cond_feat holds the hint once for both CFG halves
        self._held = None                     # (cond_feat, crossattn, versions): strong refs of the prepared tensors
        self._cond_fp = None                  # (fingerprints, engine generation, hint_repeat)
        self._graph = None
        self._graph_sig = None
        self._static = None

    def invalidate(self, drop_graph: bool = True) -> None:
        """Forget the prepared conditioning (next call re-runs the hint stem and the text K/V projections). The captured
        graph only depends on shapes and on buffer addresses that survive a new conditioning, so a serving loop passes
        drop_graph=False between samples and keeps replaying it."""
        self._held = None
        self._cond_fp = None
        if drop_graph:
            self._graph = None

    @torch.no_grad()
    def prepare(self, c: dict) -> None:
        """Run the step-invariant work for conditioning `c` now (once per sample)."""
        eng = self.diffusion_model.engine()
        hint, ctx = c["cond_feat"], c["crossattn"]
        eng.prepare_condition(hint.float(), ctx.float(), hint_repeat=self.hint_repeat)
        self._held = (hint, ctx, hint._version, ctx._version)
        self._cond_fp = (None, eng.generation, self.hint_repeat)      # fingerprints are computed lazily, only if needed

    def _ensure_prepared(self, eng, c: dict) -> None:
        hint, ctx = c["cond_feat"], c["crossattn"]
        tag = (eng.generation, self.hint_repeat)
        if self._held is not None and self._cond_fp is not None and self._cond_fp[1:] == tag:
            h0, c0, hv, cv = self._held
            if hint is h0 and ctx is c0 and hint._version == hv and ctx._version == cv:
                return
            ops = eng.ops
            if self._cond_fp[0] is None:
                if h0._version != hv or c0._version != cv:     # the held tensors were modified in place: content unknown
                    self.prepare(c)
                    return
                self._cond_fp = ((ops.fingerprint(h0.contiguous()), ops.fingerprint(c0.contiguous())), *tag)
            fp = (ops.fingerprint(hint.contiguous()), ops.fingerprint(ctx.contiguous()))
            if fp == self._cond_fp[0]:
                self._held = (hint, ctx, hint._version, ctx._version)
                return
        self.prepare(c)

    def static_io(self):
        """(x, t, concat, eps) buffers of the captured graph, or None before the first graphed call. A caller that
        writes its inputs there and reads eps there avoids the per-step copies (the fused sampler does)."""
        return self._static

    @torch.no_grad()
    def forward(self, x: torch.Tensor, t: torch.Tensor, c: dict, *, return_static: bool = False, **kwargs) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("panacea_b200 runs on CUDA (sm_90a) only; there is no CPU path")
        eng = self.diffusion_model.engine()
        self._ensure_prepared(eng, c)
        x = x.float().contiguous()
        t = t.to(torch.int64).contiguous()
        concat = c.get("concat", None)
        concat = None if concat is None else concat.float().contiguous()
        if not self.use_cuda_graph:
            return eng.eps(x, concat, t)
        sig = (tuple(x.shape), None if concat is None else tuple(concat.shape), tuple(c["cond_feat"].shape),
               tuple(c["crossattn"].shape), eng.generation, eng.cond["guided"].data_ptr(), x.device)
        if self._graph is None or self._graph_sig != sig:
            self._capture(eng, x, concat, t, sig)
        sx, sc, st, so = self._static
        if x.data_ptr() != sx.data_ptr():
            sx.copy_(x)                       # plain device memcpy nodes (cudaMemcpyAsync), skipped when the caller already
        if t.data_ptr() != st.data_ptr():     # works in the static buffers (static_io())
            st.copy_(t)
        if sc is not None and concat.data_ptr() != sc.data_ptr():
            sc.copy_(concat)
        self._graph.replay()
        return so if return_static else so.clone()

    def _capture(self, eng, x, concat, t, sig):
        sx, st = x.clone(), t.clone()
        sc = None if concat is None else concat.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            eng.eps(sx, sc, st)          # warm-up: function attributes, TMA-map cache, allocator pools
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            so = eng.eps(sx, sc, st)
        self._graph, self._graph_sig, self._static = g, sig, (sx, sc, st, so)
