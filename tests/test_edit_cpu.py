"""Editing recorded clips (DESIGN.md section 13) without a GPU: the strength rule of the schedule, the six samplers'
plans over the cut schedule, which launches blend toward the known latent and at which noise level, a numpy
restatement of the layout change mask (the GPU test compares the kernel with it), scene-file and command-line
validation, the ctypes mirror of pn_sampler_known_args, and the SASS of the plain step kernels."""
import hashlib
import json
import math
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from philox_ref import philox_normal
from sampler_ref_ops import TorchSamplerRefOps, sampler_step_torch
from test_layout_cpu import golden, scene_arrays, write_scene
from tools.make_sampler_golden import DISC, LOOPS, guider_config

ROOT = Path(__file__).resolve().parent.parent
F32 = torch.float32


def make_sampler(name, num_steps):
    from panacea_b200.sgm.util import instantiate_from_config
    _, cls, kw, guider = [e for e in LOOPS if e[0] == name][0]
    return instantiate_from_config({"target": f"sgm.modules.diffusionmodules.sampling.{cls}",
                                    "params": dict(num_steps=num_steps, discretization_config=DISC,
                                                   guider_config=guider_config(guider), **kw)})


# ------------------------------------------------------------------------------------------------ strength
def test_strength_known_answers():
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.discretizer import LegacyDDPMDiscretization, img2img_sigmas
    from panacea_b200.sgm.util import instantiate_from_config
    full = LegacyDDPMDiscretization()(25)
    den = instantiate_from_config(DEFAULT_DENOISER)
    assert torch.equal(img2img_sigmas(full, 1.0), full) and len(full) == 26
    cut = img2img_sigmas(full, 0.6)
    assert len(cut) == 15 and torch.equal(cut, full[11:])
    assert float(cut[0]) == pytest.approx(1.97733, abs=1e-5) and float(cut[-1]) == 0.0
    assert [den.step_scalars(float(s))[0] for s in cut[:-1]] == list(range(559, 0, -40))
    one = img2img_sigmas(full, 0.08)
    assert len(one) == 2 and float(one[0]) == pytest.approx(0.1963, abs=1e-4)
    for bad in (0.04, 0.0, -0.5, 1.01, float("nan")):
        with pytest.raises(ValueError):
            img2img_sigmas(full, bad)


SIX = ["euler", "heun", "euler_ancestral", "dpmpp_2s_ancestral", "dpmpp_2m", "lms"]


def _plan_record(init, evals, host):
    return init, [(e.sigma, e.step, e.mode, e.at_stage, e.out_stage, e.end, e.kw) for e in evals], host


@pytest.mark.parametrize("name", SIX + ["euler_churn"])
def test_plan_at_strength_is_the_plan_of_the_cut_schedule(name):
    from panacea_b200.sgm.modules.diffusionmodules.discretizer import img2img_sigmas
    s = make_sampler(name, 25)
    got = _plan_record(*s.plan(25, 0.6), s.host_scalars)
    ref = make_sampler(name, 25)
    sig = img2img_sigmas(ref.discretization(25, device="cpu"), 0.6).to(F32)
    ref.host_scalars = {"ancestral": [], "mult": [], "lms": []}
    init = {"coef": (math.sqrt(1.0 + float(sig[0]) ** 2.0),)}
    want = _plan_record(init, ref._plan(sig, init), ref.host_scalars)
    assert got == want
    assert max(e[1] for e in got[1]) == 13 and got[0]["coef"][0] == pytest.approx(math.sqrt(1 + 1.97733 ** 2), rel=1e-5)
    full = make_sampler(name, 25)
    full_plan = _plan_record(*full.plan(25), full.host_scalars)
    assert len(full_plan[1]) > len(got[1]) and full_plan == _plan_record(*make_sampler(name, 25).plan(25, 1.0),
                                                                         full.host_scalars)


# ------------------------------------------------------------------------------------------------ blended launches
def known_step_torch(mode, x, net=None, *, known=None, mask=None, known_seed=0, known_draw=0, known_sigma=0.0, **kw):
    """pn_sampler_step_known restated on top of sampler_step_torch (include/panacea_b200.h)."""
    if known is None:
        return sampler_step_torch(mode, x, net, **kw)
    probe = torch.empty_like(x)
    sampler_step_torch(mode, x.clone(), net, **{**kw, "out": probe, "x_in_next": None,
                                                  "hist": None if kw.get("hist") is None else kw["hist"].clone()})
    dst = sampler_step_torch(mode, x, net, **kw)
    n = x.numel()
    kn = known.reshape(-1).clone()
    if np.float32(known_sigma) != 0:
        xi = torch.from_numpy(philox_normal(known_seed, known_draw, n))
        kn = kn + torch.tensor(known_sigma, dtype=F32) * xi
    m = mask[:, None].expand_as(x).reshape(-1)
    o = probe.reshape(-1)
    o = torch.where(m == 1, o, torch.where(m == 0, kn, m * o + (1 - m) * kn))
    dst.reshape(-1).copy_(o)
    if kw.get("x_in_next") is not None:
        halves = kw.get("halves", 2)
        kw["x_in_next"].reshape(-1).copy_(torch.cat([o * torch.tensor(kw.get("c_in_next", 0.0), dtype=F32)] * halves))
    return dst


class Recorder(TorchSamplerRefOps):
    def __init__(self):
        self.calls = []

    def sampler_step(self, mode, x, net=None, **kw):
        self.calls.append((mode, {k: v for k, v in kw.items() if not torch.is_tensor(v)}, "known" in kw))
        return known_step_torch(mode, x, net, **kw)


def _run(name, strength, known=None, mask=None, seed=0):
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    from panacea_b200.sgm.util import instantiate_from_config
    s = make_sampler(name, 10)
    s.ops = Recorder()
    g = torch.Generator().manual_seed(7)
    net = lambda xi, t, cc: torch.randn(xi.shape, generator=g) * 0.5
    x = torch.randn(2, 4, 3, 5, generator=torch.Generator().manual_seed(1))
    torch.manual_seed(seed)
    out = s(BoundDenoiser(instantiate_from_config(DEFAULT_DENOISER), net), x, {}, {}, strength=strength, known=known, mask=mask)
    return s, out


@pytest.mark.parametrize("name", SIX + ["euler_churn"])
def test_the_end_launches_blend_at_the_level_they_leave(name):
    known = torch.randn(2, 4, 3, 5)
    s, out = _run(name, 0.6, known, torch.zeros(2, 3, 5))
    _, evals = s.plan(10, 0.6)
    calls = s.ops.calls
    blended = [c for c in calls if c[2]]
    assert len(calls) == len(evals) + 1 and len(blended) == 1 + sum(e.end for e in evals)
    assert calls[0][2] and all(c[2] == e.end for c, e in zip(calls[1:], evals))        # stage launches do not blend
    assert [c[1]["known_draw"] for c in blended] == list(range(len(blended)))
    assert len({c[1]["known_seed"] for c in blended}) == 1
    step_start = {}
    for e in evals:
        step_start.setdefault(e.step, e.sigma)                # the sigma the step's first evaluation sees
    want = [step_start[i] for i in sorted(step_start)] + [0.0]
    assert [c[1]["known_sigma"] for c in blended] == want
    assert torch.equal(out, known)                            # mask 0: the last launch leaves the known latent


def test_defaults_and_mask_one_leave_the_sample_unchanged():
    _, plain = _run("euler_churn", 1.0)
    _, ones = _run("euler_churn", 1.0, torch.randn(2, 4, 3, 5), torch.ones(2, 3, 5))
    assert torch.equal(plain, ones)


def test_known_and_mask_are_checked():
    x = torch.randn(2, 4, 3, 5)
    for known, mask, msg in ((x, None, "together"), (None, torch.ones(2, 3, 5), "together"),
                             (x, torch.ones(2, 3, 4), "shaped"), (x[:1], torch.ones(2, 3, 5), "shaped"),
                             (x, torch.full((2, 3, 5), 1.5), r"\[0, 1\]"), (x, torch.full((2, 3, 5), float("nan")), "finite")):
        with pytest.raises(ValueError, match=msg):
            _run("euler", 0.6, known, mask)


# ------------------------------------------------------------------------------------------------ change mask
def change_mask_ref(a, b, cell=8, dilate=1):
    """numpy restatement of pn_layout_change_mask: a, b [T, 19, H, 6w] -> [T, H/cell, 6w/cell] float32 in {0, 1}."""
    a, b = np.asarray(a), np.asarray(b)
    T, _, H, Wt = a.shape
    hc, wc = H // cell, Wt // 6 // cell
    cells = (a != b).any(1).reshape(T, hc, cell, 6 * wc, cell).any((2, 4)).reshape(T, hc, 6, wc)
    pad = np.pad(cells, ((0, 0), (dilate, dilate), (0, 0), (dilate, dilate)))
    out = np.zeros_like(cells)
    for dy in range(2 * dilate + 1):
        for dx in range(2 * dilate + 1):
            out |= pad[:, dy:dy + hc, :, dx:dx + wc]
    return out.reshape(T, hc, 6 * wc).astype(np.float32)


def _pair(H=32, w=48, T=2):
    a = np.zeros((T, 19, H, 6 * w), np.float32)
    return a, a.copy()


def test_change_mask_restatement_borders_seams_and_dilation():
    a, b = _pair()
    b[0, 18, 31, 47] = 1.0                     # bottom-right pixel of panel 0, ray channel only
    b[1, 0, 0, 48] = 1.0                       # top-left pixel of panel 1
    m0, m1, m3 = (change_mask_ref(a, b, 8, d) for d in (0, 1, 3))
    assert m0.shape == (2, 4, 36) and m0.sum() == 2 and m0[0, 3, 5] == 1 and m0[1, 0, 6] == 1
    assert m1[0, 2:4, 4:6].all() and m1[0].sum() == 4            # the corner cell grows into its panel only
    assert m1[0, :, 6:].sum() == 0 and m1[1, :, :6].sum() == 0     # nothing crosses the seam at x = 6 cells
    assert m1[1, 0:2, 6:8].all() and m1[1].sum() == 4
    assert m3[0, 0:4, 2:6].all() and m3[0].sum() == 16 and m3[1, 0:4, 6:10].all() and m3[1].sum() == 16
    assert change_mask_ref(a, a, 8, 3).sum() == 0


# ------------------------------------------------------------------------------------------------ scene and CLI
def _scene(tmp_path, frames=True, name="scene.npz", T=4):
    from PIL import Image
    arrays = scene_arrays(golden("layout_512"))
    keep = arrays["box_frame"] < T
    extra = {}
    if frames:
        for f in range(T):
            Image.fromarray(np.full((32, 6 * 64, 3), 10 * f, np.uint8)).save(tmp_path / f"f{f}.png")
        extra["frame_files"] = np.array([f"f{f}.png" for f in range(T)])
    Image.fromarray(np.zeros((32, 6 * 64, 3), np.uint8)).save(tmp_path / "cond.png")
    return write_scene(tmp_path, {k: v for k, v in arrays.items() if not k.startswith("map")} | extra | {
        "num_frames": np.array(T), "box_frame": arrays["box_frame"][keep], "labels": arrays["labels"][keep],
        "corners": arrays["corners"][keep], "cond_frame": np.array("cond.png")}, name)


def test_frame_files_are_read_and_checked(tmp_path):
    from panacea_b200 import layout as L
    from panacea_b200.inference import LayoutDataset
    scene = L.load_scene(_scene(tmp_path))
    assert [p.name for p in scene.frame_files] == ["f0.png", "f1.png", "f2.png", "f3.png"]
    ds = LayoutDataset(_scene(tmp_path), 4, (32, 64), True, 1, device="cpu", edit=True)
    assert ds.cond_frame is None and ds.scene.frame_files is not None
    with pytest.raises(L.SceneError, match="frame_files"):
        LayoutDataset(_scene(tmp_path, frames=False), 4, (32, 64), True, 1, device="cpu", edit=True)
    arrays = dict(np.load(_scene(tmp_path)))
    with pytest.raises(L.SceneError, match="frame_files"):
        L.load_scene(write_scene(tmp_path, {**arrays, "frame_files": arrays["frame_files"][:3]}, "short.npz"))


def test_change_mask_needs_scenes_of_one_length(tmp_path):
    from panacea_b200 import layout as L
    a = L.load_scene(_scene(tmp_path, T=4))
    b = L.load_scene(_scene(tmp_path, T=3, name="b.npz"))
    with pytest.raises(L.SceneError, match="frames"):
        L.change_mask(a, b, range(3), (32, 64), 1, device="cpu")


@pytest.mark.parametrize("args, message", [
    (["--strength", "0.5", "--clips", "2"], "--clips"),
    (["--strength", "0.5", "--cond_frame", "x.png"], "--cond_frame"),
    (["--mask_from", "a.npz", "--strength", "0.5"], "--layout"),
    (["--layout", "b.npz", "--mask_from", "a.npz"], "needs --strength"),
    (["--strength", "1.5"], r"\(0, 1\]"),
    (["--layout", "b.npz", "--mask_from", "a.npz", "--strength", "0.5", "--mask_dilate", "-1"], "mask_dilate"),
])
def test_cli_rejects_bad_edit_combinations(args, message):
    from panacea_b200 import inference as INF
    with pytest.raises(ValueError, match=message):
        INF.main(["--name", "edit", *args])


# ------------------------------------------------------------------------------------------------ ABI and SASS
def test_sampler_known_struct_matches_header_field_order():
    from panacea_b200 import _lib
    text = (ROOT / "include" / "panacea_b200.h").read_text()
    body = re.search(r"typedef struct pn_sampler_known_args \{(.*?)\} pn_sampler_known_args;", text, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = [part.strip().split()[-1].lstrip("*") for decl in body.split(";") if decl.strip() for part in decl.split(",")]
    assert fields == [f[0] for f in _lib.SamplerKnownArgs._fields_]


def test_plain_step_kernels_compile_to_the_sass_they_had_before_the_known_flag(tmp_path):
    """The KNOWN = false instantiations of sampler_step_kernel against instruction fingerprints of the kernel before
    the flag existed (tests/golden/sampler_step_sass.json, taken with the nvcc recorded there)."""
    from panacea_b200 import build
    nvcc = Path(build.NVCC)
    cuobjdump = nvcc.with_name("cuobjdump")
    if not nvcc.exists() or not cuobjdump.exists():
        pytest.skip(f"no nvcc / cuobjdump at {nvcc.parent}")
    want = json.loads((ROOT / "tests" / "golden" / "sampler_step_sass.json").read_text())
    version = subprocess.run([str(nvcc), "--version"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
    if version != want["nvcc"]:
        pytest.skip(f"fingerprints were taken with {want['nvcc']}, this is {version}")
    obj = tmp_path / "sampler.o"
    subprocess.run([str(nvcc), *build.NVCC_FLAGS, "-c", str(build.CSRC / "sampler.cu"), "-o", str(obj)], check=True)
    sass = subprocess.run([str(cuobjdump), "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    got = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        m = re.search(r"sampler_step_kernelILi(\d)ELb0E", name)
        if m:
            ins = [x.group(1).strip() for x in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", body)]
            got[m.group(1)] = hashlib.sha256("\n".join(ins).encode()).hexdigest()
    assert got == want["instructions_sha256"]
