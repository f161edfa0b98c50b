"""Editing recorded clips on the GPU (DESIGN.md section 13):

  * pn_sampler_step_known in every mode, both guiders, with the network output as eps or as D, with and without the
    launch's own noise: mask 1 is bitwise pn_sampler_step, mask 0 is bitwise known + s xi (fp32 product, then fp32
    sum), a soft mask is within fp32 rounding of an fp64 blend of the two;
  * the change-mask kernel is bitwise the numpy restatement of test_edit_cpu on a seeded scene with a box moved, one
    added and one removed;
  * on the small model of the scene tests: mask 0 returns the recorded latent and its reconstruction bitwise, a
    one-box layout edit keeps the latent bitwise outside the change mask and changes it inside, the fused and the
    plain-callable loops agree, an edit replays the CUDA graph of a generated clip, and the command line edits a
    layout scene."""
import os

import numpy as np
import pytest
import torch

from panacea_b200 import layout as L
from philox_ref import philox_normal
from test_edit_cpu import change_mask_ref
from test_layout_cpu import golden, scene_arrays, write_scene
from test_samplers_gpu import MODES, SHAPE, _rand
from test_scene_gpu import CFG, T, _small

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from panacea_b200.ops import NativeOps
    return NativeOps()


@pytest.mark.parametrize("noise", ["none", "philox"])
@pytest.mark.parametrize("denoised", [False, True])
@pytest.mark.parametrize("halves", [2, 1])
@pytest.mark.parametrize("mode", list(MODES))
def test_sampler_step_known(ops, mode, halves, denoised, noise):
    spec = dict(MODES[mode])
    out_stage, x_eval_stage = spec.pop("out_stage", False), spec.pop("x_eval_stage", False)
    n = int(np.prod(SHAPE))
    x, stage, hist = _rand(SHAPE, 1, 10.0), _rand(SHAPE, 3, 10.0), _rand((4,) + SHAPE, 4, 3.0)
    net = _rand((halves * SHAPE[0],) + SHAPE[1:], 2)
    known = _rand(SHAPE, 6, 2.0)
    kw = dict(spec, halves=halves, sigma_q=14.5, cfg_scale=5.0, c_in_next=0.0685, net_is_denoised=denoised)
    if noise == "philox":
        kw.update(noise_scale=1.003, noise_amp=0.37, seed=0x1234_5678_9ABC, draw=5)
    s, kseed, kdraw = 3.25, 0xFEED_0000_1234, 9
    g = torch.Generator().manual_seed(8)
    soft = torch.rand((SHAPE[0], *SHAPE[2:]), generator=g)
    soft[:, :4] = 0.0
    soft[:, 4:8] = 1.0
    masks = {"one": torch.ones(SHAPE[0], *SHAPE[2:]), "zero": torch.zeros(SHAPE[0], *SHAPE[2:]), "soft": soft}

    def run(mask):
        xx, st, hh = x.clone(), stage.clone(), hist.clone()
        x_in = torch.full((halves * SHAPE[0],) + SHAPE[1:], float("nan"), device="cuda")
        extra = {} if mask is None else dict(known=known, mask=mask.cuda(), known_seed=kseed, known_draw=kdraw, known_sigma=s)
        dst = ops.sampler_step(net=net if spec["mode"] != 5 else None, x=xx, x_eval=st if x_eval_stage else None,
                               out=st if out_stage else None, hist=hh, x_in_next=x_in, **kw, **extra)
        torch.cuda.synchronize()
        return [t.cpu() for t in (dst, xx, st, hh, x_in)]
    plain = run(None)
    names = ("out", "x", "stage", "hist", "x_in_next")
    for got, ref, what in zip(run(masks["one"]), plain, names):
        assert torch.equal(got, ref), f"mask 1: {what}"
    xi = philox_normal(kseed, kdraw, n)
    kn = torch.from_numpy(known.cpu().numpy().reshape(-1) + np.float32(s) * xi).reshape(SHAPE)   # fp32 ops
    c_in = np.float32(kw["c_in_next"])
    zero = run(masks["zero"])
    assert torch.equal(zero[0], kn), "mask 0: out"
    assert torch.equal(zero[3], plain[3]), "mask 0: hist"
    assert torch.equal(zero[4], torch.cat([kn * c_in] * halves)), "mask 0: x_in_next"
    got = run(masks["soft"])
    m = soft[:, None].double()
    want = m * plain[0].double() + (1 - m) * kn.double()
    err = (got[0].double() - want).abs()
    bound = 2.0 ** -21 * (plain[0].double().abs() + kn.double().abs())            # a few fp32 roundings of the operands
    assert (err <= bound).all(), (err - bound).max()
    assert torch.equal(got[3], plain[3])
    assert torch.equal(got[4], torch.cat([got[0] * c_in] * halves))


def _edited_arrays(arrays, move=0, remove=1, add_from=2):
    """A box moved 3 m along x, one removed and a copy of another added 4 m to its side, on every frame."""
    corners, labels, frames = arrays["corners"].copy(), arrays["labels"].copy(), arrays["box_frame"].copy()
    corners[move] += np.array([3.0, 0.0, 0.0], np.float32)
    added = corners[add_from] + np.array([0.0, 4.0, 0.0], np.float32)
    keep = np.arange(len(labels)) != remove
    return {**arrays, "corners": np.concatenate([corners[keep], added[None]]),
            "labels": np.concatenate([labels[keep], labels[add_from:add_from + 1]]),
            "box_frame": np.concatenate([frames[keep], frames[add_from:add_from + 1]])}


@pytest.mark.parametrize("dilate", [0, 1, 3])
def test_change_mask_kernel_equals_the_restatement(tmp_path, dilate):
    g = golden("layout_512")
    H, w = g["image_hw"]
    arrays = scene_arrays(g)
    a = L.load_scene(write_scene(tmp_path, arrays, "a.npz"))
    b = L.load_scene(write_scene(tmp_path, _edited_arrays(arrays), "b.npz"))
    frames = range(a.num_frames)
    got = L.change_mask(a, b, frames, (H, w), dilate)
    again = L.change_mask(a, b, frames, (H, w), dilate)
    ra, rb = (L.render_layout(sc, frames, H, w).cpu().numpy() for sc in (a, b))
    want = change_mask_ref(ra, rb, 8, dilate)
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    assert got.shape == (a.num_frames, H // 8, 6 * w // 8)
    assert np.array_equal(got.cpu().numpy(), want)
    assert 0 < want.sum() < want.size / 2
    assert L.change_mask(a, a, frames, (H, w), dilate).sum().item() == 0


# ------------------------------------------------------------------------------------------------ the model
def _scene_pair(tmp_path):
    """The 256 x 512 golden scene shrunk to 64 x 128 per view and T frames, with recorded frames; and the same scene with
    one box moved."""
    from PIL import Image
    arrays = scene_arrays(golden("layout_512"))
    keep = arrays["box_frame"] < T
    l2i = arrays["lidar2img"].copy()
    l2i[:, :2] *= 0.25
    rng = np.random.default_rng(0)
    for f in range(T):
        Image.fromarray(rng.integers(0, 256, (64, 6 * 128, 3), dtype=np.uint8)).save(tmp_path / f"rec{f}.png")
    base = {k: v for k, v in arrays.items() if not k.startswith("map")}
    base.update(num_frames=np.array(T), lidar2img=l2i, box_frame=arrays["box_frame"][keep], labels=arrays["labels"][keep],
                corners=arrays["corners"][keep], frame_files=np.array([f"rec{f}.png" for f in range(T)]))
    base.pop("cond_frame", None)
    orig = write_scene(tmp_path, base, "orig.npz")
    edited = dict(base, corners=base["corners"].copy())
    edited["corners"][_visible_box(L.load_scene(orig), base["box_frame"])] += np.array([2.0, 0.0, 0.0], np.float32)
    return orig, write_scene(tmp_path, edited, "edited.npz")


def _visible_box(scene, box_frame):
    """Index (into the file's boxes) of the first frame-0 box that some camera keeps at 64 x 128."""
    for j, idx in enumerate(np.nonzero(box_frame == 0)[0]):
        for l2i in scene.lidar2img.values():
            if len(L.project_boxes(scene.corners[0][j:j + 1], scene.labels[0][j:j + 1], l2i, 64, 128)["bbox"]):
                return idx
    raise AssertionError("the test scene has no box in view on frame 0")


def _recording_encoder(m):
    """Records the latents m.encode_first_stage returns: it samples the posterior, so z0 is only known as returned."""
    seen, enc = [], m.encode_first_stage
    m.encode_first_stage = lambda x: (seen.append(enc(x)), seen[-1])[1]
    return seen


def _layout_batch(path, edit=True):
    from torch.utils.data import DataLoader
    from panacea_b200.inference import LayoutDataset
    ds = LayoutDataset(path, T, (64, 128), True, 1, edit=edit)
    batch = next(iter(DataLoader(ds, batch_size=1)))
    return ds, {k: v.cuda() if isinstance(v, torch.Tensor) else v for k, v in batch.items()}


def test_mask_zero_returns_the_recorded_latent_and_its_reconstruction():
    from torch.utils.data import DataLoader
    from panacea_b200.inference import SyntheticBEVDataset
    m, _ = _small("bf16")
    batch = next(iter(DataLoader(SyntheticBEVDataset(1, T, (64, 128)), batch_size=1)))
    batch = {k: v.cuda() if isinstance(v, torch.Tensor) else v for k, v in batch.items()}
    seen = _recording_encoder(m)
    torch.manual_seed(3)
    log = m.edit_images(batch, 0.6, mask=torch.zeros(T, 8, 96))
    z0 = seen[-1]
    assert torch.equal(log["sample_latents"], z0)
    assert torch.equal(log["samples"], log["reconstructions"])
    assert log["edit_mask"].shape == (T, 8, 96) and log["edit_mask"].sum() == 0
    torch.manual_seed(3)
    free = m.edit_images(batch, 0.6)
    assert not torch.equal(free["sample_latents"], z0) and free["edit_mask"].min() == 1
    assert set(free) >= {"inputs", "reconstructions", "samples", "sample_latents", "control", "cond_img"}


def test_one_box_edit_changes_only_the_masked_latent(tmp_path):
    orig, edited = _scene_pair(tmp_path)
    ds, batch = _layout_batch(edited)
    mask = L.change_mask(L.load_scene(orig), ds.scene, ds.frames(0), (64, 128), 1)
    assert 0 < mask.sum() < mask.numel() / 2
    m, _ = _small("bf16")
    seen = _recording_encoder(m)
    torch.manual_seed(4)
    log = m.edit_images(batch, 0.5, mask=mask)
    z0 = seen[-1]
    keep = (mask == 0)[:, None].expand_as(z0)
    assert torch.equal(log["sample_latents"][keep], z0[keep])
    inside = ~keep
    assert (log["sample_latents"][inside] != z0[inside]).float().mean() > 0.99
    assert torch.equal(log["edit_mask"], mask)


def test_fused_and_plain_callable_loops_agree_when_editing(tmp_path):
    """In parity mode, so that a blend applied differently by the two loops cannot hide under bf16 network error."""
    from panacea_b200.pipeline import DEFAULT_DENOISER
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    from panacea_b200.sgm.util import instantiate_from_config
    m, _ = _small("parity")
    w, den = m.model, instantiate_from_config(DEFAULT_DENOISER)
    _, batch = _layout_batch(_scene_pair(tmp_path)[1])
    log, c, uc, N, shape, z0 = m._log_inputs(batch, 8)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(z0.shape, generator=g).cuda()
    mask = torch.rand((z0.shape[0], *z0.shape[2:]), generator=g).cuda()
    mask[:, :, :40] = 0.0
    outs = []
    for d in (BoundDenoiser(den, w), lambda xx, sigma, cc: den(w, xx, sigma, cc)):
        torch.manual_seed(6)
        outs.append(m.sampler(d, x, c, uc, num_steps=10, strength=0.6, known=z0, mask=mask).cpu())
    fused, plain = outs
    rel = ((fused - plain).norm() / fused.norm()).item()
    assert rel < 5e-3, rel
    print(f"EDIT fused vs plain-callable rel-L2 {rel:.3e}")
    zc = z0.cpu()
    assert torch.equal(fused[:, :, :, :40], zc[:, :, :, :40]) and torch.equal(plain[:, :, :, :40], zc[:, :, :, :40])


def test_an_edit_replays_the_graph_of_a_generated_clip(tmp_path):
    m, _ = _small("bf16")
    w = m.model
    captures = []
    cap = w._capture
    w._capture = lambda *a, **k: (captures.append(1), cap(*a, **k))[1]
    _, batch = _layout_batch(_scene_pair(tmp_path)[1])
    torch.manual_seed(0)
    m.log_images(batch)
    graph = w._graph
    m.edit_images(batch, 0.6, mask=torch.zeros(T, 8, 96))
    assert len(captures) == 1 and w._graph is graph


def test_inference_entry_point_edits_a_layout_scene(tmp_path):
    from panacea_b200 import inference as INF
    from panacea_b200.frame_io import CAMERA_VIEWS
    orig, edited = _scene_pair(tmp_path)
    INF.main(["--name", "edit", "--base", CFG, "--inferdir", str(tmp_path / "out"), "--layout", str(edited),
              "--mask_from", str(orig), "--strength", "0.5", "--image_hw", "64", "128", "--randomize_zero_init"])
    fake = tmp_path / "out" / "edit" / "fake"
    dirs = sorted(os.listdir(fake))
    assert dirs == sorted(f"{cam}_edited__{cam}__{T - 1:06d}" for cam in CAMERA_VIEWS)
    for d in dirs:
        assert sorted(os.listdir(fake / d)) == [f"_{i:06}.jpg" for i in range(T)]
