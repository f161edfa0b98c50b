"""Pasting the recorded pixels back outside an edit, and user-drawn edit masks, on the GPU (DESIGN.md section 13):

  * pn_composite_frames against the numpy restatement of test_composite_cpu on seeded cell masks at 32 x 64 and
    256 x 512 per view, feather 0, 1, 8 and 64, recorded frames made from bytes: alpha, the output where alpha = 0 (the
    recorded byte centre) and where alpha = 1 (the decode) bitwise, the ramp within fp32 rounding of an fp64 blend;
  * pn_mask_cells bitwise against the restatement;
  * both kernels bitwise the same over two calls;
  * on the small model of the scene tests: a composited edit's plain decode is bitwise the uncomposited edit, its
    frames quantise to the recorded bytes where alpha = 0 and are the decode where alpha = 1, and under one seed it is
    bitwise the edit composed by hand from its steps;
  * the command line with a layout change mask and a drawn mask writes a lossless `samples` strip whose pixels are the
    recorded bytes outside the mask and its ramp."""
import numpy as np
import pytest
import torch

from panacea_b200 import layout as L
from panacea_b200.composite import composite_frames
from panacea_b200.frame_io import _to_uint8_hwc
from test_composite_cpu import alpha_ref, byte_centre, mask_cells_ref
from test_edit_gpu import _layout_batch, _scene_pair
from test_scene_gpu import CFG, T, _small

pytestmark = pytest.mark.gpu


def _inputs(T_, H, w, seed):
    g = np.random.default_rng(seed)
    Wt = 6 * w
    rec = torch.from_numpy(g.integers(0, 256, (T_, 3, H, Wt)).astype(np.float32) / np.float32(127.5) - np.float32(1))
    dec = torch.from_numpy((g.random((T_, 3, H, Wt)) * 2.4 - 1.2).astype(np.float32))
    cells = (g.random((T_, H // 8, Wt // 8)) < 0.04).astype(np.float32)
    cells[0, :, : w // 8] = 0                                          # an empty panel
    cells[0, :, w // 8: 2 * w // 8] *= g.random((H // 8, w // 8)).astype(np.float32)   # soft values > 0 regenerate
    cells[-1, 1:, 2 * w // 8: 3 * w // 8] = 1                          # a panel mostly regenerated
    return dec, rec, torch.from_numpy(cells)


@pytest.mark.parametrize("feather", [0, 1, 8, 64])
@pytest.mark.parametrize("hw", [(32, 64), (256, 512)])
def test_composite_kernel_equals_the_restatement(hw, feather):
    H, w = hw
    dec, rec, cells = _inputs(2, H, w, seed=H + feather)
    out, alpha = composite_frames(dec.cuda(), rec.cuda(), cells.cuda(), feather)
    again, alpha2 = composite_frames(dec.cuda(), rec.cuda(), cells.cuda(), feather)
    torch.cuda.synchronize()
    assert torch.equal(out, again) and torch.equal(alpha, alpha2)
    out, alpha = out.cpu().numpy(), alpha.cpu().numpy()
    want = alpha_ref(cells.numpy(), H, w, feather)
    assert np.array_equal(alpha, want)
    k, d = byte_centre(rec.numpy()), dec.numpy()
    a = np.broadcast_to(want[:, None], d.shape)
    zero, one = a == 0, a == 1
    ramp = ~zero & ~one
    assert zero.any() and one.any() and (ramp.any() == (feather > 0))
    assert np.array_equal(out[zero], k[zero]) and np.array_equal(out[one], d[one])
    blend = k.astype(np.float64) + a.astype(np.float64) * (d.astype(np.float64) - k)
    err = np.abs(out.astype(np.float64) - blend)[ramp]
    bound = 2.0 ** -22 * (np.abs(d) + np.abs(k))[ramp]
    assert (err <= bound).all(), (err - bound).max() if err.size else None


@pytest.mark.parametrize("dilate", [0, 1, 3])
@pytest.mark.parametrize("hw", [(32, 64), (256, 512)])
def test_mask_cells_kernel_equals_the_restatement(hw, dilate):
    H, w = hw
    g = np.random.default_rng(dilate)
    px = np.where(g.random((3, H, 6 * w)) < 0.002, g.integers(1, 256, (3, H, 6 * w)), 0).astype(np.uint8)
    px[1, H - 1, w - 1] = 9                                            # a corner pixel at the seam
    got = L.mask_cells(px, dilate)
    again = L.mask_cells(px, dilate)
    torch.cuda.synchronize()
    assert torch.equal(got, again) and got.shape == (3, H // 8, 6 * w // 8)
    want = mask_cells_ref(px, 8, dilate)
    assert np.array_equal(got.cpu().numpy(), want) and 0 < want.sum() < want.size


def _recorded_bytes(tmp_path):
    from PIL import Image
    return np.stack([np.asarray(Image.open(tmp_path / f"rec{f}.png").convert("RGB")) for f in range(T)])


def test_a_composited_edit_keeps_the_recorded_bytes_outside_the_mask(tmp_path):
    orig, edited = _scene_pair(tmp_path)
    ds, batch = _layout_batch(edited)
    mask = L.change_mask(L.load_scene(orig), ds.scene, ds.frames(0), (64, 128), 1)
    m, _ = _small("bf16")
    torch.manual_seed(4)
    plain = m.edit_images(batch, 0.6, mask=mask)
    torch.manual_seed(4)
    log = m.edit_images(batch, 0.6, mask=mask, composite=8)
    assert torch.equal(log["decoded_samples"], plain["samples"])
    assert torch.equal(log["sample_latents"], plain["sample_latents"])
    alpha = log["composite_alpha"].cpu().numpy()
    assert log["composite_alpha"].shape == (T, 64, 768)
    assert np.array_equal(alpha, alpha_ref(mask.cpu().numpy(), 64, 128, 8))
    rec = _recorded_bytes(tmp_path)
    got = np.stack([_to_uint8_hwc(f) for f in log["samples"]])
    zero, one = alpha == 0, alpha == 1
    assert zero.any() and one.any()
    assert np.array_equal(got[zero], rec[zero])
    s, d = log["samples"].permute(0, 2, 3, 1).cpu().numpy(), plain["samples"].permute(0, 2, 3, 1).cpu().numpy()
    assert np.array_equal(s[one], d[one])
    assert (np.stack([_to_uint8_hwc(f) for f in plain["samples"]])[zero] != rec[zero]).any()   # the decode alone is not


def test_a_composited_edit_is_the_edit_by_hand(tmp_path):
    """Under one seed, edit_images with a change mask and composite=8 is bitwise _log_inputs -> _initial_noise ->
    (z0 + sigma eps) / sqrt(1 + sigma^2) -> sampler(strength, known=z0, mask) -> decode -> composite_frames: this pins
    the edit's draws (the encoder's posterior sample, the initial noise, the churn seed, the known region's seed)."""
    from panacea_b200.sgm.modules.diffusionmodules.sampling import BoundDenoiser
    orig, edited = _scene_pair(tmp_path)
    ds, batch = _layout_batch(edited)
    mask = L.change_mask(L.load_scene(orig), ds.scene, ds.frames(0), (64, 128), 1)
    m, _ = _small("bf16")
    torch.manual_seed(9)
    log = m.edit_images(batch, 0.6, mask=mask, composite=8)
    torch.manual_seed(9)
    ref, c, uc, N, shape, z0 = m._log_inputs(batch, 8)
    eps = m._initial_noise(c, N * T, shape)
    sigma = float(m.sampler.sigmas(strength=0.6)[0])
    x = (z0 + sigma * eps) / (1.0 + sigma ** 2) ** 0.5
    lat = m.sampler(BoundDenoiser(m.denoiser, m.model), x, c, uc=uc, strength=0.6, known=z0, mask=mask)
    dec = m.decode_first_stage(lat)
    frames, alpha = composite_frames(dec, ref["inputs"], mask, 8)
    assert torch.equal(log["inputs"], ref["inputs"]) and torch.equal(log["edit_mask"], mask)
    assert torch.equal(log["sample_latents"], lat) and torch.equal(log["decoded_samples"], dec)
    assert torch.equal(log["samples"], frames) and torch.equal(log["composite_alpha"], alpha)
    assert not torch.equal(frames, dec)


def test_inference_entry_point_composites_a_drawn_and_a_layout_mask(tmp_path):
    from PIL import Image
    from panacea_b200 import inference as INF
    orig, edited = _scene_pair(tmp_path)
    drawn = np.zeros((64, 768), np.uint8)
    drawn[20:30, 3 * 128 + 40: 3 * 128 + 70] = 255                       # a region on CAM_BACK the layout does not describe
    Image.fromarray(drawn).save(tmp_path / "m.png")
    out = tmp_path / "out"
    INF.main(["--name", "edit", "--base", CFG, "--inferdir", str(out), "--layout", str(edited), "--mask_from", str(orig),
              "--mask_image", str(tmp_path / "m.png"), "--strength", "0.6", "--composite", "8", "--image_hw", "64", "128",
              "--randomize_zero_init"])
    strips = sorted((out / "edit" / "allimages" / "samples").glob("*.png"))
    assert len(strips) == 1 and len(list((out / "edit" / "allimages" / "decoded_samples").glob("*.png"))) == 1
    strip = np.asarray(Image.open(strips[0]).convert("RGB")).reshape(T, 64, 768, 3)
    ds = INF.LayoutDataset(edited, T, (64, 128), True, 1, edit=True)
    cells = torch.maximum(L.change_mask(L.load_scene(orig), ds.scene, ds.frames(0), (64, 128), 1),
                          L.mask_cells(L.read_edit_mask(tmp_path / "m.png", T, (64, 128)), 1))
    alpha = alpha_ref(cells.cpu().numpy(), 64, 128, 8)
    zero = alpha == 0
    assert zero.any() and (alpha[:, 20:30, 3 * 128 + 40: 3 * 128 + 70] == 1).all()
    assert np.array_equal(strip[zero], _recorded_bytes(tmp_path)[zero])
