"""Pasting the recorded pixels back outside an edit and user-drawn edit masks (DESIGN.md section 13), without a GPU:
a numpy restatement of pn_composite_frames (the GPU test compares the kernel with it) checked on hand cases, why the
recorded pixels are written as byte centres, the pixel-to-cell pooling of pn_mask_cells, `read_edit_mask`, the command
line's refusals and the ctypes signatures of both entry points."""
import re
import types
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import ndimage

from test_edit_cpu import change_mask_ref

ROOT = Path(__file__).resolve().parent.parent
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")
F32 = np.float32


# ------------------------------------------------------------------------------------------------ restatement
def alpha_ref(cells, H, w, feather):
    """alpha [T, H, 6w] fp32 of pn_composite_frames from cells [T, H/cell, 6w/cell]: per panel, the exact Euclidean
    distance transform gives the nearest regenerated pixel, hence the integer d2; then the fp32 formula."""
    cells = np.asarray(cells)
    T, hc, _ = cells.shape
    cell = H // hc
    px = np.repeat(np.repeat(cells > 0, cell, 1), cell, 2)                         # [T, H, 6w]
    alpha = np.zeros(px.shape, F32)
    reach = F32(feather + 1)
    for t in range(T):
        for v in range(6):
            on = px[t, :, v * w:(v + 1) * w]
            if not on.any():
                continue
            idx = ndimage.distance_transform_edt(~on, return_distances=False, return_indices=True)
            yy, xx = np.indices(on.shape)
            d2 = (idx[0] - yy) ** 2 + (idx[1] - xx) ** 2
            ramp = np.maximum(F32(0), F32(1) - np.sqrt(d2.astype(F32)) / reach)
            alpha[t, :, v * w:(v + 1) * w] = np.where(d2 == 0, F32(1), ramp)
    return alpha


def byte_centre(recorded):
    """k = (b + 0.5) / 127.5 - 1 with b = clamp(rint((recorded + 1) 127.5), 0, 255), fp32."""
    b = np.clip(np.rint((np.asarray(recorded, F32) + F32(1)) * F32(127.5)), 0, 255).astype(F32)
    return (b + F32(0.5)) / F32(127.5) - F32(1)


def _brute_alpha(cells, H, w, feather):
    """The definition itself, min over the panel's cells of dx^2 + dy^2 in pixel units: checks the EDT restatement."""
    T, hc, Wc = cells.shape
    cell = H // hc
    out = np.zeros((T, H, 6 * w), F32)
    ys, xs = np.arange(H)[:, None], np.arange(w)[None, :]
    for t in range(T):
        for v in range(6):
            d2 = np.full((H, w), np.iinfo(np.int64).max)
            for cy, cx in zip(*np.nonzero(cells[t, :, v * w // cell:(v + 1) * w // cell] > 0)):
                dy = np.maximum(0, np.maximum(cy * cell - ys, ys - (cy * cell + cell - 1)))
                dx = np.maximum(0, np.maximum(cx * cell - xs, xs - (cx * cell + cell - 1)))
                d2 = np.minimum(d2, dx * dx + dy * dy)
            if (d2 == np.iinfo(np.int64).max).all():
                continue
            ramp = np.maximum(F32(0), F32(1) - np.sqrt(d2.astype(F32)) / F32(feather + 1))
            out[t, :, v * w:(v + 1) * w] = np.where(d2 == 0, F32(1), ramp)
    return out


def _cells(T=2, H=32, w=48, cell=8):
    return np.zeros((T, H // cell, 6 * w // cell), F32)


def test_alpha_restatement_hand_cases():
    H, w = 32, 48
    c = _cells()
    assert (alpha_ref(c, H, w, 8) == 0).all()                                      # no regenerated cell: alpha 0
    c[0, 1, 5] = 1.0                                      # panel 0, cell column 5: its right edge is the seam at x = 47
    c[1, 0, 6] = 0.5                                      # panel 1, top-left cell: any value > 0 regenerates
    a0 = alpha_ref(c, H, w, 0)
    assert set(np.unique(a0)) == {0.0, 1.0} and a0[0].sum() == 64 and a0[0, 8:16, 40:48].all()
    a64 = alpha_ref(c, H, w, 64)
    assert (a64[0, :, w:] == 0).all() and (a64[1, :, :w] == 0).all()               # nothing crosses a seam
    assert (a64[0, :, :w] > 0).all() and a64[1, :, w:2 * w].min() > 0 and (a64[1, :, 2 * w:] == 0).all()
    assert a64[0, 12, 39] == F32(1) - F32(1) / F32(65)                             # one pixel left of the cell
    assert a64[0, 17, 39] == F32(1) - np.sqrt(F32(5)) / F32(65)                    # d2 = 2^2 + 1^2
    a8 = alpha_ref(c, H, w, 8)
    assert a8[0, 12, 31] == 0 and a8[0, 12, 32] == F32(1) - F32(8) / F32(9)        # dx 9 reaches 0, dx 8 does not
    for F in (0, 1, 8, 64):
        assert np.array_equal(alpha_ref(c, H, w, F), _brute_alpha(c, H, w, F)), F
    g = np.random.default_rng(0)
    rnd = (g.random((2, 4, 36)) < 0.1).astype(F32)
    for F in (0, 3, 17):
        assert np.array_equal(alpha_ref(rnd, H, w, F), _brute_alpha(rnd, H, w, F)), F


def test_byte_centre_survives_the_writers_quantiser_and_the_plain_read_does_not():
    from panacea_b200.frame_io import _to_uint8_hwc
    u = np.arange(256, dtype=np.uint8)
    read = u.astype(F32) / F32(127.5) - F32(1)                                     # what the datasets hand over
    back = lambda x: _to_uint8_hwc(torch.from_numpy(np.asarray(x, F32)).reshape(1, 1, 256))[0]
    plain = back(read)
    assert (plain != u).sum() == 63 and (plain[plain != u] == u[plain != u] - 1).all()
    assert plain[1] == 0 and plain[2] == 1
    assert np.array_equal(np.rint((read + F32(1)) * F32(127.5)).astype(np.uint8), u)
    assert np.array_equal(back(byte_centre(read)), u)


def test_composite_frames_checks_its_arguments():
    from panacea_b200.composite import composite_frames
    d = torch.zeros(2, 3, 16, 96)
    c = torch.zeros(2, 2, 12)
    for args, msg in (((d[:, :2], d, c, 8), "decoded"), ((d, d[:1], c, 8), "recorded"), ((d, d, c[:1], 8), "cells"),
                      ((d, d, torch.zeros(2, 2, 10), 8), "cells"), ((d, d, c, 65), "feather"), ((d, d, c, -1), "feather")):
        with pytest.raises(ValueError, match=msg):
            composite_frames(*args)


def test_edit_without_a_mask_cannot_composite():
    from panacea_b200.sgm.models.diffusion import DiffusionEngine3D
    with pytest.raises(ValueError, match="composite"):
        DiffusionEngine3D.edit_images(types.SimpleNamespace(input_key="jpg"), {"jpg": None}, 0.6, composite=8)


# ------------------------------------------------------------------------------------------------ pixel masks
def mask_cells_ref(pixels, cell=8, dilate=1):
    """pn_mask_cells restated: a cell is 1 when any of its pixels is nonzero, then change_mask_ref's dilation."""
    p = np.asarray(pixels)[:, None] != 0
    return change_mask_ref(p, np.zeros_like(p), cell, dilate)


def test_pixel_mask_pools_and_dilates_within_panels():
    p = np.zeros((2, 32, 6 * 48), np.uint8)
    p[0, 31, 47] = 255                                     # bottom-right pixel of panel 0
    p[1, 0, 48] = 1                                        # top-left pixel of panel 1
    m0, m1 = mask_cells_ref(p, 8, 0), mask_cells_ref(p, 8, 1)
    assert m0.shape == (2, 4, 36) and m0.sum() == 2 and m0[0, 3, 5] == 1 and m0[1, 0, 6] == 1
    assert m1[0, 2:4, 4:6].all() and m1[0].sum() == 4 and m1[1, 0:2, 6:8].all() and m1[1].sum() == 4


def test_read_edit_mask_formats(tmp_path):
    from PIL import Image
    from panacea_b200 import layout as L
    img = np.zeros((32, 6 * 64), np.uint8)
    img[3, 5], img[4, 6], img[5, 7] = 127, 128, 255
    Image.fromarray(np.stack([img] * 3, -1)).save(tmp_path / "m.png")
    got = L.read_edit_mask(tmp_path / "m.png", 4, (32, 64))
    assert got.dtype == np.uint8 and got.shape == (4, 32, 384) and got.sum() == 8
    assert (got[:, 4, 6] == 1).all() and (got[:, 5, 7] == 1).all() and (got[:, 3, 5] == 0).all()
    per_frame = np.zeros((4, 32, 384), bool)
    per_frame[2, 10, 100] = True
    np.save(tmp_path / "m.npy", per_frame)
    got = L.read_edit_mask(tmp_path / "m.npy", 4, (32, 64))
    assert got.dtype == np.uint8 and got.sum() == 1 and got[2, 10, 100] == 1
    np.save(tmp_path / "u.npy", per_frame.astype(np.uint8) * 7)
    assert np.array_equal(L.read_edit_mask(tmp_path / "u.npy", 4, (32, 64)), got)


@pytest.mark.parametrize("make, message", [
    (lambda d: np.save(d / "x.npy", np.zeros((4, 32, 384), np.float32)), r"bool or uint8.*float32"),
    (lambda d: np.save(d / "x.npy", np.zeros((3, 32, 384), bool)), r"expected 4 frames, got 3"),
    (lambda d: np.save(d / "x.npy", np.zeros((4, 32, 383), bool)), r"expected shape \(4, 32, 384\).*\(4, 32, 383\)"),
    (lambda d: np.save(d / "x.npy", np.zeros((32, 384), bool)), r"expected shape \(4, 32, 384\).*\(32, 384\)"),
    (lambda d: __import__("PIL.Image").Image.fromarray(np.zeros((32, 380), np.uint8)).save(d / "x.png"),
     r"expected a 384 x 32 image, got 380 x 32"),
])
def test_read_edit_mask_rejections(tmp_path, make, message):
    from panacea_b200 import layout as L
    make(tmp_path)
    path = next(tmp_path.glob("x.*"))
    with pytest.raises(ValueError, match=message):
        L.read_edit_mask(path, 4, (32, 64))


# ------------------------------------------------------------------------------------------------ command line
@pytest.mark.parametrize("args, message", [
    (["--mask_image", "m.png"], "--mask_image.*needs --strength"),
    (["--composite", "8"], "--composite.*needs --strength"),
    (["--strength", "0.5", "--composite", "8"], "--composite needs an edit mask"),
    (["--strength", "0.5", "--mask_image", "m.png", "--composite", "65"], "--composite must lie in 0 .. 64"),
    (["--strength", "0.5", "--mask_image", "m.png", "--composite", "-1"], "--composite must lie in 0 .. 64"),
])
def test_cli_rejects_bad_mask_and_composite_combinations(args, message):
    from panacea_b200 import inference as INF
    with pytest.raises(ValueError, match=message):
        INF.main(["--name", "edit", *args])


@pytest.mark.parametrize("shape, message", [((32, 6 * 64), "384 x 32"), ((32, 6 * 48), "288 x 32")])
def test_cli_rejects_a_mask_image_that_does_not_fit(tmp_path, shape, message):
    from PIL import Image
    from panacea_b200 import inference as INF
    Image.fromarray(np.zeros(shape, np.uint8)).save(tmp_path / "m.png")
    with pytest.raises(ValueError, match=f"--mask_image.*expected a 384 x 16 image, got {message}"):
        INF.main(["--name", "edit", "--base", CFG, "--strength", "0.5", "--image_hw", "16", "64", "--mask_image",
                  str(tmp_path / "m.png")])


def test_cli_rejects_a_mask_npy_with_the_wrong_frame_count(tmp_path):
    from panacea_b200 import inference as INF
    np.save(tmp_path / "m.npy", np.zeros((8, 32, 384), bool))                      # the tiny config has T = 4
    with pytest.raises(ValueError, match="--mask_image.*expected 4 frames, got 8"):
        INF.main(["--name", "edit", "--base", CFG, "--strength", "0.5", "--image_hw", "32", "64", "--mask_image",
                  str(tmp_path / "m.npy"), "--composite", "8"])


# ------------------------------------------------------------------------------------------------ ABI
def _header_params(name):
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "panacea_b200.h").read_text(), flags=re.S)
    params = re.search(r"\bint %s\((.*?)\);" % name, text, flags=re.S).group(1)
    return [" ".join(p.split()[:-1]) for p in params.split(",")]


@pytest.mark.parametrize("name", ["pn_mask_cells", "pn_composite_frames"])
def test_ctypes_signatures_follow_the_header(name):
    import ctypes as C
    from panacea_b200 import _lib
    res, args = _lib.SIGNATURES[name]
    kinds = {C.c_void_p: "pointer", C.c_int64: "int64_t"}
    want = ["pointer" if "*" in p else p for p in _header_params(name)]
    assert res is C.c_int and [kinds[a] for a in args] == want
