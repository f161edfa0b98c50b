"""Scene files and the ControlNet's 19-channel layout maps (DESIGN.md section 12).

A scene file is one `.npz` that describes what a generated scene holds, frame by frame: 3-D boxes with class labels,
map polylines in ego metres and the six cameras' `lidar2img` matrices. `render_layout` turns the frames of one clip
into the hint `cond_img` [T, 19, H, 6w] the checkpoint was trained on, with the contract of the reference's dataset
(sgm/data/nuscenes_video/nuscenes_datasets_video.py, MyDataset, and render.py). Host code here does the per-primitive
geometry in fp64 numpy (projection, hull-canvas clipping, painter's order, polyline resampling, the ray range); one
launch of `pn_render_layout` (csrc/layout.cu) rasterises all T x 6 panels x 19 channels on the GPU.

Panel p of a frame is camera `frame_io.CAMERA_VIEWS[p]` (the dataset's `camera_views`, :509) and uses that camera's
own matrix (the dataset indexes its matrices through `viewid`, :264-271). Channels, all k/255 in fp32:
  0..2   boxes painted far to near: the front face (corners 4..7) filled in 0.5 palette[label+1] + 127.5, then the 12
         edges in palette[label+1] reversed (BGR), 2 px wide (:307-341, :525);
  3..12  one channel per class of CLASS_NAMES: the minimum over boxes of int(3 depth) on each box's 2-D rectangle
         (:286-305), 255 elsewhere;
  13..15 map polylines drawn 4 px wide in MAP_COLORS_BGR on white (render.py:21-100, 168-199);
  16..18 camera-ray directions normalised by one min and max over all panels and components (:382-412).
The reference draws the map lines with cv2.LINE_AA on a float64 canvas, where OpenCV does not anti-alias, so every
channel is a plain overwrite.

Scene file keys (arrays; `np.savez`):
  num_frames   ()            frames in the scene; a scene of K clips of T frames sharing m has K(T-m)+m (m = 1 default)
  cameras      (6,) str      the camera of each row of lidar2img (any order, each of CAMERA_VIEWS once)
  lidar2img    (6, 4, 4)     ego -> image, held in fp32 as the reference's dataset holds it
  box_frame    (M,) int      frame of each box
  labels       (M,) int      class index into CLASS_NAMES
  corners      (M, 8, 3)     box corners in ego metres, mmdet3d's LiDARInstance3DBoxes.corners order; or
  boxes        (M, 7)        bottom centre x, y, z, size dx, dy, dz, yaw (see `box_corners`)
  map_frame    (L,) int      frame of each polyline (optional, with the next three)
  map_labels   (L,) int      index into MAP_CLASSES
  map_lengths  (L,) int      points per polyline (>= 2)
  map_points   (sum, 2|3)    the polylines' points in ego metres, concatenated (z = 0 when 2-D)
  prompt       () str        optional caption; without it `caption` writes one from the class counts
  cond_frame   () str        optional path (relative to the file) of the conditioning frame, an [H, 6w] RGB image
  frame_files  (num_frames,) str  optional paths (relative to the file) of the scene's recorded frames, [H, 6w] RGB
                             images: the clip that editing starts from (DESIGN.md section 13)

`change_mask` compares two scenes' renders at latent resolution: where an edited scene differs from its original.
`read_edit_mask` and `mask_cells` take a mask the user drew instead, and bring it to the same form.
"""
from __future__ import annotations

from dataclasses import dataclass
from pathlib import Path

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .frame_io import CAMERA_VIEWS

# nuscenes_datasets_video.py:127-130 (this list, not the one at :81, is the class order of channels 3..12)
CLASS_NAMES = ("car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
               "pedestrian", "traffic_cone")
# nuscenes_datasets_video.py:232-252; box label l is drawn in row l + 1
BOX_PALETTE = np.array([
    [255, 255, 255], [128, 64, 128], [244, 35, 232], [70, 70, 70], [102, 102, 156], [190, 153, 153], [153, 153, 153],
    [250, 170, 30], [220, 220, 0], [107, 142, 35], [152, 251, 152], [0, 130, 180], [220, 20, 60], [255, 0, 0],
    [0, 0, 142], [0, 0, 70], [0, 60, 100], [0, 80, 100], [0, 0, 230], [119, 11, 32]], dtype=np.int64)
# nuscenes_datasets_video.py:120-124 (class ids) and render.py:103-110 (BGR colours)
MAP_CLASSES = ("ped_crossing", "divider", "boundary")
MAP_COLORS_BGR = ((255, 0, 0), (0, 0, 255), (0, 255, 0))
# nuscenes_datasets_video.py:118, 360, 370-376: the map ROI in metres; the nuScenes pipeline stores polylines
# normalised to it, see `map_from_normalized`
MAP_ROI = (60.0, 30.0)
DEPTH_CLIP = (0.1, 51.2)          # :428
BOX_LINE_WIDTH = 2                # :525
MAP_LINE_WIDTH = 4                # :378
MAP_SAMPLES = 200                 # render.py:52
HINT_CHANNELS = 19
LATENT_CELL = 8                   # pixels per latent cell side: the VAE's downsampling factor
_PRIM = 16                        # PN_LAYOUT_PRIM_FLOATS
_RECT, _QUAD, _BOX_SEG, _MAP_SEG = 0, 1, 2, 3
# draw_rect over corners 0..3 and 4..7 (:71-78, 338-339), after the four edges i -> i+4 (:332-336)
_BOX_EDGES = ((0, 4), (1, 5), (2, 6), (3, 7), (3, 0), (0, 1), (1, 2), (2, 3), (7, 4), (4, 5), (5, 6), (6, 7))


class SceneError(ValueError):
    pass


def _reach(thickness: int) -> float:
    """Distance from a segment within which pixel centres are inked: a cv2.line of thickness t covers t + 1 pixels
    across (its outline is filled inclusively)."""
    return (thickness + 1) / 2


def box_corners(boxes: np.ndarray) -> np.ndarray:
    """[M, 7] (bottom centre x, y, z, size dx, dy, dz, yaw) -> [M, 8, 3] corners in the order of mmdet3d's
    LiDARInstance3DBoxes.corners: unit corners (0,0,0),(0,0,1),(0,1,1),(0,1,0),(1,0,0),(1,0,1),(1,1,1),(1,1,0) minus
    (0.5, 0.5, 0), scaled by the size, rotated by yaw about z, moved to the bottom centre. Corners 4..7 are the +x face."""
    boxes = np.asarray(boxes, dtype=np.float64)
    unit = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]], np.float64)
    local = (unit - np.array([0.5, 0.5, 0.0]))[None] * boxes[:, None, 3:6]
    c, s = np.cos(boxes[:, 6])[:, None], np.sin(boxes[:, 6])[:, None]
    x, y = local[..., 0], local[..., 1]
    return np.stack([c * x - s * y, s * x + c * y, local[..., 2]], -1) + boxes[:, None, 0:3]


def map_from_normalized(points: np.ndarray) -> np.ndarray:
    """Polyline points as the nuScenes map pipeline stores them (x, y in [0, 1] over the ROI) -> ego metres, as the
    reference's dataset converts them (:370-376)."""
    roi = np.array(MAP_ROI)
    out = np.array(points, dtype=np.float64)
    out[:, :2] = out[:, :2] * (roi + 2) - roi / 2
    return out


@dataclass
class Scene:
    num_frames: int
    lidar2img: dict                # camera name -> [4, 4] float64 holding fp32 values
    corners: list                  # per frame [n, 8, 3] float64 holding fp32 values
    labels: list                   # per frame [n] int64
    polylines: list                # per frame [(map class, [k, 3] float64)] in drawing order
    prompt: str | None = None
    cond_frame: Path | None = None
    frame_files: list | None = None   # per frame, the Path of the recorded [H, 6w] RGB frame


def _need(cond, msg):
    if not cond:
        raise SceneError(msg)


def _finite(name, a):
    _need(np.issubdtype(a.dtype, np.number) and np.isfinite(a).all(), f"{name}: values must be finite numbers")


def _int_array(z, name, shape_len):
    a = np.asarray(z[name])
    _need(a.ndim == 1 and a.shape[0] == shape_len and (a.size == 0 or np.issubdtype(a.dtype, np.integer)),
          f"{name}: expected {shape_len} integers, got {a.dtype} {a.shape}")
    return a.astype(np.int64)


def load_scene(path) -> Scene:
    """Reads and validates a scene file (keys in the module docstring). Raises SceneError on anything malformed."""
    path = Path(path)
    with np.load(path, allow_pickle=False) as z:
        keys = set(z.files)
        for k in ("num_frames", "cameras", "lidar2img", "box_frame", "labels"):
            _need(k in keys, f"{path.name}: missing {k!r}")
        nf = np.asarray(z["num_frames"])
        _need(nf.shape == () and np.issubdtype(nf.dtype, np.integer) and int(nf) >= 1, "num_frames: a positive integer")
        F = int(nf)
        cams = [str(c) for c in np.asarray(z["cameras"]).reshape(-1)]
        _need(sorted(cams) == sorted(CAMERA_VIEWS), f"cameras: expected each of {CAMERA_VIEWS} once, got {cams}")
        l2i = np.asarray(z["lidar2img"])
        _need(l2i.shape == (6, 4, 4), f"lidar2img: expected (6, 4, 4), got {l2i.shape}")
        _finite("lidar2img", l2i)
        l2i = l2i.astype(np.float32).astype(np.float64)
        _need(all(abs(np.linalg.det(m)) > 0 for m in l2i), "lidar2img: every matrix must be invertible")

        labels = np.asarray(z["labels"])
        M = labels.shape[0] if labels.ndim == 1 else -1
        _need(M >= 0, f"labels: expected a vector, got {labels.shape}")
        labels = _int_array(z, "labels", M)
        _need(((labels >= 0) & (labels < len(CLASS_NAMES))).all(), f"labels: class indices must lie in [0, {len(CLASS_NAMES)})")
        box_frame = _int_array(z, "box_frame", M)
        _need(((box_frame >= 0) & (box_frame < F)).all(), "box_frame: frame indices must lie in [0, num_frames)")
        _need(("corners" in keys) != ("boxes" in keys), "give exactly one of 'corners' and 'boxes'")
        if "corners" in keys:
            corners = np.asarray(z["corners"])
            _need(corners.shape == (M, 8, 3), f"corners: expected ({M}, 8, 3), got {corners.shape}")
            _finite("corners", corners)
        else:
            boxes = np.asarray(z["boxes"])
            _need(boxes.shape == (M, 7), f"boxes: expected ({M}, 7), got {boxes.shape}")
            _finite("boxes", boxes)
            _need((boxes[:, 3:6] > 0).all(), "boxes: sizes must be positive")
            corners = box_corners(boxes)
        corners = corners.astype(np.float32).astype(np.float64)     # LiDARInstance3DBoxes holds fp32

        map_keys = ("map_frame", "map_labels", "map_lengths", "map_points")
        polylines = [[] for _ in range(F)]
        if any(k in keys for k in map_keys):
            _need(all(k in keys for k in map_keys), f"map: give all of {map_keys}")
            L = np.asarray(z["map_lengths"]).reshape(-1).shape[0]
            lengths = _int_array(z, "map_lengths", L)
            mlabels = _int_array(z, "map_labels", L)
            mframe = _int_array(z, "map_frame", L)
            pts = np.asarray(z["map_points"])
            _need(pts.ndim == 2 and pts.shape[1] in (2, 3), f"map_points: expected (P, 2) or (P, 3), got {pts.shape}")
            _finite("map_points", pts)
            _need((lengths >= 2).all() and lengths.sum() == pts.shape[0], "map_lengths: each >= 2, summing to the points")
            _need(((mlabels >= 0) & (mlabels < len(MAP_CLASSES))).all(), f"map_labels: must lie in [0, {len(MAP_CLASSES)})")
            _need(((mframe >= 0) & (mframe < F)).all(), "map_frame: frame indices must lie in [0, num_frames)")
            pts = pts.astype(np.float64)
            if pts.shape[1] == 2:
                pts = np.concatenate([pts, np.zeros((pts.shape[0], 1))], 1)
            starts = np.concatenate([[0], np.cumsum(lengths)[:-1]])
            for i in range(L):
                polylines[mframe[i]].append((int(mlabels[i]), pts[starts[i]:starts[i] + lengths[i]]))
        prompt = str(z["prompt"]) if "prompt" in keys else None
        cond = path.parent / str(z["cond_frame"]) if "cond_frame" in keys else None
        files = None
        if "frame_files" in keys:
            ff = np.asarray(z["frame_files"])
            _need(ff.shape == (F,) and ff.dtype.kind == "U", f"frame_files: expected {F} paths, got {ff.dtype} {ff.shape}")
            files = [path.parent / str(f) for f in ff]
    return Scene(F, {c: l2i[i] for i, c in enumerate(cams)},
                 [corners[box_frame == f] for f in range(F)], [labels[box_frame == f] for f in range(F)],
                 [sorted(p, key=lambda e: e[0]) for p in polylines], prompt, cond, files)


def caption(labels) -> str:
    """The clip's caption when the scene file has none: the object count and the classes with their counts."""
    counts = np.bincount(np.asarray(labels, dtype=np.int64), minlength=len(CLASS_NAMES))
    parts = [f"{n} {CLASS_NAMES[i].replace('_', ' ')}" for i, n in enumerate(counts) if n]
    what = ", ".join(parts) if parts else "no annotated objects"
    return f"A street scene seen by six surround-view cameras, with {int(counts.sum())} objects: {what}."


# ------------------------------------------------------------------------------------------- host geometry (fp64)
def _convex_hull(p: np.ndarray) -> np.ndarray:
    """Counter-clockwise convex hull (monotone chain) of [n, 2] points, collinear points dropped."""
    pts = sorted(set(map(tuple, p.tolist())))
    if len(pts) < 3:
        return np.array(pts)

    def half(seq):
        out = []
        for q in seq:
            while len(out) >= 2 and ((out[-1][0] - out[-2][0]) * (q[1] - out[-2][1])
                                     - (out[-1][1] - out[-2][1]) * (q[0] - out[-2][0])) <= 0:
                out.pop()
            out.append(q)
        return out
    lower, upper = half(pts), half(reversed(pts))
    return np.array(lower[:-1] + upper[:-1])


def _clip_half_plane(poly, axis, bound, keep_below):
    """Sutherland-Hodgman against x_axis <= bound (keep_below) or >= bound; crossings put the clipped coordinate
    exactly on the bound."""
    inside = (lambda q: q[axis] <= bound) if keep_below else (lambda q: q[axis] >= bound)
    out = []
    for i in range(len(poly)):
        a, b = poly[i - 1], poly[i]
        if inside(b):
            if not inside(a):
                out.append(_crossing(a, b, axis, bound))
            out.append(b)
        elif inside(a):
            out.append(_crossing(a, b, axis, bound))
    return out


def _crossing(a, b, axis, bound):
    o = 1 - axis
    q = [0.0, 0.0]
    q[axis] = bound
    q[o] = a[o] + (bound - a[axis]) * (b[o] - a[o]) / (b[axis] - a[axis])
    return tuple(q)


def hull_canvas_bbox(points: np.ndarray, W: int, H: int):
    """Bounding box (xmin, ymin, xmax, ymax) of convex hull(points) intersected with the canvas [0, W] x [0, H], or None
    when that intersection has no area. The reference raises on an intersection without area (a hull that only
    touches the canvas, or a degenerate hull); here such a box is skipped."""
    poly = [tuple(q) for q in _convex_hull(points).tolist()]
    if len(poly) < 3:
        return None
    for axis, bound, below in ((0, 0.0, False), (0, float(W), True), (1, 0.0, False), (1, float(H), True)):
        poly = _clip_half_plane(poly, axis, bound, below)
        if not poly:
            return None
    q = np.array(poly)
    area = 0.5 * abs(np.dot(q[:, 0], np.roll(q[:, 1], -1)) - np.dot(q[:, 1], np.roll(q[:, 0], -1)))
    if len(poly) < 3 or area == 0.0:
        return None
    return q[:, 0].min(), q[:, 1].min(), q[:, 0].max(), q[:, 1].max()


def project_boxes(corners: np.ndarray, labels: np.ndarray, lidar2img: np.ndarray, H: int, W: int) -> dict:
    """The 2-D annotations of one panel (:414-475): corners projected with the depth clipped to DEPTH_CLIP before the
    divide; a box is kept when its mean clipped depth exceeds the lower clip and its hull meets the canvas, and dropped
    when its 2-D box is both wider than W - 100 and taller than H - 100. Returns bbox [n, 4], depth [n] (mean clipped
    depth), label [n] and corners [n, 8, 2] (image coordinates) of the kept boxes, in input order."""
    keep = {"bbox": [], "depth": [], "label": [], "corners": []}
    N = corners.shape[0]
    if N:
        p = np.concatenate([corners.reshape(-1, 3), np.ones((N * 8, 1))], axis=-1) @ lidar2img.T
        p[:, 2] = np.clip(p[:, 2], a_min=DEPTH_CLIP[0], a_max=DEPTH_CLIP[1])
        p[:, 0] /= p[:, 2]
        p[:, 1] /= p[:, 2]
        uv, dep = p[:, :2].reshape(N, 8, 2), p[:, 2].reshape(N, 8)
        for j in np.nonzero(dep.mean(1) > DEPTH_CLIP[0])[0]:
            bb = hull_canvas_bbox(uv[j], W, H)
            if bb is None or ((bb[2] - bb[0]) > W - 100 and (bb[3] - bb[1]) > H - 100):
                continue
            keep["bbox"].append(bb)
            keep["depth"].append(dep[j].mean())
            keep["label"].append(labels[j])
            keep["corners"].append(uv[j])
    return {"bbox": np.array(keep["bbox"], np.float64).reshape(-1, 4), "depth": np.array(keep["depth"], np.float64),
            "label": np.array(keep["label"], np.int64), "corners": np.array(keep["corners"], np.float64).reshape(-1, 8, 2)}


def resample_polyline(points: np.ndarray, num: int = MAP_SAMPLES) -> np.ndarray:
    """`num` points equally spaced in arc length along a polyline [k, 3], arc length measured in x-y (as shapely's
    LineString.length and interpolate measure it, z interpolated along)."""
    a, b = points[:-1], points[1:]
    dx, dy = a[:, 0] - b[:, 0], a[:, 1] - b[:, 1]
    seg = np.sqrt(dx * dx + dy * dy)
    cum = np.cumsum(seg)
    dist = np.linspace(0, cum[-1], num)
    idx = np.searchsorted(cum, dist, side="right")            # first segment whose end lies beyond the distance
    out = np.repeat(points[-1:], num, axis=0)
    inner = idx < len(seg)
    i = idx[inner]
    before = np.where(i > 0, cum[np.maximum(i - 1, 0)], 0.0)
    frac = (dist[inner] - before) / seg[i]
    p0, p1 = points[i], points[i + 1]
    pt = (p1 - p0) * frac[:, None] + p0
    pt = np.where((frac <= 0)[:, None], p0, np.where((frac >= 1)[:, None], p1, pt))
    out[inner] = pt
    return out


def project_polyline(samples: np.ndarray, lidar2img: np.ndarray, H: int, W: int) -> np.ndarray:
    """Integer pixel positions [k, 2] of the resampled points that are in front of the camera and inside
    [0, W-1) x [0, H-1), rounded (render.py:21-29, 53-64). Consecutive kept points are joined by a segment."""
    cam = (lidar2img @ np.concatenate([samples, np.ones([len(samples), 1])], axis=-1).T)[:3, :].T
    cam = cam[~np.isnan(cam[:, 0]) & ~np.isnan(cam[:, 1])]
    depth = cam[:, 2]
    uv = cam[:, :2] / cam[:, 2].reshape(-1, 1)
    ok = (0 <= uv[:, 0]) & (uv[:, 0] < W - 1) & (0 <= uv[:, 1]) & (uv[:, 1] < H - 1) & (depth > 0)
    return np.round(uv[ok]).astype(np.int64)


def ray_params(scene: Scene, H: int, w: int) -> np.ndarray:
    """[6 * 12 + 2] fp64 for pn_render_layout: per panel rows 0..2 of img2lidar (inverted in fp32 by torch, as the
    reference's dataset inverts it, :499), then the min and max ray component over all panels. The ray is affine in
    the pixel position, so its extremes lie at the panel corners."""
    l2i = np.stack([scene.lidar2img[c] for c in CAMERA_VIEWS]).astype(np.float32)
    img2lidar = torch.from_numpy(l2i).inverse().numpy().astype(np.float64)
    m = img2lidar[:, :3, :]                                       # [6, 3, 4]
    u = np.array([0.0, w - 1, 0.0, w - 1])[None, None, :]
    v = np.array([0.0, 0.0, H - 1, H - 1])[None, None, :]
    col = lambda k: m[:, :, k:k + 1]
    far = ((col(0) * (2.0 * u) + col(1) * (2.0 * v)) + col(2) * 2.0) + col(3)
    near = ((col(0) * u + col(1) * v) + col(2)) + col(3)
    d = far - near
    return np.concatenate([m.reshape(-1), [d.min(), d.max()]])


def panel_primitives(scene: Scene, frame: int, camera: str, H: int, W: int) -> np.ndarray:
    """[n, 16] fp32 records of pn_render_layout (include/panacea_b200.h) for one panel: depth rectangles, then the
    boxes far to near (fill key 2j, edges key 2j+1), then the map segments in drawing order."""
    l2i = scene.lidar2img[camera]
    ann = project_boxes(scene.corners[frame], scene.labels[frame], l2i, H, W)
    recs = []

    def rec(kind, key, rgb, radius, pts):
        r = np.zeros(_PRIM, np.float64)
        r[0], r[1], r[2:5], r[5] = kind, key, rgb, radius
        r[8:8 + len(pts)] = pts
        recs.append(r)
    for (x0, y0, x1, y1), d, lab in zip(ann["bbox"], ann["depth"], ann["label"]):
        rec(_RECT, lab, (int(d * 3), 0, 0), 0, (int(x0), int(y0), int(x1), int(y1)))
    order = np.argsort(ann["depth"])[::-1]
    for j, b in enumerate(order):
        col = BOX_PALETTE[ann["label"][b] + 1]
        c = ann["corners"][b].astype(np.int64)                    # int() of each coordinate (:325, 334)
        face = c[4:8].copy()
        face[:, 0] = np.clip(face[:, 0], 0, W)
        face[:, 1] = np.clip(face[:, 1], 0, H)
        rec(_QUAD, 2 * j, [int(v * 0.5 + 255 * 0.5) for v in col], 0, face.reshape(-1))
        for a, e in _BOX_EDGES:
            rec(_BOX_SEG, 2 * j + 1, col[::-1], _reach(BOX_LINE_WIDTH), (c[a, 0], c[a, 1], c[e, 0], c[e, 1]))
    segs, key = [], 0
    for cls, pts in scene.polylines[frame]:
        uv = project_polyline(resample_polyline(pts), l2i, H, W)
        n = max(len(uv) - 1, 0)
        r = np.zeros((n, _PRIM), np.float64)
        r[:, 0], r[:, 1], r[:, 2:5], r[:, 5] = _MAP_SEG, key + np.arange(n), MAP_COLORS_BGR[cls], _reach(MAP_LINE_WIDTH)
        r[:, 8:10], r[:, 10:12] = uv[:-1], uv[1:]
        segs.append(r)
        key += n
    return np.concatenate([np.array(recs, np.float64).reshape(-1, _PRIM)] + segs).astype(np.float32)


def render_layout(scene: Scene, frames, H: int, w: int, device="cuda") -> torch.Tensor:
    """The hint `cond_img` [T, 19, H, 6w] (fp32, on `device`) of the scene frames `frames`, in one kernel launch."""
    frames = list(frames)
    per_panel = [panel_primitives(scene, f, cam, H, w) for f in frames for cam in CAMERA_VIEWS]
    offsets = np.concatenate([[0], np.cumsum([len(p) for p in per_panel])]).astype(np.int32)
    prims = np.concatenate(per_panel + [np.zeros((1, _PRIM), np.float32)])    # never empty
    dev = torch.device(device)
    out = torch.empty(len(frames), HINT_CHANNELS, H, len(CAMERA_VIEWS) * w, dtype=torch.float32, device=dev)
    d_prims = torch.from_numpy(prims).to(dev)
    d_off = torch.from_numpy(offsets).to(dev)
    d_rays = torch.from_numpy(ray_params(scene, H, w)).to(dev)
    _lib.check(_lib.load().pn_render_layout(ptr(d_prims), ptr(d_off), ptr(d_rays), ptr(out), len(frames), H, w,
                                            _lib.stream(dev)), "pn_render_layout")
    return out


def _cell_mask(entry: str, T: int, H: int, w: int, dilate: int, sources) -> torch.Tensor:
    """[T, H/8, 6w/8] fp32 in {0, 1} from the cell-mask entry point `entry` over the device tensors `sources()`, which
    are made only once the size and `dilate` have passed their checks; dilated by `dilate` cells within each panel."""
    _need(H % LATENT_CELL == 0 and w % LATENT_CELL == 0, f"image size {H} x {w} is not a multiple of {LATENT_CELL}")
    _need(int(dilate) >= 0, f"dilate must be >= 0, got {dilate}")
    src = sources()
    out = torch.empty(T, H // LATENT_CELL, len(CAMERA_VIEWS) * w // LATENT_CELL, dtype=torch.float32, device=src[0].device)
    lib = _lib.load()
    _lib.check(getattr(lib, entry)(*map(ptr, src), ptr(out), T, H, w, LATENT_CELL, int(dilate), _lib.stream(out.device)), entry)
    return out


def change_mask(scene_a: Scene, scene_b: Scene, frames, image_hw, dilate: int = 1, device="cuda") -> torch.Tensor:
    """[T, H/8, 6w/8] fp32 in {0, 1} on `device`: 1 at the latent cells where the layout maps of the two scenes' frames
    `frames` differ in any channel, dilated by `dilate` cells within each panel (pn_layout_change_mask)."""
    if scene_a.num_frames != scene_b.num_frames:
        raise SceneError(f"the scenes hold {scene_a.num_frames} and {scene_b.num_frames} frames; a change mask needs the same count")
    H, w = image_hw
    frames = list(frames)
    return _cell_mask("pn_layout_change_mask", len(frames), H, w, dilate,
                      lambda: [render_layout(sc, frames, H, w, device) for sc in (scene_a, scene_b)])


def read_edit_mask(path, num_frames: int, image_hw) -> np.ndarray:
    """A user-drawn edit mask as uint8 [T, H, 6w] on the host, 1 where the clip is to be regenerated. An image file
    (read as greyscale, a pixel is set when >= 128) is one mask for every frame; a `.npy` file holds one mask per frame,
    bool or uint8 [T, H, 6w] (nonzero is set), since what is edited moves from frame to frame. Raises ValueError with
    the expected and the actual value when the shape, dtype or frame count is wrong."""
    from PIL import Image
    path = Path(path)
    H, w = image_hw
    want = (num_frames, H, len(CAMERA_VIEWS) * w)
    if path.suffix == ".npy":
        a = np.load(path, allow_pickle=False)
        if a.dtype not in (np.bool_, np.uint8):
            raise ValueError(f"{path.name}: expected a bool or uint8 array, got {a.dtype}")
        if a.ndim != 3:
            raise ValueError(f"{path.name}: expected shape {want} (frames, H, 6w), got {a.shape}")
        if a.shape[0] != num_frames:
            raise ValueError(f"{path.name}: expected {num_frames} frames, got {a.shape[0]}")
        if a.shape != want:
            raise ValueError(f"{path.name}: expected shape {want} (frames, H, 6w), got {a.shape}")
        return (a != 0).astype(np.uint8)
    img = np.asarray(Image.open(path).convert("L"))
    if img.shape != want[1:]:
        raise ValueError(f"{path.name}: expected a {want[2]} x {want[1]} image, got {img.shape[1]} x {img.shape[0]}")
    return np.ascontiguousarray(np.broadcast_to((img >= 128).astype(np.uint8), want))


def mask_cells(pixels, dilate: int = 1, device="cuda") -> torch.Tensor:
    """[T, H/8, 6w/8] fp32 in {0, 1} on `device`, the form of `change_mask`: 1 at the latent cells holding a nonzero
    pixel of `pixels` (uint8 [T, H, 6w], e.g. from `read_edit_mask`), dilated by `dilate` cells within each panel
    (pn_mask_cells)."""
    pixels = torch.as_tensor(np.ascontiguousarray(pixels, dtype=np.uint8))
    _need(pixels.dim() == 3 and pixels.shape[2] % len(CAMERA_VIEWS) == 0, f"expected uint8 [T, H, 6w], got {tuple(pixels.shape)}")
    T, H, Wt = pixels.shape
    return _cell_mask("pn_mask_cells", T, H, Wt // len(CAMERA_VIEWS), dilate, lambda: [pixels.to(device)])
