"""Writes tests/golden/layout_*.pt: two seeded scenes rendered by the reference's own dataset code.

Runs on a CPU development box that has the reference tree and OpenCV (cv2); nothing on the GPU side needs either. It
imports the unmodified drawing methods of sgm/data/nuscenes_video/nuscenes_datasets_video.py (MyDataset._get_2d_annos,
draw_bboxes, draw_corners, render_directions) and render.py (Renderer.render_camera_views_from_vectors), with minimal
stand-ins for the packages they import but this box does not have: shapely's MultiPoint.convex_hull, box and
LineString.interpolate are restated below, mmcv's DataContainer and the nuScenes / mmdet / mmdet3d imports are empty.

Each golden holds the scene file's arrays, the reference's uint8 hint [T, 16, H, 6w] for channels 0..15 and
[3, H, 6w] for the ray channels (the same in every frame, since the cameras do not change; checked here), zlib-packed,
and its intermediates: per frame and panel the 2-D boxes, depths, labels and projected corners, and the kept,
rounded points of every polyline. Box corners are made from centre, size and yaw with the mmdet3d formula in fp32.

  python tools/make_layout_golden.py [--reference /path/to/reference]
"""
from __future__ import annotations

import argparse
import importlib.util
import math
import sys
import types
import zlib
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
CAMERA_VIEWS = ["CAM_FRONT", "CAM_FRONT_RIGHT", "CAM_BACK_RIGHT", "CAM_BACK", "CAM_BACK_LEFT", "CAM_FRONT_LEFT"]
DATA_ORDER = ["CAM_FRONT", "CAM_FRONT_RIGHT", "CAM_FRONT_LEFT", "CAM_BACK", "CAM_BACK_LEFT", "CAM_BACK_RIGHT"]
CAM_YAW = {"CAM_FRONT": 0.0, "CAM_FRONT_RIGHT": -55.0, "CAM_BACK_RIGHT": -110.0, "CAM_BACK": 180.0,
           "CAM_BACK_LEFT": 110.0, "CAM_FRONT_LEFT": 55.0}


# ----------------------------------------------------------------------------------------------- shapely stand-in
class _Coords:
    def __init__(self, pts):
        self.coords = [tuple(p) for p in pts]


class _Polygon:
    def __init__(self, pts):
        self.pts = [tuple(p) for p in pts]
        self.exterior = _Coords(self.pts + self.pts[:1])

    def intersects(self, other):
        return len(_clip(self.pts, other.bounds)) > 0

    def intersection(self, other):
        pts = _clip(self.pts, other.bounds)
        area = 0.5 * abs(sum(pts[i - 1][0] * pts[i][1] - pts[i][0] * pts[i - 1][1] for i in range(len(pts))))
        if len(pts) < 3 or area == 0:
            raise ValueError("intersection without area (shapely returns a line or point, which has no exterior)")
        return _Polygon(pts)


def _box(x0, y0, x1, y1):
    p = _Polygon([(x0, y0), (x1, y0), (x1, y1), (x0, y1)])
    p.bounds = (x0, y0, x1, y1)
    return p


def _hull(points):
    """Gift wrapping, counter-clockwise, collinear points dropped."""
    pts = sorted(set(tuple(map(float, p[:2])) for p in points))
    if len(pts) < 3:
        raise ValueError("degenerate hull")
    cross = lambda o, a, b: (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])
    hull, cur = [], pts[0]
    while True:
        hull.append(cur)
        nxt = pts[0] if pts[0] != cur else pts[1]
        for q in pts:
            c = cross(cur, nxt, q)
            if c < 0 or (c == 0 and math.dist(cur, q) > math.dist(cur, nxt)):
                nxt = q
        cur = nxt
        if cur == hull[0]:
            return hull


def _clip(poly, bounds):
    x0, y0, x1, y1 = bounds
    for axis, b, keep in ((0, x0, lambda v, b: v >= b), (0, x1, lambda v, b: v <= b),
                          (1, y0, lambda v, b: v >= b), (1, y1, lambda v, b: v <= b)):
        out, o = [], 1 - axis
        for i in range(len(poly)):
            p, q = poly[i - 1], poly[i]
            pin, qin = keep(p[axis], b), keep(q[axis], b)
            if pin != qin:
                c = [0.0, 0.0]
                c[axis] = b
                c[o] = p[o] + (b - p[axis]) * (q[o] - p[o]) / (q[axis] - p[axis])
                out.append(tuple(c))
            if qin:
                out.append(q)
        poly = out
        if not poly:
            return []
    return poly


class _MultiPoint:
    def __init__(self, pts):
        self.convex_hull = _Polygon(_hull(np.asarray(pts)))


class _LineString:
    """GEOS LengthIndexedLine semantics: length and distances in x-y, z interpolated along."""

    def __init__(self, pts):
        self.pts = np.asarray(pts, dtype=np.float64)
        self.seg = [math.sqrt((b[0] - a[0]) ** 2 + (b[1] - a[1]) ** 2) for a, b in zip(self.pts[:-1], self.pts[1:])]
        total = 0.0
        for s in self.seg:
            total += s
        self.length = total

    def interpolate(self, d):
        total = 0.0
        for i, s in enumerate(self.seg):
            if total + s > d:
                frac = (d - total) / s
                p0, p1 = self.pts[i], self.pts[i + 1]
                if frac <= 0:
                    return _Coords([p0])
                if frac >= 1:
                    return _Coords([p1])
                return _Coords([(p1 - p0) * frac + p0])
            total += s
        return _Coords([self.pts[-1]])


def _load_reference(ref: Path):
    stubs = {
        "shapely": {}, "shapely.geometry": {"MultiPoint": _MultiPoint, "box": _box, "LineString": _LineString},
        "mmcv": {}, "mmcv.parallel": {"DataContainer": type("DataContainer", (), {})},
        "projects": {}, "projects.mmdet3d_plugin": {}, "projects.mmdet3d_plugin.datasets": {"CustomNuScenesDataset": None},
        "nuscenes": {}, "nuscenes.utils": {}, "nuscenes.utils.data_classes": {"Box": None},
        "pyquaternion": {"Quaternion": None}, "mmdet": {}, "mmdet.datasets": {}, "mmdet.datasets.builder": {"PIPELINES": None},
        "einops": {"rearrange": None}, "matplotlib": {}, "matplotlib.pyplot": {},
    }
    for name, attrs in stubs.items():
        mod = types.ModuleType(name)
        mod.__dict__.update(attrs)
        sys.modules[name] = mod
    src = ref / "sgm" / "data" / "nuscenes_video"
    sys.path.insert(0, str(src))
    import render                                                     # noqa: E402  (the reference's render.py)
    spec = importlib.util.spec_from_file_location("ref_nuscenes_dataset", src / "nuscenes_datasets_video.py")
    ds = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ds)
    return ds, render


# ----------------------------------------------------------------------------------------------- scenes
def _lidar2img(cam, H, W):
    f = 0.79 * W
    K = np.array([[f, 0, W / 2, 0], [0, f, H / 2 + 6, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    yaw = math.radians(CAM_YAW[cam])
    fwd, left = np.array([math.cos(yaw), math.sin(yaw), 0.0]), np.array([-math.sin(yaw), math.cos(yaw), 0.0])
    R = np.stack([-left, [0.0, 0.0, -1.0], fwd])                      # camera x right, y down, z forward
    pos = np.array([1.0, 0.0, 1.6]) + 0.8 * fwd
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, -R @ pos
    return (K @ E).astype(np.float32)


def _corners(boxes):
    """mmdet3d LiDARInstance3DBoxes.corners in fp32 torch."""
    b = torch.from_numpy(boxes).float()
    unit = torch.tensor([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]],
                        dtype=torch.float32) - torch.tensor([0.5, 0.5, 0.0])
    local = b[:, None, 3:6] * unit[None]
    c, s = torch.cos(b[:, 6]), torch.sin(b[:, 6])
    rot_t = torch.stack([torch.stack([c, s, torch.zeros_like(c)], -1), torch.stack([-s, c, torch.zeros_like(c)], -1),
                         torch.tensor([0.0, 0.0, 1.0]).expand(len(b), 3)], 1)          # rotation_3d_in_axis, axis 2
    return (torch.einsum("naj,njk->nak", local, rot_t) + b[:, None, :3]).numpy()


def make_scene(seed, T, H, W):
    rng = np.random.default_rng(seed)
    boxes, labels, frames, lines = [], [], [], []
    for t in range(T):
        dx = -1.2 * t                                                  # the ego drives forward along x
        fixed = [
            ([9.0, 6.4, 0.0, 4.4, 1.9, 1.6, 0.3], 0),                  # across the front panel's left edge
            ([1.0, 2.6, 0.0, 4.6, 1.9, 1.7, 0.05], 0),                 # beside the ego: partly behind several cameras
            ([4.5, 0.0, -0.5, 14.0, 6.0, 5.0, 0.0], 1),                # fills the front panel: dropped
            ([14.0, -1.0, 0.0, 4.5, 1.9, 1.6, 0.1], 0),                # two overlapping cars
            ([16.5, -1.4, 0.0, 4.5, 1.9, 1.6, -0.1], 0),
            ([-12.0, 3.0, 0.0, 0.7, 0.7, 1.8, 0.0], 8),
        ]
        for b, lab in fixed:
            boxes.append([b[0] + (dx if lab != 1 else 0.0), *b[1:]])
            labels.append(lab)
            frames.append(t)
        for _ in range(int(rng.integers(8, 14))):
            ang, r = rng.uniform(-math.pi, math.pi), rng.uniform(4.0, 45.0)
            lab = int(rng.integers(0, 10))
            size = {0: (4.5, 1.9, 1.6), 1: (7.0, 2.5, 3.0), 3: (11.0, 2.9, 3.4), 8: (0.7, 0.7, 1.8)}.get(lab, (1.5, 1.0, 1.2))
            boxes.append([r * math.cos(ang), r * math.sin(ang), rng.uniform(-0.3, 0.3), *size, rng.uniform(-math.pi, math.pi)])
            labels.append(lab)
            frames.append(t)
        xs = np.linspace(-30, 30, 7)
        for y, cls in ((1.75, 1), (-1.75, 1), (5.25, 1), (7.5, 2), (-7.5, 2)):
            pts = np.stack([xs + dx % 6, y + 0.3 * np.sin(xs / 9 + seed)], 1)
            lines.append((t, cls, pts))
        lines.append((t, 0, np.array([[12 + dx, -6.0], [12 + dx, 6.0], [15 + dx, 6.0], [15 + dx, -6.0], [12 + dx, -6.0]])))
        # leaves the front panel to the right and comes back
        lines.append((t, 2, np.array([[8.0, 0.0], [10.0, -9.0], [14.0, -12.0], [20.0, -3.0], [30.0, 0.0]])))
        # behind the front camera, and one from behind to in front of it
        lines.append((t, 1, np.array([[-6.0, -3.0, 0.0], [-20.0, -3.0, 0.2]])))
        lines.append((t, 0, np.array([[-4.0, 0.5], [6.0, 0.5]])))
    boxes = np.array(boxes, np.float64)
    corners = _corners(boxes)
    return {
        "num_frames": np.array(T), "cameras": np.array(DATA_ORDER),
        "lidar2img": np.stack([_lidar2img(c, H, W) for c in DATA_ORDER]),
        "box_frame": np.array(frames), "labels": np.array(labels), "corners": corners,
        "map_frame": np.array([l[0] for l in lines]), "map_labels": np.array([l[1] for l in lines]),
        "map_lengths": np.array([len(l[2]) for l in lines]),
        "map_points": np.concatenate([np.pad(l[2], ((0, 0), (0, 3 - l[2].shape[1]))) for l in lines]),
    }, boxes


def render_reference(ds, render, scene, H, W):
    """The reference's hint of every frame (uint8 channels 0..15, rays 16..18) and its intermediates."""
    me = types.SimpleNamespace(classes=ds.class_names, viewid={c: DATA_ORDER.index(c) for c in CAMERA_VIEWS})
    T = int(scene["num_frames"])
    l2i = scene["lidar2img"]
    colors = np.array([[255, 255, 255], [128, 64, 128], [244, 35, 232], [70, 70, 70], [102, 102, 156], [190, 153, 153],
                       [153, 153, 153], [250, 170, 30], [220, 220, 0], [107, 142, 35], [152, 251, 152], [0, 130, 180],
                       [220, 20, 60], [255, 0, 0], [0, 0, 142], [0, 0, 70], [0, 60, 100], [0, 80, 100], [0, 0, 230],
                       [119, 11, 32]])
    kept, orig_draw = [], render.draw_visible_polyline_cv2
    orig_poly = render.draw_polyline_ego_on_img

    def record_line(line, **kw):
        kept[-1] = np.array(line, np.int64)
        return orig_draw(line, **kw)

    def record_poly(*a, **kw):
        kept.append(np.zeros((0, 2), np.int64))
        return orig_poly(*a, **kw)
    render.draw_visible_polyline_cv2, render.draw_polyline_ego_on_img = record_line, record_poly
    renderer = render.Renderer(ds.cat2id_map, ds.roi_size, "nusc")
    starts = np.concatenate([[0], np.cumsum(scene["map_lengths"])[:-1]])
    img = np.zeros((H, W, 3), np.uint8)
    hint, inter, rays = [], [], None
    for t in range(T):
        sel = scene["box_frame"] == t
        ann = ds.MyDataset._get_2d_annos(me, (H, W), None, scene["corners"][sel], scene["labels"][sel], l2i)
        panels, frame_inter = [], {"bbox": [], "depth": [], "label": [], "corners": [], "lines": []}
        for view in CAMERA_VIEWS:
            v = me.viewid[view]
            b, lab, dep, cor = (ann[k][v] for k in ("gt_bbox2d", "gt_label2d", "gt_depth2d", "gt_corners3d"))
            depth_img = ds.MyDataset.draw_bboxes(me, img, b, lab, dep, colors)
            corner_img = ds.MyDataset.draw_corners(me, img, cor, lab, dep, colors, linewidth=2)
            panels.append(np.concatenate([corner_img, depth_img], -1))
            for k, x in (("bbox", b), ("depth", dep), ("label", lab), ("corners", cor)):
                frame_inter[k].append(torch.from_numpy(np.asarray(x, np.float64 if k != "label" else np.int64)))
        vectors = {c: [] for c in range(3)}
        for i in np.nonzero(scene["map_frame"] == t)[0]:
            vectors[int(scene["map_labels"][i])].append(scene["map_points"][starts[i]:starts[i] + scene["map_lengths"][i]].copy())
        kept.clear()
        maps = renderer.render_camera_views_from_vectors(vectors, [img] * 6, np.stack([l2i[me.viewid[c]] for c in CAMERA_VIEWS]), 4, None)
        n_lines = sum(len(x) for x in vectors.values())
        assert len(kept) == 6 * n_lines
        frame_inter["lines"] = [[torch.from_numpy(kept[p * n_lines + j]) for j in range(n_lines)] for p in range(6)]
        m = np.concatenate(maps, 1)
        assert (m == np.round(m)).all() and m.min() >= 0 and m.max() <= 255     # LINE_AA does not blend on float64
        img2lidar = torch.from_numpy(l2i).inverse().numpy()
        r = np.concatenate(ds.MyDataset.render_directions(me, (H, W, 3), img2lidar, CAMERA_VIEWS), 1)
        assert rays is None or np.array_equal(rays, r)
        rays = r
        hint.append(np.concatenate([np.concatenate(panels, 1), m.astype(np.uint8)], -1).transpose(2, 0, 1))
        inter.append(frame_inter)
    render.draw_visible_polyline_cv2, render.draw_polyline_ego_on_img = orig_draw, orig_poly
    return np.stack(hint), rays.transpose(2, 0, 1).copy(), inter


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default="/root/reference")
    args = ap.parse_args()
    ds, render = _load_reference(Path(args.reference))
    for name, seed, (H, W) in (("layout_448", 1, (256, 448)), ("layout_512", 2, (256, 512))):
        scene, boxes = make_scene(seed, 8, H, W)
        hint, rays, inter = render_reference(ds, render, scene, H, W)
        pack = lambda a: {"shape": list(a.shape), "zlib": zlib.compress(np.ascontiguousarray(a, np.uint8).tobytes(), 9)}
        out = {"image_hw": (H, W), "scene": {k: torch.from_numpy(np.asarray(v)) if v.dtype.kind != "U" else [str(c) for c in v]
                                             for k, v in scene.items()},
               "boxes": torch.from_numpy(boxes), "hint_0_15": pack(hint), "rays": pack(rays), "intermediates": inter}
        path = ROOT / "tests" / "golden" / f"{name}.pt"
        torch.save(out, path)
        print(f"{path}: {path.stat().st_size / 1e6:.2f} MB, hint {hint.shape}")


if __name__ == "__main__":
    main()
