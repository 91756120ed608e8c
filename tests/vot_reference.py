"""TEST INFRASTRUCTURE ONLY (checker) for the VOT protocol (siammask_b200/vot.py, C ABI `sm_vot_overlap`).  Nothing
under `siammask_b200/` imports this module.

`polygon_overlap` restates the VOT toolkit's `compute_polygon_overlap` (non-legacy rasteriser, bounds (0, 0, W, H)) in
plain Python / numpy the way the C code runs it: float32 where C uses float, Python floats where it uses double, full
per-polygon masks.  `track_vot` restates tools/test.py:318-366 for one sequence ('VOT' dataset, mask_enable=False) on
top of `oracle.ref_loop.siamese_init` / `siamese_track`, and `result_lines` the result-file writer of :402-406.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import ref_loop

f32 = np.float32


def _c_round(v: float) -> float:
    t = float(math.trunc(v))
    return t + math.copysign(1.0, v) if abs(v - t) >= 0.5 else t


def _bounds(p):
    """compute_bounds + bounds_round of 4 float32 points: (left, top, right, bottom) float32."""
    xs, ys = p[0::2], p[1::2]
    left, top, right, bottom = f32(np.inf), f32(np.inf), f32(-np.inf), f32(-np.inf)
    for x, y in zip(xs, ys):
        top, bottom = (y if y < top else top), (y if y > bottom else bottom)
        left, right = (x if x < left else left), (x if x > right else right)
    return [f32(math.floor(left)), f32(math.floor(top)), f32(math.ceil(right)), f32(math.ceil(bottom))]


def _cmax(a, b):
    return a if a > b else b


def _cmin(a, b):
    return a if a < b else b


def _clip(b, W, H):
    return [_cmax(b[0], f32(0)), _cmax(b[1], f32(0)), _cmin(b[2], f32(W)), _cmin(b[3], f32(H))]


def _area(b):
    return f32(f32(b[2] - b[0]) * f32(b[3] - b[1]))


def _rasterize(xs, ys, width, height):
    """rasterize_polygon, non-legacy branch, on the rounded polygon: uint8 mask [height, width]."""
    mask = np.zeros((height, width), np.uint8)
    n = len(xs)
    for py in range(height):
        nodes = []
        j = n - 1
        for i in range(n):
            yi, yj = int(ys[i]), int(ys[j])
            if (yi <= py < yj) or (yj <= py < yi) or (yi < py <= yj) or (yj < py <= yi) or (yi == yj == py):
                r = float(f32(ys[j] - ys[i]))
                k = float(f32(xs[j] - xs[i]))
                if r != 0:
                    nodes.append(int(float(xs[i]) + float(f32(f32(py) - ys[i])) / r * k))
            j = i
        nodes.sort()
        i = 0
        while i < len(nodes) - 1:
            if nodes[i] == nodes[i + 1]:
                i += 1
                continue
            if nodes[i] >= width:
                break
            if nodes[i + 1] >= 0:
                a, b = max(nodes[i], 0), min(nodes[i + 1], width - 1)
                mask[py, a:b + 1] = 1
            i += 2
    return mask


def polygon_overlap(poly_a, poly_b, W: int, H: int) -> np.float32:
    """compute_polygon_overlap(poly_a, poly_b, bounds (0, 0, W, H)) for two 8-value polygons (rounded to float32 first,
    as pyvotkit's Polygon stores them).  An empty union gives the NaN 0xFFC00000, as x86 computes 0.0f / 0.0f."""
    pa, pb = np.asarray(poly_a, np.float32).reshape(8), np.asarray(poly_b, np.float32).reshape(8)
    b1, b2 = _clip(_bounds(pa), W, H), _clip(_bounds(pb), W, H)
    x, y = _cmin(b1[0], b2[0]), _cmin(b1[1], b2[1])
    width = int(f32(_cmax(b1[2], b2[2]) - x)) + 1
    height = int(f32(_cmax(b1[3], b2[3]) - y)) + 1
    a1, a2 = float(_area(b1)), float(_area(b2))

    def div(a, b):                                   # C double division: +-inf or NaN where b == 0
        if b == 0:
            return math.nan if a == 0 or math.isnan(a) else math.copysign(math.inf, a) * math.copysign(1.0, b)
        return a / b
    if div(a1, a2) < 1e-10 or div(a2, a1) < 1e-10 or width < 1 or height < 1:
        return f32(0)
    bi = [_cmax(b1[0], b2[0]), _cmax(b1[1], b2[1]), _cmin(b1[2], b2[2]), _cmin(b1[3], b2[3])]
    inter = _area(bi)
    den = f32(f32(_area(b1) + _area(b2)) - inter)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = f32(inter / den)
    if (f32(0) if f32(0) > q else q) == 0:
        return f32(0)
    masks = []
    for p in (pa, pb):
        xs = [f32(_c_round(float(f32(v - x)))) for v in p[0::2]]
        ys = [f32(_c_round(float(f32(v - y)))) for v in p[1::2]]
        masks.append(_rasterize(xs, ys, width, height))
    m1, m2 = masks[0].astype(bool), masks[1].astype(bool)
    inter_n, union_n = int((m1 & m2).sum()), int((m1 | m2).sum())
    if union_n == 0:
        return np.array([0xFFC00000], np.uint32).view(np.float32)[0]
    return f32(f32(inter_n) / f32(union_n))


def get_axis_aligned_bbox(region):
    """utils/bbox_helper.py:52-75 for an 8-value polygon, in float64 numpy: the vertices' centre, and their axis-aligned
    extent scaled by sqrt(|p0 p1| * |p1 p2| / extent area), plus one pixel.  (cx, cy, w, h)."""
    pts = np.asarray(region, np.float64).reshape(4, 2)
    centre = pts.mean(axis=0)
    extent = pts.max(axis=0) - pts.min(axis=0)
    scale = np.sqrt(np.linalg.norm(pts[0] - pts[1]) * np.linalg.norm(pts[1] - pts[2]) / (extent[0] * extent[1]))
    size = scale * extent + 1
    return centre[0], centre[1], size[0], size[1]


def track_vot(model, frames, gt, hp, overlap=polygon_overlap, device="cuda"):
    """tools/test.py:318-366 for one VOT sequence, mask_enable=False: frames (numpy HWC or uint8 CUDA tensors), gt
    float64 [T, 8], the hp dict of siamese_init.  Returns (regions, lost_times)."""
    regions = []
    start_frame, lost_times = 0, 0
    for f, im in enumerate(frames):
        if f == start_frame:  # init
            cx, cy, w, h = get_axis_aligned_bbox(gt[f])
            target_pos = np.array([cx, cy])
            target_sz = np.array([w, h])
            state = ref_loop.siamese_init(im, target_pos, target_sz, model, hp, device=device)
            regions.append(1)
        elif f > start_frame:  # tracking
            state = ref_loop.siamese_track(state, im, False, False, device=device)
            pos, sz = state["target_pos"], state["target_sz"]
            location = np.array([pos[0] - sz[0] / 2, pos[1] - sz[1] / 2, sz[0], sz[1]])
            gt_polygon = ((gt[f][0], gt[f][1]), (gt[f][2], gt[f][3]), (gt[f][4], gt[f][5]), (gt[f][6], gt[f][7]))
            pred_polygon = ((location[0], location[1]), (location[0] + location[2], location[1]),
                            (location[0] + location[2], location[1] + location[3]),
                            (location[0], location[1] + location[3]))
            H, W = (im.shape[0], im.shape[1])
            b_overlap = overlap(np.asarray(gt_polygon).reshape(8), np.asarray(pred_polygon).reshape(8), W, H)
            if b_overlap:
                regions.append(location)
            else:  # lost
                regions.append(2)
                lost_times += 1
                start_frame = f + 5  # skip 5 frames
        else:  # skip
            regions.append(0)
    return regions, lost_times


def result_lines(regions, float2str) -> str:
    """The VOT result file of tools/test.py:402-406; float2str(v) formats one value as vot_float2str("%.4f", v)."""
    out = ""
    for x in regions:
        out += "{:d}\n".format(x) if isinstance(x, int) else ",".join(float2str(i) for i in x) + "\n"
    return out
