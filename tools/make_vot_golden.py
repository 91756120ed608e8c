"""Generates tests/golden/vot_overlap.npz from the reference's own code.  TEST INFRASTRUCTURE ONLY; it needs the
reference source tree (SIAMMASK_REFERENCE) and the region library `oracle/build_ref.py` compiles from it:

    python tools/make_vot_golden.py

Overlaps come from the reference's compute_polygon_overlap (pyvotkit's region.c, called as vot_overlap calls it) on
seeded polygon pairs; the bbox rows from its utils/bbox_helper.get_axis_aligned_bbox.  Cases:
  random quads and rotated rectangles; axis-aligned boxes at integer and exact .5 coordinates (rounding half away from
  zero); polygons partly or wholly outside the frame and past column W; zero-area, collinear and single-point polygons
  and bow-ties; duplicate nodes; tiny against huge; disjoint bounding boxes; identical degenerate polygons (NaN); frame
  sizes from 1x1 to 1920x1080.  With bounds (0, 0, W, H) the a1 / a2 < 1e-10 exit fires only when a clipped box area is
  zero or negative (a positive area is at least 1 and at most (W+1)(H+1)); the zero-area and outside rows take it.
"""
from __future__ import annotations

import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "vot_overlap.npz")
SIZES = [(1, 1), (2, 3), (17, 9), (320, 240), (640, 360), (1280, 720), (1920, 1080)]


def _rect(x, y, w, h):
    return [x, y, x + w, y, x + w, y + h, x, y + h]


def _rotated(cx, cy, w, h, a):
    c, s = np.cos(a), np.sin(a)
    pts = [(-w / 2, -h / 2), (w / 2, -h / 2), (w / 2, h / 2), (-w / 2, h / 2)]
    return [v for dx, dy in pts for v in (cx + c * dx - s * dy, cy + s * dx + c * dy)]


def pairs(rng):
    """(poly_a, poly_b, (W, H)) rows covering the cases of the module docstring."""
    out = []
    for W, H in SIZES:
        def rnd(n):
            return rng.uniform(-0.2 * W - 5, 1.2 * W + 5, n), rng.uniform(-0.2 * H - 5, 1.2 * H + 5, n)

        for _ in range(12):                                              # random quads (often self-intersecting)
            xa, ya = rnd(4)
            xb, yb = rnd(4)
            out.append((np.stack([xa, ya], 1).ravel(), np.stack([xb, yb], 1).ravel(), (W, H)))
        for _ in range(12):                                              # rotated rectangles vs axis-aligned boxes
            cx, cy = rng.uniform(0, W), rng.uniform(0, H)
            w, h = rng.uniform(1, W / 2 + 2), rng.uniform(1, H / 2 + 2)
            a = _rotated(cx, cy, w, h, rng.uniform(-np.pi, np.pi))
            b = _rect(cx - w / 2 + rng.uniform(-w / 4, w / 4), cy - h / 2 + rng.uniform(-h / 4, h / 4), w, h)
            out.append((a, b, (W, H)))
        for _ in range(8):                                               # integer and .5 coordinates
            x, y = rng.randint(-3, W + 3), rng.randint(-3, H + 3)
            w, h = rng.randint(0, W // 2 + 3), rng.randint(0, H // 2 + 3)
            a = np.asarray(_rect(x, y, w, h), float) + rng.choice([0.0, 0.5, -0.5], 8)
            b = np.asarray(_rect(x + rng.randint(-2, 3), y + rng.randint(-2, 3), w, h), float) + 0.5
            out.append((a, b, (W, H)))
        out.append((_rect(W - 3.5, 0.5, 10, H / 2 + 1), _rect(W - 1, 0, 4, H), (W, H)))      # past column W
        out.append((_rect(-50, -50, 20, 20), _rect(W + 10, H + 10, 5, 5), (W, H)))           # wholly outside
        out.append((_rect(W + 20, 1, 10, 10), _rect(1, H + 20, 10, 10), (W, H)))             # outside, two sides
        out.append((_rect(0, 0, W, H), _rect(-1, -1, W + 2, H + 2), (W, H)))                 # the whole frame
        out.append(([1.2, 1.2] * 4, [1.2, 1.2] * 4, (W, H)))                                 # one point twice: NaN
        out.append(([0.5, 0.5, W * 0.7, H * 0.7, W * 0.35, H * 0.35, 0.5, 0.5], _rect(0, 0, W, H), (W, H)))  # collinear
        out.append(([0, 0, W / 2, 0, W / 2, 0, 0, 0], _rect(0, 0, W, H), (W, H)))            # zero area
        out.append(([0, 0, W, H, W, 0, 0, H], _rect(W / 4, H / 4, W / 2, H / 2), (W, H)))    # bow-tie
        out.append((_rect(2, 2, W / 2, H / 2), [2, 2, 2, 2, 2 + W / 2, 2, 2, 2 + H / 2], (W, H)))  # duplicate node
        out.append((_rect(W / 2, H / 2, 1e-3, 1e-3), _rect(-1e5, -1e5, 2e5, 2e5), (W, H)))  # tiny vs huge
        out.append((_rect(0, 0, W / 3, H / 3), _rect(W / 2, H / 2, W / 3, H / 3), (W, H)))  # disjoint boxes
    # the smallest positive area ratio the clipped bounds allow: a 1x1 box against the whole 1920x1080 frame (4.8e-7,
    # above the 1e-10 exit)
    out.append((_rect(5, 5, 1, 1), _rect(-100, -100, 1e6, 1e6), (1920, 1080)))
    return out


def reference_bbox():
    ref = os.environ.get("SIAMMASK_REFERENCE", "/root/reference")
    spec = importlib.util.spec_from_file_location("ref_bbox_helper", os.path.join(ref, "utils", "bbox_helper.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.get_axis_aligned_bbox


def main():
    from oracle import build_ref
    if build_ref.build() is None:
        raise SystemExit("the reference tree is required")
    lib = build_ref.load()
    rng = np.random.RandomState(2024)
    rows = pairs(rng)
    a = np.asarray([np.asarray(r[0], np.float64) for r in rows]).astype(np.float32)
    b = np.asarray([np.asarray(r[1], np.float64) for r in rows]).astype(np.float32)
    size = np.asarray([r[2] for r in rows], np.int32)
    ov = np.asarray([lib.overlap(a[i], b[i], *size[i]) for i in range(len(rows))], np.float32)
    # get_axis_aligned_bbox rows: rotated rectangles, random quads and axis-aligned boxes with .5 coordinates
    bb_in = [np.asarray(_rotated(*rng.uniform(20, 600, 2), *rng.uniform(5, 200, 2), rng.uniform(-3, 3)))
             for _ in range(40)]
    bb_in += [rng.uniform(0, 1000, 8) for _ in range(20)]
    bb_in += [np.asarray(_rect(*rng.randint(0, 500, 2), *rng.randint(1, 300, 2)), float) + 0.5 for _ in range(10)]
    bb_in = np.asarray(bb_in, np.float64)
    gab = reference_bbox()
    bb_out = np.asarray([gab(r) for r in bb_in], np.float64)
    np.savez_compressed(OUT, poly_a=a, poly_b=b, size=size, overlap_bits=ov.view(np.uint32), bbox_in=bb_in,
                        bbox_out=bb_out)
    print(f"wrote {OUT}: {len(rows)} pairs ({int(np.isnan(ov).sum())} NaN, {int((ov == 0).sum())} zero), "
          f"{len(bb_in)} bbox rows")


if __name__ == "__main__":
    main()
