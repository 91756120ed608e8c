"""TEST INFRASTRUCTURE ONLY (checker) for `siammask_b200.rotated_box` (C ABI `sm_rotated_box_ragged`): SiamMask's
rotated box of tools/test.py:284-303 restated in numpy, one mask at a time.

The reference thresholds the pasted mask, runs cv2.findContours(RETR_EXTERNAL, CHAIN_APPROX_NONE), takes the contour
with the largest cv2.contourArea (np.argmax: the first maximum) and, if that area is over 100, returns
cv2.boxPoints(cv2.minAreaRect(contour)); otherwise the rectangle cxy_wh_2_rect(target_pos, target_sz) of the state
before its clamps.  Here:

  * components: 8-connected components of the foreground; pixels outside the frame are background;
  * contour area: the outer border of each component followed as Suzuki & Abe (1985) do from its raster-first pixel,
    doubled shoelace area through the pixel centres (an exact integer; cv2.contourArea is half of it);
  * selection: the largest area; on equal areas the component whose raster-first pixel is last in raster order
    (cv2 4.x returns RETR_EXTERNAL contours in reverse raster order of those pixels, and np.argmax takes the first);
    the contour is used only if its area is over 100;
  * rectangle: over the edges of the convex hull of the component's pixel centres (Andrew's monotone chain over the
    row-wise leftmost and rightmost pixels sorted by (y, x), collinear points dropped, starting at the raster-first
    hull point), the one of least area, compared exactly in integers; on equal areas the first edge.  Its vertices
    p + (a*e + b*n) / |e|^2 (p the edge's first hull point, e the edge, n = (-e_y, e_x), a / b the integer extremes of
    the hull's projections) are one float64 division and one addition each, then rounded to float32 as boxPoints
    returns them, in boxPoints' order;
  * boxPoints' order (cv2 4.x angle in [-90, 0)): with wd the one of +-e, +-n that has x >= 0 and y < 0 and
    hd = (-wd_y, wd_x), the vertices are (min wd, max hd), (min wd, min hd), (max wd, min hd), (max wd, max hd);
  * fallback: (x0, y0), (x0 + w, y0), (x0 + w, y0 + h), (x0, y0 + h) with x0 = cx - w / 2, y0 = cy - h / 2, float64.

cv2's minAreaRect is not the exact minimum: on near-ties its float arithmetic may pick another edge.  `margin` of the
result measures how close the runner-up rectangle (edges neither parallel nor perpendicular to the chosen one) is, so
tests compare with cv2 only where the choice is clear.
"""
from __future__ import annotations

import numpy as np
from scipy import ndimage

AREA_MIN2 = 200                   # contourArea > 100, doubled
FLAG_FALLBACK, FLAG_CONTOUR = 0, 1

# OpenCV's chain-code directions: 0 = east, counterclockwise on screen (y down)
DIRS = ((1, 0), (1, -1), (0, -1), (-1, -1), (-1, 0), (-1, 1), (0, 1), (1, 1))


def trace_outer(fg: np.ndarray, y: int, x: int) -> list:
    """The outer border through (x, y), a component's raster-first pixel, as Suzuki & Abe's border following returns
    it: a list of (x, y) pixel centres, the start first."""
    H, W = fg.shape

    def on(d, px, py):
        qx, qy = px + DIRS[d][0], py + DIRS[d][1]
        return 0 <= qx < W and 0 <= qy < H and bool(fg[qy, qx])

    # (3.1) clockwise from the west neighbour for the first foreground neighbour
    first = next((d for d in (4, 3, 2, 1, 0, 7, 6, 5) if on(d, x, y)), None)
    if first is None:
        return [(x, y)]
    p1 = (x + DIRS[first][0], y + DIRS[first][1])
    prev, cur = p1, (x, y)
    pts = []
    while True:
        pts.append(cur)
        d0 = DIRS.index((prev[0] - cur[0], prev[1] - cur[1]))
        # (3.3) counterclockwise from the neighbour after prev
        d = next(((d0 + k) % 8 for k in range(1, 9) if on((d0 + k) % 8, *cur)))
        nxt = (cur[0] + DIRS[d][0], cur[1] + DIRS[d][1])
        if nxt == (x, y) and cur == p1:                     # (3.5)
            return pts
        prev, cur = cur, nxt


def area2(pts) -> int:
    """Twice the shoelace area of a closed polygon of integer points (cv2.contourArea, doubled)."""
    s = 0
    n = len(pts)
    for i in range(n):
        (x0, y0), (x1, y1) = pts[i], pts[(i + 1) % n]
        s += x0 * y1 - x1 * y0
    return abs(s)


def components(fg: np.ndarray):
    """(labels, roots): the 8-connected labelling of fg and, per label 1.., the raster index of its first pixel."""
    lab, n = ndimage.label(fg, structure=np.ones((3, 3), bool))
    flat = lab.ravel()
    idx = np.nonzero(flat)[0]
    roots = np.full(n + 1, -1, np.int64)
    # first occurrence of each label in raster order
    u, first = np.unique(flat[idx], return_index=True)
    roots[u] = idx[first]
    return lab, roots


def contour_areas(fg: np.ndarray) -> dict:
    """{raster index of the first pixel: doubled outer-contour area} of every component."""
    fg = np.asarray(fg, bool)
    _, roots = components(fg)
    W = fg.shape[1]
    return {int(r): area2(trace_outer(fg, int(r) // W, int(r) % W)) for r in roots[1:]}


def convex_hull(lab: np.ndarray, label: int) -> list:
    """Hull vertices (x, y) of one component from its row-wise leftmost and rightmost pixels: Andrew's monotone chain
    over the points sorted by (y, x), first chain then second, collinear points dropped."""
    pts = []
    for y in range(lab.shape[0]):
        xs = np.nonzero(lab[y] == label)[0]
        if xs.size:
            pts.append((int(xs[0]), y))
            if xs[-1] != xs[0]:
                pts.append((int(xs[-1]), y))
    pts.sort(key=lambda p: (p[1], p[0]))

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])

    lo = []
    for p in pts:
        while len(lo) >= 2 and cross(lo[-2], lo[-1], p) <= 0:
            lo.pop()
        lo.append(p)
    hi = []
    for p in reversed(pts):
        while len(hi) >= 2 and cross(hi[-2], hi[-1], p) <= 0:
            hi.pop()
        hi.append(p)
    return lo[:-1] + hi[:-1]


def _extent(hull, i):
    """Edge i of the hull: (p, e, amin, amax, bmin, bmax) with a = e . (q - p), b = n . (q - p) over the hull."""
    M = len(hull)
    p, q = hull[i], hull[(i + 1) % M]
    ex, ey = q[0] - p[0], q[1] - p[1]
    a = [ex * (h[0] - p[0]) + ey * (h[1] - p[1]) for h in hull]
    b = [-ey * (h[0] - p[0]) + ex * (h[1] - p[1]) for h in hull]
    return p, (ex, ey), min(a), max(a), min(b), max(b)


def min_area_rect(hull):
    """(vertices float64 [4, 2] rounded to float32, chosen edge index, margin): the least-area rectangle over the hull
    edges in boxPoints' order; margin = area of the best rectangle of another orientation / the least area - 1 (inf if
    there is none)."""
    M = len(hull)
    ext = [_extent(hull, i) for i in range(M)]
    q = [(e[3] - e[2]) * (e[5] - e[4]) for e in ext]          # area * |e|^2
    L = [e[1][0] ** 2 + e[1][1] ** 2 for e in ext]
    best = 0
    for i in range(1, M):
        if q[i] * L[best] < q[best] * L[i]:                    # exact: the first of equal areas stays
            best = i
    p, (ex, ey), amin, amax, bmin, bmax = ext[best]
    others = [q[j] / L[j] for j in range(M)
              if ext[j][1][0] * ey - ext[j][1][1] * ex != 0 and ext[j][1][0] * ex + ext[j][1][1] * ey != 0]
    margin = min(others) / (q[best] / L[best]) - 1 if others else float("inf")
    # boxPoints' width direction: the rotation k of e with x >= 0, y < 0
    rots = [(ex, ey), (-ey, ex), (-ex, -ey), (ey, -ex)]
    k = next(k for k, (dx, dy) in enumerate(rots) if dx >= 0 and dy < 0)
    cyc = [(amin, bmax), (amin, bmin), (amax, bmin), (amax, bmax)]
    Lf = np.float64(L[best])
    out = np.zeros((4, 2))
    for j in range(4):
        a, b = cyc[(k + j) % 4]
        nx, ny = a * ex - b * ey, a * ey + b * ex
        out[j] = (np.float32(np.float64(p[0]) + np.float64(nx) / Lf), np.float32(np.float64(p[1]) + np.float64(ny) / Lf))
    return out, best, margin


def fallback_polygon(cxcywh) -> np.ndarray:
    """cxy_wh_2_rect of (target_pos, target_sz) as the reference's 4 corners, float64 [8]."""
    cx, cy, w, h = (np.float64(v) for v in cxcywh)
    x0, y0 = cx - w / 2, cy - h / 2
    return np.array([x0, y0, x0 + w, y0, x0 + w, y0 + h, x0, y0 + h])


def rotated_box(fg, cxcywh):
    """One stream: (polygon float64 [8], flag, doubled area of the chosen contour (or of the largest, on fallback; 0
    without foreground), margin)."""
    fg = np.asarray(fg, bool)
    lab, roots = components(fg)
    W = fg.shape[1]
    best_key, best_label = (-1, -1), 0
    for label in range(1, len(roots)):
        r = int(roots[label])
        key = (area2(trace_outer(fg, r // W, r % W)), r)
        if key > best_key:
            best_key, best_label = key, label
    a2 = max(best_key[0], 0)
    if a2 <= AREA_MIN2:
        return fallback_polygon(cxcywh), FLAG_FALLBACK, a2, float("inf")
    box, _, margin = min_area_rect(convex_hull(lab, best_label))
    return box.reshape(-1), FLAG_CONTOUR, a2, margin


def rotated_boxes(masks, fallback):
    """rotated_box for a list of masks [H_i, W_i] and fallback float64 [N, 4] (cx, cy, w, h): (poly [N, 8], flag [N],
    area2 [N], margin [N])."""
    out = [rotated_box(m, f) for m, f in zip(masks, np.asarray(fallback, np.float64).reshape(-1, 4))]
    return (np.array([o[0] for o in out]).reshape(-1, 8), np.array([o[1] for o in out], np.int32),
            np.array([o[2] for o in out], np.int64), np.array([o[3] for o in out]))


def cv2_rotated_box(fg, cxcywh):
    """tools/test.py:284-303 itself with cv2: (polygon float64 [8], flag, doubled area of the chosen contour, every
    contour's doubled area in cv2's order)."""
    import cv2
    cs = cv2.findContours(np.asarray(fg, np.uint8), cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)[-2]
    areas = [cv2.contourArea(c) for c in cs]
    a2 = [int(round(2 * a)) for a in areas]
    if len(cs) and np.max(areas) > 100:
        c = cs[int(np.argmax(areas))].reshape(-1, 2)
        return cv2.boxPoints(cv2.minAreaRect(c)).astype(np.float64).reshape(-1), FLAG_CONTOUR, max(a2), a2
    return fallback_polygon(cxcywh), FLAG_FALLBACK, max(a2, default=0), a2


def _ellipse(rng, H, W):
    yy, xx = np.mgrid[:H, :W]
    cx, cy = rng.uniform(-0.1, 1.1) * W, rng.uniform(-0.1, 1.1) * H
    a, b = rng.uniform(2, max(3, W / 3)), rng.uniform(2, max(3, H / 3))
    th = rng.uniform(0, np.pi)
    X = (xx - cx) * np.cos(th) + (yy - cy) * np.sin(th)
    Y = -(xx - cx) * np.sin(th) + (yy - cy) * np.cos(th)
    return (X / a) ** 2 + (Y / b) ** 2 < 1


def _rotated_rect(rng, H, W):
    yy, xx = np.mgrid[:H, :W]
    cx, cy = rng.uniform(0, W), rng.uniform(0, H)
    a, b = rng.uniform(1, max(2, W / 3)), rng.uniform(0.5, max(1, H / 3))
    th = rng.choice([0, np.pi / 2, np.pi / 4, rng.uniform(0, np.pi)])
    X = (xx - cx) * np.cos(th) + (yy - cy) * np.sin(th)
    Y = -(xx - cx) * np.sin(th) + (yy - cy) * np.cos(th)
    return (np.abs(X) <= a) & (np.abs(Y) <= b)


def _square(H, W, y, x, n):
    m = np.zeros((H, W), bool)
    m[y:y + n, x:x + n] = True
    return m


def seeded_mask(rng, kind: str, H: int, W: int) -> np.ndarray:
    """One test mask of a named kind, bool [H, W]."""
    m = np.zeros((H, W), bool)
    if kind == "ellipse":
        m = _ellipse(rng, H, W)
    elif kind == "rect":
        m = _rotated_rect(rng, H, W)
    elif kind == "salt":
        m = _ellipse(rng, H, W) | (rng.random((H, W)) < rng.choice([0.002, 0.05, 0.3]))
    elif kind == "lines":                      # one-pixel lines and diagonals (area 0) next to a blob
        for _ in range(rng.integers(1, 6)):
            y0, x0 = rng.integers(0, H), rng.integers(0, W)
            n = int(rng.integers(2, max(3, min(H, W))))
            dy, dx = [(0, 1), (1, 0), (1, 1), (1, -1)][rng.integers(0, 4)]
            for t in range(n):
                y, x = y0 + t * dy, x0 + t * dx
                if 0 <= y < H and 0 <= x < W:
                    m[y, x] = True
        if rng.random() < 0.5:
            m |= _ellipse(rng, H, W)
    elif kind == "corners":                    # blobs touching only at corners: one 8-connected component
        n = int(rng.integers(3, 9))
        y, x = int(rng.integers(0, max(1, H - 2 * n))), int(rng.integers(0, max(1, W - 2 * n)))
        m |= _square(H, W, y, x, n) | _square(H, W, y + n, x + n, n)
        if rng.random() < 0.5:
            m |= _square(H, W, y + 2 * n, x, n)
    elif kind == "holes":                      # a ring with blobs inside its hole
        yy, xx = np.mgrid[:H, :W]
        cx, cy = rng.uniform(0.3, 0.7) * W, rng.uniform(0.3, 0.7) * H
        r0 = rng.uniform(4, max(5, min(H, W) / 2.5))
        r1 = r0 * rng.uniform(0.4, 0.8)
        d = np.hypot(xx - cx, yy - cy)
        m = (d < r0) & (d >= r1)
        m |= d < r1 * rng.uniform(0.1, 0.7)
        m |= (rng.random((H, W)) < 0.01) & (d < r1)
    elif kind == "edges":                      # blobs cut by the frame edges
        for _ in range(int(rng.integers(1, 5))):
            m |= _ellipse(rng, H, W)
        side = rng.integers(0, 4)
        if side == 0:
            m[0, :] = True
        elif side == 1:
            m[-1, :] = True
        elif side == 2:
            m[:, 0] = True
        else:
            m[:, -1] = True
    elif kind == "equal":                      # equal-area blobs: the raster-last first pixel wins
        n = int(rng.integers(6, 20))
        for _ in range(int(rng.integers(2, 5))):
            y, x = int(rng.integers(0, max(1, H - n))), int(rng.integers(0, max(1, W - n)))
            m[y:y + n, x:x + n] = True
    elif kind in ("area100", "area101"):       # an 11x11 square: contour area 100; a bump on a side adds 1
        y, x = int(rng.integers(0, H - 12)), int(rng.integers(0, W - 12))
        m[y:y + 11, x:x + 11] = True
        if kind == "area101":
            m[y + 5, x + 11] = True
    elif kind == "pixel":
        m[rng.integers(0, H), rng.integers(0, W)] = True
    elif kind == "ones":
        m[:] = True
    elif kind != "zeros":
        raise ValueError(kind)
    return m


KINDS = ("ellipse", "rect", "salt", "lines", "corners", "holes", "edges", "equal", "area100", "area101", "pixel",
         "ones", "zeros")


def seeded_masks(seed: int, n: int):
    """n (mask, kind) pairs over every kind, on frames from 1 x W and H x 1 up to 160 x 240."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        if kind in ("area100", "area101"):
            H, W = int(rng.integers(14, 80)), int(rng.integers(14, 80))
        elif i % 29 == 0:
            H, W = (1, int(rng.integers(1, 200))) if rng.random() < 0.5 else (int(rng.integers(1, 200)), 1)
        else:
            H, W = int(rng.integers(2, 160)), int(rng.integers(2, 240))
        out.append((seeded_mask(rng, kind, H, W), kind))
    return out
