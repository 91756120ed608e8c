"""Generates tests/golden/rbox_cv2.npz: seeded masks of every kind in tests/rbox_reference.py with cv2's own rotated
box of tools/test.py:284-303 (findContours, contourArea, boxPoints(minAreaRect)).  TEST INFRASTRUCTURE ONLY; needs
cv2:

    python tools/make_rbox_golden.py

Contents: masks (uint8, the masks' pixels back to back), shape [N, 2] (h, w), fallback [N, 4] (cx, cy, w, h), and cv2's
poly [N, 8] (float64), flag [N] (1 contour, 0 fallback) and area2 [N] (twice the largest contour area).
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rbox_reference as R  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "rbox_cv2.npz")


def main():
    masks = R.seeded_masks(7, 390)
    rng = np.random.default_rng(7)
    fb = np.column_stack([rng.uniform(-20, 200, len(masks)), rng.uniform(-20, 150, len(masks)),
                          rng.uniform(10, 80, len(masks)), rng.uniform(10, 80, len(masks))])
    out = [R.cv2_rotated_box(m, f) for (m, _), f in zip(masks, fb)]
    np.savez_compressed(OUT, masks=np.concatenate([m.reshape(-1) for m, _ in masks]).astype(np.uint8),
                        shape=np.array([m.shape for m, _ in masks], np.int64), fallback=fb,
                        poly=np.array([o[0] for o in out]), flag=np.array([o[1] for o in out], np.int32),
                        area2=np.array([o[2] for o in out], np.int64))
    print("wrote", OUT, len(masks), "masks")


if __name__ == "__main__":
    main()
