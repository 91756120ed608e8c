"""`ops.rotated_box` (C ABI `sm_rotated_box_ragged`) against the numpy restatement of tests/rbox_reference.py (flags,
doubled areas and polygons bit for bit) and against cv2's outputs in tests/golden/rbox_cv2.npz."""
import os

import numpy as np
import pytest
import torch

import rbox_reference as R
from conftest import GOLDEN
from siammask_b200 import ops

pytestmark = pytest.mark.gpu


def _check(masks, fb, label=""):
    poly, flag, area2 = ops.rotated_box([torch.from_numpy(np.ascontiguousarray(m)).cuda() for m in masks], fb)
    want = R.rotated_boxes(masks, fb)
    np.testing.assert_array_equal(flag.cpu().numpy(), want[1], err_msg=label)
    np.testing.assert_array_equal(area2.cpu().numpy(), want[2], err_msg=label)
    np.testing.assert_array_equal(poly.cpu().numpy().view(np.uint64), want[0].view(np.uint64), err_msg=label)
    return poly, flag, area2, want


def test_golden_masks_equal_restatement_and_cv2():
    z = np.load(os.path.join(GOLDEN, "rbox_cv2.npz"))
    off = np.concatenate([[0], np.cumsum(z["shape"].prod(1))])
    masks = [z["masks"][off[i]:off[i + 1]].reshape(h, w).astype(bool) for i, (h, w) in enumerate(z["shape"])]
    poly, flag, area2, want = _check(masks, z["fallback"], "golden")
    np.testing.assert_array_equal(flag.cpu().numpy(), z["flag"])
    np.testing.assert_array_equal(area2.cpu().numpy(), z["area2"])
    clear = (z["flag"] == 0) | (want[3] > 1e-5)
    print(f"golden: {int((z['flag'] == 1).sum())} contour results, {int((~clear).sum())} near-ties")
    np.testing.assert_allclose(poly.cpu().numpy()[clear], z["poly"][clear], rtol=0, atol=1e-3)


def test_seeded_ragged_batches_including_tall_flat_and_hd_frames():
    rng = np.random.default_rng(11)
    masks = [m for m, _ in R.seeded_masks(21, 300)]
    masks.append(R.seeded_mask(rng, "lines", 1, 400))                      # a 1-pixel-high frame
    masks.append(np.ones((1, 300), bool))
    hd = R.seeded_mask(rng, "salt", 1080, 1920)
    masks.append(hd)
    masks.append(R.seeded_mask(rng, "holes", 1080, 1920))
    fb = np.column_stack([rng.uniform(-50, 300, len(masks)), rng.uniform(-50, 300, len(masks)),
                          rng.uniform(5, 90, len(masks)), rng.uniform(5, 90, len(masks))])
    _check(masks, fb, "ragged")
    # one size: a [N,H,W] bool tensor
    same = [R.seeded_mask(rng, k, 120, 160) for k in R.KINDS if k not in ("area100", "area101")]
    t = torch.from_numpy(np.stack(same)).cuda()
    poly, flag, area2 = ops.rotated_box(t, fb[:len(same)])
    want = R.rotated_boxes(same, fb[:len(same)])
    np.testing.assert_array_equal(poly.cpu().numpy().view(np.uint64), want[0].view(np.uint64))


def test_seg_thr_below_minus_one_and_threshold_on_a_pasted_value():
    """seg_thr < -1 makes every pixel foreground, the pasted border value -1 included; a threshold equal to a pasted
    value keeps exactly the pixels above it."""
    rng = np.random.default_rng(5)
    prob = torch.rand(2, 127, 127, device="cuda")
    maps = np.array([[[1.3, 0.1, -30.0], [0.05, 1.1, -10.0]], [[2.0, 0.0, 40.0], [0.0, 2.0, 25.0]]])
    pasted = [ops.warp_affine(prob[i:i + 1], maps[i], (300, 200), -1.0)[0] for i in range(2)]
    for thr in (-1.5, float(pasted[0][100, 100])):
        masks = [p > thr for p in pasted]
        fb = rng.uniform(10, 100, (2, 4))
        poly, flag, area2 = ops.rotated_box(masks, fb)
        want = R.rotated_boxes([m.cpu().numpy() for m in masks], fb)
        np.testing.assert_array_equal(flag.cpu().numpy(), want[1])
        np.testing.assert_array_equal(area2.cpu().numpy(), want[2])
        np.testing.assert_array_equal(poly.cpu().numpy(), want[0])
        if thr < -1:
            assert (area2.cpu().numpy() == 2 * 299 * 199).all()


def test_repeated_calls_are_bit_identical():
    masks = [torch.from_numpy(m).cuda() for m, _ in R.seeded_masks(4, 130)]
    fb = np.tile([50.0, 40.0, 20.0, 30.0], (len(masks), 1))
    first = [t.cpu().numpy() for t in ops.rotated_box(masks, fb)]
    for _ in range(3):
        again = [t.cpu().numpy() for t in ops.rotated_box(masks, fb)]
        for a, b in zip(first, again):
            np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8))


def test_rejects_bad_arguments():
    m = torch.zeros(10, 10, dtype=torch.bool, device="cuda")
    with pytest.raises(ValueError):
        ops.rotated_box([m], np.zeros((2, 4)))
    with pytest.raises(ValueError):
        ops.rotated_box([m.float()], np.zeros((1, 4)))
    with pytest.raises(ValueError):
        ops.rotated_box([torch.zeros(1, 40000, dtype=torch.bool, device="cuda")], np.zeros((1, 4)))
