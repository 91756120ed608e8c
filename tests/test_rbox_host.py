"""The rotated-box restatement (tests/rbox_reference.py) against cv2 itself, the golden file the GPU tests read, the
polygon-entry replay of VotScore restated in numpy, and the C ABI of `sm_rotated_box_ragged` (no device needed)."""
import ctypes
import os
from collections import Counter

import numpy as np
import pytest

import rbox_reference as R
import vot_eval_reference as E
import vot_poly_reference as P
from conftest import GOLDEN
from siammask_b200 import _lib, ops

cv2 = pytest.importorskip("cv2")
NEAR_TIE = 1e-5


def _fallback(m):
    return (m.shape[1] / 2 + 0.3, m.shape[0] / 2 - 0.7, 10.5, 7.25)


def test_restatement_equals_cv2_on_seeded_masks():
    masks = R.seeded_masks(1, 2600)
    assert {k for _, k in masks} == set(R.KINDS)
    near = selected = 0
    worst = 0.0
    for i, (m, kind) in enumerate(masks):
        poly, flag, a2, margin = R.rotated_box(m, _fallback(m))
        cpoly, cflag, ca2, careas = R.cv2_rotated_box(m, _fallback(m))
        assert (flag, a2) == (cflag, ca2), (i, kind, m.shape)
        # every contour RETR_EXTERNAL returns is one of the components' outer borders, with its exact area
        assert not Counter(careas) - Counter(R.contour_areas(m).values()), (i, kind)
        if flag == R.FLAG_FALLBACK:
            np.testing.assert_array_equal(poly, cpoly)
            continue
        selected += 1
        if margin <= NEAR_TIE:
            near += 1
            continue
        d = np.abs(poly - cpoly).max()
        worst = max(worst, d)
        assert d <= 1e-3, (i, kind, m.shape, poly, cpoly, margin)
    print(f"rotated box vs cv2: {selected} contour results, {near} near-ties (runner-up within {NEAR_TIE:g}), "
          f"max vertex difference elsewhere {worst:.3g} px")
    assert selected > 800 and near < 0.01 * selected


def test_threshold_and_tie_cases():
    square = R.seeded_mask(np.random.default_rng(0), "area100", 30, 30)
    assert R.rotated_box(square, (5, 5, 2, 2))[1:3] == (R.FLAG_FALLBACK, 200)
    bump = R.seeded_mask(np.random.default_rng(0), "area101", 30, 30)
    assert R.rotated_box(bump, (5, 5, 2, 2))[1:3] == (R.FLAG_CONTOUR, 202)
    m = np.zeros((40, 40), bool)                      # four equal squares: the raster-last first pixel wins
    for y, x in ((2, 2), (2, 25), (25, 2), (25, 25)):
        m[y:y + 12, x:x + 12] = True
    poly, flag, a2, _ = R.rotated_box(m, (0, 0, 1, 1))
    assert flag == R.FLAG_CONTOUR and a2 == 242
    assert poly.reshape(4, 2).min(0).tolist() == [25.0, 25.0]
    np.testing.assert_array_equal(poly, R.cv2_rotated_box(m, (0, 0, 1, 1))[0])
    np.testing.assert_array_equal(R.rotated_box(np.zeros((3, 4), bool), (1, 2, 3, 4))[0], [-0.5, 0, 2.5, 0, 2.5, 4, -0.5, 4])


def test_golden_file_matches_cv2():
    z = np.load(os.path.join(GOLDEN, "rbox_cv2.npz"))
    off = np.concatenate([[0], np.cumsum(z["shape"].prod(1))])
    for i, (h, w) in enumerate(z["shape"]):
        m = z["masks"][off[i]:off[i + 1]].reshape(h, w)
        poly, flag, a2, _ = R.cv2_rotated_box(m, z["fallback"][i])
        assert (flag, a2) == (z["flag"][i], z["area2"][i])
        np.testing.assert_array_equal(poly, z["poly"][i])


def test_polygon_replay_matches_result_file_round_trip(tmp_path):
    """The polygon replay of sm_vot_trajectory_overlap_poly, rint(float32(v) * 1e4) / 1e4 per value, is what writing
    "%.4f" and reading it back gives, ties at .xxxx5 and negative values included."""
    rng = np.random.default_rng(3)
    vals = np.concatenate([rng.uniform(-50, 700, 2000), np.arange(-20, 20) / 1e4 + 0.00005, [-0.00004, 12.34565]])
    for v in vals:
        want = E.result_value(v)
        got = np.rint(np.float64(np.float32(v)) * 1e4) / 1e4
        assert got == want or (got == 0 and want == 0), v
    from siammask_b200 import vot
    poly = [np.array([-3.12345, 2.5, 40.00005, 1.0, 41.0, 30.25, -2.0, 29.0])]
    vot.write_result(tmp_path / "r.txt", [1] + poly)
    back = [[float(v) for v in ln.split(",")] for ln in (tmp_path / "r.txt").read_text().splitlines()[1:]]
    np.testing.assert_array_equal(back[0], E.read_back(poly)[0])
    gt = np.array([[0, 0, 0, 0, 0, 0, 0, 0], [0, 0, 30, 0, 30, 20, 0, 20]], np.float64)
    ov = P.trajectory_overlaps([[1.0]] + back, gt, 64, 48)
    assert np.isnan(ov[0]) and 0 < ov[1] < 1


def test_c_symbols_and_argument_checks():
    lib = _lib.load()
    for name in ("sm_rotated_box_ragged", "sm_rotated_box_workspace_size", "sm_tracker_update_hp_ex",
                 "sm_vot_trajectory_overlap_poly"):
        assert hasattr(lib, name)
    assert lib.sm_rotated_box_workspace_size(100, 0, 10) == 0
    n = ctypes.c_void_p(1)
    bad = [(-1, 10, 10), (1, 0, 10), (1, 10, 40000), (70000, 10, 10)]
    for N, mh, mw in bad:
        rc = lib.sm_rotated_box_ragged(n, n, N, mh, mw, 100, n, n, 1 << 20, n, n, n, None)
        assert rc != 0
        assert b"bad argument" in lib.sm_last_error()
    assert lib.sm_rotated_box_ragged(None, None, 0, 1, 1, 0, None, None, 0, None, None, None, None) == 0
    with pytest.raises(ValueError):
        ops.rotated_box(np.zeros((2, 3, 3), bool), np.zeros((2, 4)))
    with pytest.raises(ValueError):
        ops.rotated_box([], np.zeros((0, 4)))
