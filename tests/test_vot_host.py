"""Host side of the VOT protocol (siammask_b200/vot.py): the overlap and bbox restatements against the golden file the
reference's own code wrote (tools/make_vot_golden.py), the result-file format, the skip / re-init schedule of the
track_vot restatement, and the argument checks.  The live reference library (oracle/_ref, built by build()) is used
where it exists."""
import ctypes as C
import ctypes.util
import os

import numpy as np
import pytest
import torch

import vot_reference
from conftest import GOLDEN
from oracle import build_ref
from siammask_b200 import ops, vot


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "vot_overlap.npz")))


@pytest.fixture(scope="module")
def region_lib():
    lib = build_ref.load()
    if lib is None:
        pytest.skip("oracle/_ref/libvot_region.so was not built (no reference tree)")
    return lib


def _bits(v):
    return np.asarray(v, np.float32).view(np.uint32)


def test_golden_covers_the_cases(golden):
    ov = golden["overlap_bits"].view(np.float32)
    W, H = golden["size"][:, 0], golden["size"][:, 1]
    assert np.isnan(ov).any() and (ov == 0).any() and (ov == 1).any() and ((ov > 0) & (ov < 1)).sum() > 100
    assert (W.min(), H.min()) == (1, 1) and (W.max(), H.max()) == (1920, 1080)
    assert (golden["poly_a"] == np.round(golden["poly_a"]) + 0.5).any()              # exact .5 coordinates
    assert (golden["poly_a"][:, 0::2] > W[:, None]).any()                              # past column W


def test_polygon_overlap_restatement_equals_golden(golden):
    for i in range(len(golden["size"])):
        got = vot_reference.polygon_overlap(golden["poly_a"][i], golden["poly_b"][i], *golden["size"][i])
        assert _bits(got) == golden["overlap_bits"][i], i


def test_get_axis_aligned_bbox_equals_golden(golden):
    for fn in (vot.get_axis_aligned_bbox, vot_reference.get_axis_aligned_bbox):
        got = np.asarray([fn(r) for r in golden["bbox_in"]], np.float64)
        np.testing.assert_array_equal(got.view(np.uint64), golden["bbox_out"].view(np.uint64))


def test_live_library_equals_golden_and_restatement(golden, region_lib):
    for i in range(len(golden["size"])):
        assert _bits(region_lib.overlap(golden["poly_a"][i], golden["poly_b"][i], *golden["size"][i])) == \
            golden["overlap_bits"][i], i
    rng = np.random.RandomState(7)
    for i in range(150):
        W, H = int(rng.randint(1, 400)), int(rng.randint(1, 300))
        a, b = rng.uniform(-30, W + 30, 8), rng.uniform(-30, W + 30, 8)
        a[1::2], b[1::2] = rng.uniform(-30, H + 30, 4), rng.uniform(-30, H + 30, 4)
        if i % 3 == 0:                                                   # boxes on the half-pixel grid
            a, b = np.round(a * 2) / 2, np.round(b * 2) / 2
        assert _bits(region_lib.overlap(a, b, W, H)) == _bits(vot_reference.polygon_overlap(a, b, W, H)), i


def _c_float2str(v) -> str:
    """pyvotkit's vot_float2str("%.4f", v): the value as a C float, through libc's snprintf."""
    libc = C.CDLL(ctypes.util.find_library("c"))
    buf = C.create_string_buffer(100)
    libc.snprintf(buf, 100, b"%.4f", C.c_double(float(np.float32(v))))
    return buf.value.decode()


def test_write_result_equals_reference_writer(tmp_path):
    rng = np.random.RandomState(3)
    locs = [rng.uniform(-50, 2000, 4) for _ in range(40)]
    locs += [np.array([0.03125, 1 / 3, 2.00005, -0.0]), np.array([1e-5, 123456.78125, 0.5, 7.99995])]
    regions = [1] + locs[:10] + [2, 0, 0, 0, 0, 1] + locs[10:]
    path = tmp_path / "seq_001.txt"
    vot.write_result(path, regions)
    assert path.read_bytes() == vot_reference.result_lines(regions, _c_float2str).encode()


_frame = [0]          # frame the fake tracker last saw


def test_track_vot_restatement_schedule(monkeypatch):
    """Codes of the restated loop: init 1, a failure 2, four skipped frames 0 and a re-init 1 on the fifth from that
    frame's ground truth; a NaN overlap is not a failure."""
    inits = []

    def fake_init(im, pos, sz, *a, **k):
        inits.append(int(im[0, 0, 0]))
        return {"target_pos": np.asarray(pos, float).copy(), "target_sz": np.asarray(sz, float).copy()}

    def fake_track(state, im, *a, **k):
        _frame[0] = int(im[0, 0, 0])
        return state
    monkeypatch.setattr(vot_reference.ref_loop, "siamese_init", fake_init)
    monkeypatch.setattr(vot_reference.ref_loop, "siamese_track", fake_track)
    T = 16
    frames = [np.full((20, 30, 3), f, np.uint8) for f in range(T)]
    gt = np.asarray([[f, 1, f + 5, 1, f + 5, 6, f, 6] for f in range(T)], np.float64)
    verdict = {2: 0.0, 3: float("nan"), 8: 0.0, 14: 0.0}
    regions, lost = vot_reference.track_vot(None, frames, gt, {}, overlap=lambda a, b, W, H: verdict.get(_frame[0], 0.5))
    codes = [r if isinstance(r, int) else 3 for r in regions]
    # frame 3 is skipped (the NaN verdict is never asked), frame 7 re-initialises, frame 8 tracks and fails again;
    # the failure at frame 14 would re-initialise at 19, past the end
    assert codes == [1, 3, 2, 0, 0, 0, 0, 1, 2, 0, 0, 0, 0, 1, 2, 0]
    assert lost == 3 and inits == [0, 7, 13]
    verdict = {3: float("nan")}
    regions, lost = vot_reference.track_vot(None, frames, gt, {}, overlap=lambda a, b, W, H: verdict.get(_frame[0], 0.5))
    assert lost == 0 and all(not isinstance(r, int) for r in regions[1:])           # NaN is truthy


def test_gt_checks():
    ok = np.tile(np.array([[1.0, 1, 9, 1, 9, 9, 1, 9]]), (3, 1))
    assert vot.check_gt([ok, ok[:1]])[1].shape == (1, 8)
    for bad in ([ok[:, :4]], [ok[0]], [np.zeros((0, 8))], [np.where(np.eye(3, 8) > 0, np.nan, ok)],
                [np.where(np.eye(3, 8) > 0, np.inf, ok)], [ok * 2 ** 21]):
        with pytest.raises(ValueError):
            vot.check_gt(bad)
    with pytest.raises(ValueError):
        vot.get_axis_aligned_bbox([1.0, 2, 3, 4])


def test_vot_overlap_argument_checks():
    a = torch.zeros(2, 8)
    for args in ((a, a), (a.double(), a), (torch.zeros(2, 4), torch.zeros(2, 4))):
        with pytest.raises(ValueError):
            ops.vot_overlap(*args, (10, 10))
