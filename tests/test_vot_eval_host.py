"""VOT scoring without a GPU: the numpy restatement in tests/vot_eval_reference.py against the golden file made by the
reference's pysot benchmarks (tools/make_vot_eval_golden.py), the device's "%.4f" round-trip formula against libc, and
`VotScore`'s argument checks."""
import ctypes
import ctypes.util
import os

import numpy as np
import pytest

import vot_eval_reference as R
from conftest import GOLDEN
from siammask_b200 import vot


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "vot_eval.npz")))


def _regions(rec, T):
    return [int(r[0]) if r[0] != vot.CODE_LOCATION else r[1:] for r in rec[:T]]


def test_restatement_matches_golden(golden):
    K, G, Tmax, _ = golden["rec"].shape
    for k in range(K):
        accs, eaos, fails = [], [], []
        for g in range(G):
            T = int(golden["length"][g])
            W, H = golden["size"][g]
            traj = R.read_back(_regions(golden["rec"][k, g], T))
            a = R.trajectory_overlaps(traj, golden["gt"][g, :T], W, H, burnin=R.BURNIN)
            e = R.trajectory_overlaps(traj, golden["gt"][g, :T], W - 1, H - 1)
            np.testing.assert_array_equal(a.view(np.uint32), golden["acc_overlap_bits"][k, g, :T], err_msg=f"{k} {g}")
            np.testing.assert_array_equal(e.view(np.uint32), golden["eao_overlap_bits"][k, g, :T], err_msg=f"{k} {g}")
            accs.append(a)
            eaos.append(e)
            fails.append(R.failures(traj))
        acc, rob, lost = R.accuracy_robustness(accs, [len(f) for f in fails])
        assert lost == golden["lost_number"][k]
        np.testing.assert_allclose([acc, rob], [golden["accuracy"][k], golden["robustness"][k]], rtol=1e-12)
        curve = R.expected_overlaps(eaos, fails, Tmax)
        ulps = np.abs(curve.view(np.int32).astype(np.int64) - golden["curve"][k].view(np.int32))
        assert (np.isnan(curve) == np.isnan(golden["curve"][k])).all()
        assert ulps[~np.isnan(curve)].max() <= 1
        assert abs(R.eao(curve, 100, 356) - golden["eao_vot2018"][k]) <= 1e-7
        assert abs(R.eao(curve, 46, 291) - golden["eao_vot2019"][k]) <= 1e-7


def test_golden_covers_the_cases(golden):
    T, rec = golden["length"], golden["rec"]
    codes = rec[..., 0]
    assert (T < 100).any() and ((T >= 100) & (T <= 356)).any() and (T > 356).any()
    assert (golden["size"] == 2).all(1).any()
    lost = [(k, g, f) for k, g, f in zip(*np.nonzero(codes == vot.CODE_LOST))]
    assert any(f == 1 for _, _, f in lost)
    assert any(f == T[g] - 5 for _, g, f in lost)                   # empty last fragment
    assert any(f > T[g] - 5 for _, g, f in lost)                    # dropped point
    eao_nan = golden["eao_overlap_bits"] == 0xFFC00000              # the rasteriser's empty union
    assert eao_nan.any()
    assert any((codes[k, g] == vot.CODE_LOST).any() for k, g in zip(*np.nonzero(eao_nan.any(2))))
    assert any(not (codes[k, g] == vot.CODE_LOST).any() for k, g in zip(*np.nonzero(eao_nan.any(2))))
    assert golden["curve"].shape[0] == 3 and np.isfinite(golden["eao_vot2019"]).all()


def _libc_round_trip(v):
    libc = ctypes.CDLL(ctypes.util.find_library("c"))
    libc.snprintf.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_double]
    libc.strtod.restype = ctypes.c_double
    libc.strtod.argtypes = [ctypes.c_char_p, ctypes.c_void_p]
    buf = ctypes.create_string_buffer(128)
    libc.snprintf(buf, 128, b"%.4f", float(np.float32(v)))
    return libc.strtod(buf.value, None)


def _device_formula(v):
    """vot_result_value of sm_vot_trajectory_overlap: rint((double)(float)v * 1e4) / 1e4."""
    return float(np.rint(np.float64(np.float32(v)) * 1e4) / 1e4)


def test_round_trip_formula_matches_libc():
    rng = np.random.RandomState(3)
    vals = [0.03125, 0.09375, 0.15625, 1.46875, -0.03125, -1.46875, 12345.65625, -3e-5, -4.99e-5, 5e-5, 0.0, -0.0,
            0.00005, 0.99995, 1048575.96875, -1048575.03125, 2.5e-5, 123.45675]
    vals += list(rng.uniform(-2000, 2000, 2000)) + list(np.floor(rng.uniform(-500, 500, 500)) +
                                                       rng.randint(0, 16, 500) * 2 / 32 + 1 / 32)
    for v in vals:
        want, got = _libc_round_trip(v), _device_formula(v)
        assert np.float64(want).view(np.uint64) == np.float64(got).view(np.uint64), v
        assert np.float64(R.result_value(v)).view(np.uint64) == np.float64(got).view(np.uint64), v


def test_vot_score_rejects_bad_arguments():
    with pytest.raises(ValueError, match="unknown dataset"):
        vot.VotScore(4, dataset="OTB100", device="cpu")
    with pytest.raises(ValueError, match="low <= high"):
        vot.VotScore(4, low=300, high=100, device="cpu")
    with pytest.raises(ValueError, match="low <= high"):
        vot.VotScore(4, dataset=None, low=100, device="cpu")
    with pytest.raises(ValueError, match="num_combos"):
        vot.VotScore(0, device="cpu")
    s = vot.VotScore(4, dataset="OTB100", low=10, high=20, device="cpu")          # explicit bounds: any name
    assert (s.low, s.high) == (10, 20)
    s = vot.VotScore(4, dataset="VOT2019", device="cpu")
    assert (s.low, s.high) == (46, 291)
    gt = [np.tile([0, 0, 4, 0, 4, 4, 0, 4.0], (3, 1))]
    regions = [[[1, [0.0, 0.0, 2.0, 2.0], [0.0, 0.0, 2.0, 2.0]]] * 2]
    with pytest.raises(ValueError, match=r"in \[0, 4\)"):
        s.add_regions(regions, gt, [(10, 10)], combo_index=[0, 4])
    with pytest.raises(ValueError, match="distinct"):
        s.add_regions(regions, gt, [(10, 10)], combo_index=[1, 1])
    with pytest.raises(ValueError, match="2 integers"):
        s.add_regions(regions, gt, [(10, 10)], combo_index=[1, 2, 3])
    with pytest.raises(ValueError, match="2 x 2"):
        s.add_regions(regions, gt, [(1, 10)], combo_index=[1, 2])
    with pytest.raises(ValueError, match="3 frames"):
        s.add_regions([[[1, 0], [1, 0]]], gt, [(10, 10)])
    with pytest.raises(ValueError, match="0, 1 or 2"):
        s.add_regions([[[1, 0, 5], [1, 0, 0]]], gt, [(10, 10)])
    assert s._rows(None, 3).tolist() == [0, 1, 2]
    assert s._rows(np.array([3, 0]), 2).tolist() == [3, 0]
    with pytest.raises(RuntimeError, match="CUDA"):                             # checks pass; no CPU path
        s.add_regions(regions, gt, [(10, 10)], combo_index=[3, 0])
