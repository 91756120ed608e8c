"""Polygon entries of VOT results without a GPU: the numpy replay of tests/vot_poly_reference.py (with the read-back and
aggregates of tests/vot_eval_reference.py) against tests/golden/vot_eval_poly.npz, which the reference's own pysot
benchmarks computed from 8-value result files (tools/make_vot_eval_golden.py --poly)."""
import os

import numpy as np
import pytest

import vot_eval_reference as E
import vot_poly_reference as P
from conftest import GOLDEN
from siammask_b200 import vot


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "vot_eval_poly.npz")))


def regions(rec, T):
    """One trajectory of the golden in VotRunner.result()'s form: codes as ints, locations as 8 values."""
    return [int(r[0]) if r[0] != vot.CODE_LOCATION else r[1:] for r in rec[:T]]


def test_polygon_replay_matches_pysot(golden):
    K, G, Tmax, _ = golden["rec"].shape
    for k in range(K):
        accs, eaos, fails = [], [], []
        for g in range(G):
            T = int(golden["length"][g])
            W, H = golden["size"][g]
            traj = E.read_back(regions(golden["rec"][k, g], T))
            a = P.trajectory_overlaps(traj, golden["gt"][g, :T], W, H, burnin=E.BURNIN)
            e = P.trajectory_overlaps(traj, golden["gt"][g, :T], W - 1, H - 1)
            np.testing.assert_array_equal(a.view(np.uint32), golden["acc_overlap_bits"][k, g, :T], err_msg=f"{k} {g}")
            np.testing.assert_array_equal(e.view(np.uint32), golden["eao_overlap_bits"][k, g, :T], err_msg=f"{k} {g}")
            accs.append(a)
            eaos.append(e)
            fails.append(E.failures(traj))
        acc, rob, lost = E.accuracy_robustness(accs, [len(f) for f in fails])
        assert lost == golden["lost_number"][k]
        np.testing.assert_allclose([acc, rob], [golden["accuracy"][k], golden["robustness"][k]], rtol=1e-12)
        curve = E.expected_overlaps(eaos, fails, Tmax)
        assert (np.isnan(curve) == np.isnan(golden["curve"][k])).all()
        ulps = np.abs(curve.view(np.int32).astype(np.int64) - golden["curve"][k].view(np.int32))
        assert ulps[~np.isnan(curve)].max() <= 1
        assert abs(E.eao(curve, 100, 356) - golden["eao_vot2018"][k]) <= 1e-7
        assert abs(E.eao(curve, 46, 291) - golden["eao_vot2019"][k]) <= 1e-7


def test_polygon_golden_covers_the_cases(golden):
    rec, T = golden["rec"], golden["length"]
    loc = rec[..., 0] == vot.CODE_LOCATION
    vals = rec[..., 1:][loc]
    assert vals.shape[1] == 8
    scaled = np.float64(vals.astype(np.float32)) * 1e4
    assert (scaled - np.floor(scaled) == 0.5).any()                 # exact .xxxx5 ties
    assert ((vals < 0) & (vals > -5e-5)).any()                       # printed as -0.0000
    assert (vals < -1).any()                                         # negative coordinates
    W, H = golden["size"][:, 0], golden["size"][:, 1]
    g_of = np.nonzero(loc)[1]
    off = (vals[:, 0::2].max(1) > W[g_of]) | (vals[:, 1::2].max(1) > H[g_of]) | (vals.min(1) < 0)
    inside = (vals[:, 0::2].min(1) < W[g_of]) & (vals[:, 1::2].min(1) < H[g_of])
    assert (off & inside).any()                                      # partly off the frame
    nan = golden["eao_overlap_bits"] == 0xFFC00000                   # the rasteriser's empty union: NaN overlaps
    assert nan.any() and (golden["acc_overlap_bits"] == 0xFFC00000).any()
    assert (rec[..., 0] == vot.CODE_LOST).any() and (T > 356).any()
