"""VOT scoring on the device: `sm_vot_trajectory_overlap` and `VotScore` against the golden file made by the
reference's pysot benchmarks (tools/make_vot_eval_golden.py), split invariance and run-to-run bits, and `VotRunner` runs
scored end to end against the numpy restatement of tests/vot_eval_reference.py over result files."""
import os

import numpy as np
import pytest
import torch

import siammask_b200 as smb
import vot_eval_reference as R
from conftest import GOLDEN
from oracle.calibrate import calibrated_state_dict
from oracle.synthetic_video import make_frames
from siammask_b200 import ops, vot
from siammask_b200.tune import grid

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "vot_eval.npz")))


def _inputs(z, ks=None, gs=None):
    """(regions[g][k], gt list, sizes (H, W)) of the golden's trackers ks and sequences gs."""
    K, G = z["rec"].shape[:2]
    ks = range(K) if ks is None else ks
    gs = range(G) if gs is None else gs
    regions = [[[int(r[0]) if r[0] != vot.CODE_LOCATION else r[1:] for r in z["rec"][k, g, :z["length"][g]]]
                for k in ks] for g in gs]
    gt = [z["gt"][g, :z["length"][g]] for g in gs]
    sizes = [(int(z["size"][g][1]), int(z["size"][g][0])) for g in gs]
    return regions, gt, sizes


def _planes(z):
    K, G, Tmax, _ = z["rec"].shape
    rec = torch.from_numpy(np.ascontiguousarray(z["rec"].transpose(2, 1, 0, 3).reshape(Tmax, G * K, 5))).cuda()
    gt = torch.from_numpy(z["gt"].astype(np.float32)).cuda()
    seq = np.repeat(np.arange(G), K)
    i32 = lambda a: torch.as_tensor(np.asarray(a, np.int32)).cuda()       # noqa: E731
    acc, eao = ops._vot_trajectory_overlap(rec, Tmax, G * K, gt, i32(seq), i32(z["size"][seq]), i32(z["length"][seq]))
    bits = lambda t: t.cpu().numpy().view(np.uint32).reshape(Tmax, G, K).transpose(2, 1, 0)    # noqa: E731
    return bits(acc), bits(eao)


def test_overlap_planes_equal_golden(golden):
    acc, eao = _planes(golden)
    for g, T in enumerate(golden["length"]):
        np.testing.assert_array_equal(acc[:, g, :T], golden["acc_overlap_bits"][:, g, :T], err_msg=f"acc seq {g}")
        np.testing.assert_array_equal(eao[:, g, :T], golden["eao_overlap_bits"][:, g, :T], err_msg=f"eao seq {g}")
        assert (acc[:, g, T:] == 0x7FC00000).all() and (eao[:, g, T:] == 0x7FC00000).all()


def test_acc_plane_equals_vot_overlap_on_rounded_polygons(golden):
    acc, _ = _planes(golden)
    K, G = golden["rec"].shape[:2]
    for g in range(G):
        T = int(golden["length"][g])
        W, H = golden["size"][g]
        for k in range(K):
            rec = golden["rec"][k, g, :T]
            init = np.nonzero(rec[:, 0] == vot.CODE_INIT)[0]
            sel = [f for f in range(T) if rec[f, 0] == vot.CODE_LOCATION and not ((f - init >= 0) & (f - init < 10)).any()]
            if not sel:
                continue
            x, y, w, h = (np.array([R.result_value(v) for v in rec[sel, c]]) for c in range(1, 5))
            pred = np.stack([x, y, x + w, y, x + w, y + h, x, y + h], 1).astype(np.float32)
            got = ops.vot_overlap(torch.from_numpy(pred).cuda(),
                                  torch.from_numpy(golden["gt"][g, sel].astype(np.float32)).cuda(), (H, W))
            np.testing.assert_array_equal(got.cpu().numpy().view(np.uint32), acc[k, g, sel])


def _check_scores(r, z, sequences):
    np.testing.assert_array_equal(r["lost_number"], z["lost_number"])
    np.testing.assert_allclose(r["accuracy"], z["accuracy"], rtol=1e-12)
    np.testing.assert_allclose(r["robustness"], z["robustness"], rtol=1e-12)
    c, want = r["expected_overlaps"], z["curve"]
    assert c.shape == want.shape and c.dtype == np.float32
    assert (np.isnan(c) == np.isnan(want)).all()
    ok = ~np.isnan(want)
    assert np.abs(c.view(np.int32).astype(np.int64) - want.view(np.int32))[ok].max() <= 1
    np.testing.assert_allclose(r["eao"], z["eao_vot2018"], rtol=0, atol=1e-7)
    assert (r["sequences"] == sequences).all()


def test_scores_match_golden_whole_per_sequence_and_per_chunk(golden):
    K, G = golden["rec"].shape[:2]
    whole = smb.VotScore(K).add_regions(*_inputs(golden)).result()
    _check_scores(whole, golden, G)
    r19 = smb.VotScore(K, dataset="VOT2019").add_regions(*_inputs(golden)).result()
    np.testing.assert_allclose(r19["eao"], golden["eao_vot2019"], rtol=0, atol=1e-7)
    for order in (range(G), reversed(range(G))):           # growing the curve, and starting with the longest
        s = smb.VotScore(K)
        for g in order:
            s.add_regions(*_inputs(golden, gs=[g]))
        _check_scores(s.result(), golden, G)
    s = smb.VotScore(K)
    s.add_regions(*_inputs(golden, ks=[2, 0], gs=[0, 1, 2]), combo_index=[2, 0])
    s.add_regions(*_inputs(golden, ks=[1], gs=[0, 1, 2]), combo_index=[1])
    s.add_regions(*_inputs(golden, gs=[3, 4, 5]))
    _check_scores(s.result(), golden, G)


def test_repeated_runs_are_bit_identical(golden):
    K = golden["rec"].shape[0]
    runs = []
    for _ in range(2):
        s = smb.VotScore(K)
        s.add_regions(*_inputs(golden, gs=[1, 4]))
        s.add_regions(*_inputs(golden, gs=[0, 2, 3, 5]))
        runs.append((s.result(), torch.cat([s._num, s._den, s._stats, s._tail], 1).cpu().numpy()))
    np.testing.assert_array_equal(runs[0][1].view(np.uint64), runs[1][1].view(np.uint64))
    for key in ("accuracy", "robustness", "eao", "expected_overlaps"):
        np.testing.assert_array_equal(np.asarray(runs[0][0][key]).view(np.uint8), np.asarray(runs[1][0][key]).view(np.uint8))


# --------------------------------------------------------------------------------- VotRunner end to end
FAR = np.array([0.0, 0.0, 10.0, 0.0, 10.0, 10.0, 0.0, 10.0])        # a gt quad in the far corner: overlap 0


def _sequence(seed, T, fail_at=()):
    frames, boxes = make_frames(n=T, seed=seed)
    gt = np.asarray([[x, y, x + w, y, x + w, y + h, x, y + h] for (x, y, w, h) in boxes], np.float64)
    gt[0] += np.array([0.5, 0.25, -0.5, 0.25, -0.5, -0.75, 0.5, -0.75])
    for f in fail_at:
        gt[f] = FAR
    return frames, gt


def test_vot_runner_scored_like_result_files(tmp_path):
    sd = calibrated_state_dict(0)
    combos = grid([0.04, 0.2], [0.4, 0.1], [1.0])                     # K = 4
    seqs = [_sequence(0, 24, fail_at=(1, 9)), _sequence(1, 14, fail_at=(7,)), _sequence(2, 12, fail_at=(7,)),
            _sequence(3, 8)]
    net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=16, num_slots=16).load_state_dict(sd).eval().to("cuda")
    runner = smb.VotRunner(net, smb.tracker.TrackerParams(instance_size=255, out_size=127), combos)
    G, K = len(seqs), len(combos)
    Tmax = max(len(s[0]) for s in seqs)
    frame = lambda f: np.stack([s[0][min(f, len(s[0]) - 1)] for s in seqs])     # noqa: E731
    runner.open(frame(0), [s[1] for s in seqs])
    score = smb.VotScore(K)
    with pytest.raises(ValueError, match="ended"):
        score.add(runner)
    for f in range(1, Tmax):
        runner.frame(frame(f))
    regions, lost = runner.result()
    r = score.add(runner).result()
    assert (r["lost_number"] == lost.sum(0)).all() and lost.sum() >= 4
    for k in range(K):
        accs, eaos, fails = [], [], []
        for g, (frames, gt) in enumerate(seqs):
            path = tmp_path / f"s{g}_{k}.txt"
            vot.write_result(path, regions[g][k])
            traj = [list(map(float, line.split(","))) for line in path.read_text().splitlines()]
            H, W = frames[0].shape[:2]
            accs.append(R.trajectory_overlaps(traj, gt, W, H, burnin=R.BURNIN))
            eaos.append(R.trajectory_overlaps(traj, gt, W - 1, H - 1))
            fails.append(R.failures(traj))
        acc, rob, ln = R.accuracy_robustness(accs, [len(f) for f in fails])
        assert r["lost_number"][k] == ln
        np.testing.assert_allclose([r["accuracy"][k], r["robustness"][k]], [acc, rob], rtol=1e-12)
        curve = R.expected_overlaps(eaos, fails, Tmax)
        got = r["expected_overlaps"][k]
        assert (np.isnan(got) == np.isnan(curve)).all()
        ok = ~np.isnan(curve)
        assert np.abs(got.view(np.int32).astype(np.int64) - curve.view(np.int32))[ok].max() <= 1
        np.testing.assert_allclose(r["eao"][k], R.eao(curve, 100, 356), rtol=0, atol=1e-7, equal_nan=True)
