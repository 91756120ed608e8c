"""The VOT protocol on the device: `sm_vot_overlap` against the reference's compute_polygon_overlap (golden file and,
where it was built, the live library), `BatchTracker.reinit` against a fresh start, and `VotRunner` against per-stream
runs of the track_vot restatement in tests/vot_reference.py."""
import os

import numpy as np
import pytest
import torch

import siammask_b200 as smb
import vot_reference
from conftest import GOLDEN
from oracle import build_ref
from oracle.calibrate import calibrated_state_dict
from oracle.synthetic_video import make_frames
from siammask_b200 import ops, vot
from siammask_b200.tracker import BatchTracker, TrackerParams
from siammask_b200.tune import grid

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "penalty_k": 0.04, "window_influence": 0.4, "lr": 1.0}


def _params():
    return TrackerParams(instance_size=255, out_size=127, penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "vot_overlap.npz")))


def _net(sd, max_batch, num_slots=None, mask=True):
    if not mask:
        sd = {k: v for k, v in sd.items() if not k.startswith(("mask_model", "refine_model"))}
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch, num_slots=num_slots or max_batch,
                      mask=mask).load_state_dict(sd).eval().to("cuda")


def _bits(t):
    return np.asarray(t.cpu().numpy() if torch.is_tensor(t) else t, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------- 1. sm_vot_overlap
def _device_overlap(a, b, W, H):
    return ops.vot_overlap(torch.from_numpy(np.ascontiguousarray(a)).cuda(),
                           torch.from_numpy(np.ascontiguousarray(b)).cuda(), (H, W))


def test_vot_overlap_equals_golden(golden):
    sizes = {tuple(s) for s in golden["size"]}
    for W, H in sorted(sizes):
        sel = np.nonzero((golden["size"][:, 0] == W) & (golden["size"][:, 1] == H))[0]
        got = _device_overlap(golden["poly_a"][sel], golden["poly_b"][sel], W, H)
        np.testing.assert_array_equal(_bits(got), golden["overlap_bits"][sel], err_msg=f"{W}x{H}")
        for n in (1, 3):                                                 # B = 1 and 3
            got = _device_overlap(golden["poly_a"][sel[:n]], golden["poly_b"][sel[:n]], W, H)
            np.testing.assert_array_equal(_bits(got), golden["overlap_bits"][sel[:n]])
    assert np.isnan(golden["overlap_bits"].view(np.float32)).any()


def _random_pairs(rng, B, W, H):
    a = np.empty((B, 8), np.float32)
    b = np.empty((B, 8), np.float32)
    for i in range(B):
        if i % 2:                                                        # boxes near each other, half-pixel grid
            x, y, w, h = rng.uniform(-20, W), rng.uniform(-20, H), rng.uniform(0, W / 3), rng.uniform(0, H / 3)
            a[i] = np.round(np.array([x, y, x + w, y, x + w, y + h, x, y + h]) * 2) / 2
            dx, dy = rng.uniform(-w / 2, w / 2), rng.uniform(-h / 2, h / 2)
            b[i] = [x + dx, y + dy, x + dx + w, y + dy, x + dx + w, y + dy + h, x + dx, y + dy + h]
        else:
            a[i, 0::2], a[i, 1::2] = rng.uniform(-50, W + 50, 4), rng.uniform(-50, H + 50, 4)
            b[i, 0::2], b[i, 1::2] = rng.uniform(-50, W + 50, 4), rng.uniform(-50, H + 50, 4)
    return a, b


def test_vot_overlap_b257_against_restatement_and_library():
    rng = np.random.RandomState(11)
    W, H = 1280, 720
    a, b = _random_pairs(rng, 257, W, H)
    got = _device_overlap(a, b, W, H)
    again = _device_overlap(a, b, W, H)
    np.testing.assert_array_equal(_bits(got), _bits(again))              # deterministic
    want = np.asarray([vot_reference.polygon_overlap(a[i], b[i], W, H) for i in range(257)], np.float32)
    np.testing.assert_array_equal(_bits(got), _bits(want))
    lib = build_ref.load()
    if lib is None:
        pytest.skip("oracle/_ref/libvot_region.so was not built (no reference tree)")
    live = np.asarray([lib.overlap(a[i], b[i], W, H) for i in range(257)], np.float32)
    np.testing.assert_array_equal(_bits(got), _bits(live))


def test_vot_overlap_golden_against_live_library(golden):
    lib = build_ref.load()
    if lib is None:
        pytest.skip("oracle/_ref/libvot_region.so was not built (no reference tree)")
    for i in range(len(golden["size"])):
        W, H = golden["size"][i]
        assert _bits(lib.overlap(golden["poly_a"][i], golden["poly_b"][i], W, H)) == golden["overlap_bits"][i]


def test_vot_overlap_rejects_bad_arguments():
    a = torch.zeros(2, 8, device="cuda")
    with pytest.raises(ValueError):
        ops.vot_overlap(a, torch.zeros(3, 8, device="cuda"), (10, 10))
    with pytest.raises(ValueError):
        ops.vot_overlap(a, a.double(), (10, 10))
    for v in (float("nan"), float("inf"), 2.0 ** 21):
        bad = a.clone()
        bad[1, 3] = v
        with pytest.raises(ValueError):
            ops.vot_overlap(a, bad, (10, 10))
    with pytest.raises(ValueError):
        ops.vot_overlap(a, a, (0, 10))


# ---------------------------------------------------------------------------------------------- 2. reinit
def test_reinit_equals_fresh_start(sd):
    T = 6
    vids = [make_frames(n=T, seed=s) for s in range(2)]
    frames = [np.stack([v[0][t] for v in vids], 0) for t in range(T)]
    a = BatchTracker(_net(sd, 2), _params())
    a.add(frames[0], [vids[0][1][0], vids[1][1][0]], frame_index=[0, 1])
    for t in (1, 2):
        a.track(frames[t], mask=False)
    pos = np.array([[151.25, 105.5], [140.0, 99.75]])
    sz = np.array([[48.5, 64.25], [47.0, 65.0]])
    a.reinit(a.ids, frames[2], pos, sz)
    b = BatchTracker(_net(sd, 2), _params())
    b.add_state(frames[2], pos, sz, frame_index=[0, 1])
    np.testing.assert_array_equal(a.state.cpu().numpy(), b.state.cpu().numpy())
    np.testing.assert_array_equal(a.avg.cpu().numpy(), b.avg.cpu().numpy())
    for t in (3, 4, 5):
        ra, rb = a.track(frames[t], mask=False), b.track(frames[t], mask=False)
        np.testing.assert_array_equal(ra.state.cpu().numpy(), rb.state.cpu().numpy(), err_msg=f"frame {t}")


def test_reinit_rejects_bad_arguments(sd):
    frames, boxes = make_frames(n=2)
    bt = BatchTracker(_net(sd, 2), _params())
    ids = bt.add(frames[0], [boxes[0]])
    with pytest.raises(ValueError):
        bt.reinit([ids[0] + 7], frames[1], [[1.0, 2.0]], [[30.0, 30.0]])
    with pytest.raises(ValueError):
        bt.reinit(ids, frames[1], [[1.0, 2.0], [3.0, 4.0]], [[30.0, 30.0], [30.0, 30.0]])


# ---------------------------------------------------------------------------------------------- 3. VotRunner
FAR = np.array([0.0, 0.0, 10.0, 0.0, 10.0, 10.0, 0.0, 10.0])        # a gt quad in the far corner: overlap 0


def _sequence(seed, T, fail_at=()):
    frames, boxes = make_frames(n=T, seed=seed)
    gt = np.asarray([[x, y, x + w, y, x + w, y + h, x, y + h] for (x, y, w, h) in boxes], np.float64)
    gt[0] += np.array([0.5, 0.25, -0.5, 0.25, -0.5, -0.75, 0.5, -0.75])            # not a plain box at init
    for f in fail_at:
        gt[f] = FAR
    return frames, gt


def _run(runner, seqs):
    G = len(seqs)
    T = max(len(s[0]) for s in seqs)
    frame = lambda f: np.stack([s[0][min(f, len(s[0]) - 1)] for s in seqs])     # noqa: E731
    runner.open(frame(0), [s[1] for s in seqs])
    for f in range(1, T):
        runner.frame(frame(f))
    regions, lost = runner.result()
    assert lost.shape == (G, runner.K)
    return regions, lost


def _check(regions, lost, seqs, combos, ref_net, tmp_path=None):
    for g, (frames, gt) in enumerate(seqs):
        fdev = [torch.from_numpy(f).cuda() for f in frames]
        for k in range(len(combos)):
            hp = {**HP, **combos[k]}
            want, want_lost = vot_reference.track_vot(ref_net, fdev, gt, hp)
            got = regions[g][k]
            assert len(got) == len(want) == len(frames)
            assert [r if isinstance(r, int) else 3 for r in got] == [r if isinstance(r, int) else 3 for r in want], \
                (g, k)
            assert lost[g, k] == want_lost, (g, k)
            for f, (x, y) in enumerate(zip(got, want)):
                if not isinstance(x, int):
                    np.testing.assert_allclose(x, y, rtol=0, atol=1e-5, err_msg=f"sequence {g} combo {k} frame {f}")
            if tmp_path is not None:
                path = tmp_path / f"s{g}_{k}.txt"
                vot.write_result(path, got)
                mine = path.read_text().splitlines()
                theirs = vot_reference.result_lines(want, lambda v: "%.4f" % float(np.float32(v))).splitlines()
                assert len(mine) == len(theirs)
                for m, t in zip(mine, theirs):
                    if "," in t:
                        np.testing.assert_allclose([float(v) for v in m.split(",")],
                                                   [float(v) for v in t.split(",")], rtol=0, atol=1.1e-4)
                    else:
                        assert m == t


def test_vot_runner_failures_and_unequal_lengths(sd, tmp_path):
    seqs = [_sequence(0, 16, fail_at=(1, 9)),       # a failure at frame 1 and a second one later
            _sequence(1, 11, fail_at=(7,)),         # 7 + 5 >= 11: the sequence ends before the re-init
            _sequence(2, 6)]
    runner = smb.VotRunner(_net(sd, 3), _params())
    regions, lost = _run(runner, seqs)
    assert (lost[:, 0] >= [2, 1, 0]).all()                 # the injected failures (the tracker may lose more)
    _check(regions, lost, seqs, [{}], _net(sd, 1), tmp_path)


def test_vot_runner_grid_crosses_the_lane_split(sd):
    combos = grid([0.04, 0.2], [0.4, 0.1], [1.0])                     # K = 4
    seqs = [_sequence(s, 9, fail_at=((2,) if s % 2 else (6,))) for s in range(5)]    # 5 x 4 = 20 streams
    runner = smb.VotRunner(_net(sd, 20), _params(), combos)
    regions, lost = _run(runner, seqs)
    cdicts = [{"penalty_k": pk, "window_influence": wi, "lr": lr} for pk, wi, lr in combos]
    _check(regions, lost, seqs, cdicts, _net(sd, 1))


def test_vot_runner_rpn_engine(sd):
    seqs = [_sequence(3, 10, fail_at=(3,)), _sequence(4, 8)]
    runner = smb.VotRunner(_net(sd, 2, mask=False), _params())
    regions, lost = _run(runner, seqs)
    _check(regions, lost, seqs, [{}], _net(sd, 1, mask=False))


def test_vot_runner_frame_does_not_wait_for_the_device(sd):
    """A frame that neither re-initialises nor retires a stream queues its work without a host sync: frames 1-5 (no
    re-init can be due before frame 6, and the sequences are longer) run with torch's sync check set to raise.  The
    later frames re-initialise (the failure at frame 2) and retire streams, as usual."""
    seqs = [_sequence(s, 9, fail_at=(2,)) for s in range(2)]
    frames = [torch.from_numpy(np.stack([s[0][f] for s in seqs])).cuda() for f in range(9)]
    runner = smb.VotRunner(_net(sd, 2), _params())
    runner.open(frames[0], [s[1] for s in seqs])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for f in range(1, 6):
            runner.frame(frames[f])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    for f in range(6, 9):
        runner.frame(frames[f])
    regions, lost = runner.result()
    for g in range(2):                                  # the failure at frame 2 (or an earlier one) re-initialised
        assert lost[g, 0] >= 1 and any(isinstance(r, int) and r == 1 for r in regions[g][0][6:8])


def test_vot_runner_rejects_too_many_streams(sd):
    seqs = [_sequence(s, 4) for s in range(3)]
    runner = smb.VotRunner(_net(sd, 4), _params(), grid([0.04, 0.1], [0.4], [1.0]))  # 3 x 2 = 6 > 4
    with pytest.raises(ValueError):
        runner.open(np.stack([s[0][0] for s in seqs]), [s[1] for s in seqs])
    runner = smb.VotRunner(_net(sd, 4), _params())
    with pytest.raises(ValueError):
        runner.open(np.stack([s[0][0] for s in seqs]), [s[1][:, :4] for s in seqs])
    with pytest.raises(ValueError):
        runner.open(np.stack([s[0][0] for s in seqs]), [s[1] for s in seqs[:2]])
