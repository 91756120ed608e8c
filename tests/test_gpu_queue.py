"""Whole benchmarks through one engine: `sm_mask_iou_ragged` against `sm_mask_iou` per size group and numpy counts over
cv2.warpAffine, `VotRunner.open_queue` against per-sequence `open` runs and the track_vot restatement, `VotScore` of a
queue run against split adds, `ParamSweep.open_queue` against per-video `open` runs and the tune_vos restatement, the
host waits of a queue step and the argument checks."""
import cv2
import numpy as np
import pytest
import torch

import siammask_b200 as smb
import vot_reference
from oracle.calibrate import calibrated_state_dict
from oracle.synthetic_video import make_frames
from siammask_b200 import ops, schedule
from siammask_b200.tracker import IMAGE_DESC, TrackerParams, image_table
from siammask_b200.tune import grid
from sweep_reference import tune_run

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}
FAR = np.array([0.0, 0.0, 10.0, 0.0, 10.0, 10.0, 0.0, 10.0])        # a gt quad in the far corner: overlap 0


def _params():
    return TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


def _net(sd, max_batch):
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch,
                      num_slots=max_batch).load_state_dict(sd).eval().to("cuda")


# ---------------------------------------------------------------------------------------------- 1. sm_mask_iou_ragged
def _crop_back_map(cx, cy, s, W, H, side=127):
    sub = [cx - s / 2, cy - s / 2, s, s]
    k = side / sub[2]
    back = [-sub[0] * k, -sub[1] * k, W * k, H * k]
    a, b = (W - 1) / back[2], (H - 1) / back[3]
    return np.array([a, 0, -a * back[0], 0, b, -b * back[1]], np.float64)


def _counts(pasted, anno, thrs):
    out = np.zeros((len(thrs), 2), np.int64)
    tgt = anno > 0
    for i, t in enumerate(thrs):
        pred = pasted.astype(np.float64) > t
        out[i] = (pred & tgt).sum(), (pred | tgt).sum()
    return out


def _ragged_case():
    rng = np.random.RandomState(7)
    sizes = [(150, 260), (1, 300), (5, 7)]              # (H, W) of the three annotation images
    side = 127
    yy, xx = np.mgrid[0:side, 0:side]
    masks = []
    for r in range(9):
        c = rng.rand(2) * 60 + 33
        d = np.sqrt((yy - c[0]) ** 2 + (xx - c[1]) ** 2)
        masks.append((1 / (1 + np.exp((d - 30) / 6))).astype(np.float32))
    masks[4][50:56, 40:70] = np.nan                      # NaN values compare false
    masks = np.stack(masks)
    # stream -> annotation image and its map (in that image's own size)
    video = np.array([0, 0, 1, 2, 0, 1, 2, 0, 1], np.int32)
    # crop_back maps, partly and wholly off frame; the one-row image gets maps that squeeze the mask onto its row
    spec = [(70, 60, 90), (240, 20, 110), [2.0, 0, 10, 0, 0.01, -0.3], (3, 2, 6), (100, 90, 80),
            [1.0, 0, -500, 0, 0.01, -0.3], (900, 900, 40), (10, 140, 200), [0.5, 0, 200, 0, 0.02, -1.0]]
    maps = np.stack([np.asarray(m, np.float64) if isinstance(m, list) else
                     _crop_back_map(*m, sizes[v][1], sizes[v][0]) for m, v in zip(spec, video)])
    annos = [np.zeros(s, np.uint8) for s in sizes]
    annos[0][30:100, 40:120] = 1
    annos[0][110:140, 200:250] = 2
    annos[1][0, 60:200] = 3
    # image 2 (5 x 7): empty target
    return masks, maps, video, sizes, annos


def test_mask_iou_ragged_equals_uniform_per_size_and_cv2():
    masks, maps, video, sizes, annos = _ragged_case()
    md, mp = torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda()
    packed = torch.from_numpy(np.concatenate([a.reshape(-1) for a in annos])).cuda()
    table = image_table(sizes, 1)
    one = ops.warp_affine(md[:1], mp[:1], (sizes[0][1], sizes[0][0]), -1.0).cpu().numpy()[0]
    present = float(one[(one > 0.4) & (one < 0.6)][0])                              # a value of a pasted mask
    thrs = np.r_[np.arange(0.3, 0.81, 0.05), present, -1.0, np.float64(np.float32(0.35)), 0.999]
    got = ops.mask_iou_ragged(md, mp, packed, table, video, thrs).cpu().numpy()
    assert got.shape == (len(masks), len(thrs), 2)
    for v, (H, W) in enumerate(sizes):                  # sm_mask_iou on each size group alone, bit for bit
        sel = np.nonzero(video == v)[0]
        want = ops.mask_iou(md[sel], mp[sel], torch.from_numpy(annos[v][None]).cuda(), [0] * len(sel), thrs)
        np.testing.assert_array_equal(got[sel], want.cpu().numpy(), err_msg=f"size group {v}")
    for b in range(len(masks)):
        H, W = sizes[video[b]]
        cvw = cv2.warpAffine(masks[b], maps[b].reshape(2, 3), (W, H), flags=cv2.INTER_LINEAR,
                             borderMode=cv2.BORDER_CONSTANT, borderValue=-1)
        np.testing.assert_array_equal(got[b], _counts(cvw, annos[video[b]], thrs), err_msg=f"stream {b}")
    assert (got[6] == 0).all()                           # empty target and a wholly off-frame mask: empty union
    assert (got[:, :, 0] > 0).any() and (got[:, :, 1] > got[:, :, 0]).any()
    assert (one == np.float32(present)).any()


def test_mask_iou_ragged_rejects_bad_tables_and_indices():
    masks, maps, video, sizes, annos = _ragged_case()
    md, mp = torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda()
    packed = torch.from_numpy(np.concatenate([a.reshape(-1) for a in annos])).cuda()
    table = image_table(sizes, 1)
    ops.mask_iou_ragged(md, mp, packed, table, video, [0.5])
    bad = []
    for field, i, v in (("offset", 2, table["offset"][2] + 1),           # past the buffer's end
                        ("offset", 1, -1), ("h", 0, -2),
                        ("h", 2, 0)):                                        # an empty image a stream reads
        t = table.copy()
        t[field][i] = v
        bad.append(t)
    bad.append(table.astype([("offset", "<i8"), ("h", "<i8"), ("w", "<i4")]))   # not sm_image_desc rows
    bad.append(np.zeros(0, IMAGE_DESC))
    for t in bad:
        with pytest.raises(ValueError):
            ops.mask_iou_ragged(md, mp, packed, t, video, [0.5])
    for v in (np.r_[video[:-1], 3], np.r_[video[:-1], -1], video[:-1], video.astype(np.float64)):
        with pytest.raises(ValueError):
            ops.mask_iou_ragged(md, mp, packed, table, v, [0.5])
    with pytest.raises(ValueError):
        ops.mask_iou_ragged(md, mp, packed.view(1, -1), table, video, [0.5])
    with pytest.raises(ValueError):
        ops.mask_iou_ragged(md, mp, packed, table, video, [-1.5])


# ---------------------------------------------------------------------------------------------- 2. VOT queue
VOT_SIZES = [(240, 320), (256, 352), (224, 304)]
# (length, failures) of 7 sequences: a failure at frame 1, two in one sequence, one in the last 5 frames
VOT_SEQS = [(3, ()), (40, (1, 20)), (12, (9,)), (25, (4,)), (7, ()), (18, (2, 14)), (31, (28,))]


def _vot_sequences():
    seqs = []
    for g, (T, fail) in enumerate(VOT_SEQS):
        H, W = VOT_SIZES[g % 3]
        frames, boxes = make_frames(n=T, h=H, w=W, seed=g)
        gt = np.asarray([[x, y, x + w, y, x + w, y + h, x, y + h] for (x, y, w, h) in boxes], np.float64)
        gt[0] += np.array([0.5, 0.25, -0.5, 0.25, -0.5, -0.75, 0.5, -0.75])
        for f in fail:
            gt[f] = FAR
        seqs.append(([torch.from_numpy(f).cuda() for f in frames], gt))
    return seqs


COMBOS = grid([0.04, 0.2], [0.4], [1.0, 0.45])[:3]


def _run_queue(runner, seqs, sync_free_steps=()):
    runner.open_queue([s[1] for s in seqs])
    step = 0
    while runner.pending:
        need = runner.needed()
        fr = [seqs[g][0][t] for g, t in need]
        if step in sync_free_steps:
            torch.cuda.set_sync_debug_mode("error")
        try:
            runner.step(fr)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        step += 1
    return runner


@pytest.fixture(scope="module")
def vot_runs(sd):
    seqs = _vot_sequences()
    queue = _run_queue(smb.VotRunner(_net(sd, 8), _params(), COMBOS), seqs)
    single = []
    net3 = _net(sd, 3)
    for frames, gt in seqs:
        r = smb.VotRunner(net3, _params(), COMBOS)
        r.open([frames[0]], [gt])
        for f in range(1, len(frames)):
            r.frame([frames[f]])
        single.append(r)
    return seqs, queue, single


def _same_regions(a, b):
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if isinstance(x, int) != isinstance(y, int):
            return False
        if isinstance(x, int) and x != y or not isinstance(x, int) and not np.array_equal(x, y):
            return False
    return True


def test_vot_queue_plan_spreads_and_waits():
    T = [n for n, _ in VOT_SEQS]
    steps = schedule.plan(T, 3, 8)
    first = {}
    for f, st in enumerate(steps):
        for s in st.admit:
            first.setdefault(s // 3, set()).add(f)
    # step 0 admits sequences 1 (40 frames) and 6 (31) and two combinations of sequence 3 (25); the rest wait
    assert first[1] == first[6] == {0} and len(first[3]) == 2 and min(first[3]) == 0
    assert all(min(first[g]) > 0 for g in (0, 2, 4, 5))


def test_vot_queue_equals_single_sequence_runs(vot_runs, sd):
    seqs, queue, single = vot_runs
    regions, lost = queue.result()
    assert lost.shape == (len(seqs), 3)
    for g, r in enumerate(single):
        reg, lo = r.result()
        np.testing.assert_array_equal(lost[g], lo[0], err_msg=f"sequence {g}")
        for k in range(3):
            assert _same_regions(regions[g][k], reg[0][k]), (g, k)
    assert (lost[1] >= 2).all() and (lost[6] >= 1).all()
    ref_net = _net(sd, 1)
    for g, (frames, gt) in enumerate(seqs):             # and the track_vot restatement
        for k, (pk, wi, lr) in enumerate(COMBOS):
            want, want_lost = vot_reference.track_vot(ref_net, frames, gt,
                                                      {**HP, "penalty_k": pk, "window_influence": wi, "lr": lr})
            got = regions[g][k]
            assert [x if isinstance(x, int) else 3 for x in got] == [x if isinstance(x, int) else 3 for x in want]
            assert lost[g, k] == want_lost
            for x, y in zip(got, want):
                if not isinstance(x, int):
                    np.testing.assert_allclose(x, y, rtol=0, atol=1e-5, err_msg=f"sequence {g} combo {k}")


def test_vot_score_of_a_queue_run_equals_split_adds(vot_runs):
    seqs, queue, single = vot_runs
    a = smb.VotScore(3, low=1, high=30).add(queue).result()
    b = smb.VotScore(3, low=1, high=30)
    for r in single:
        b.add(r)
    b = b.result()
    np.testing.assert_array_equal(a["lost_number"], b["lost_number"])
    np.testing.assert_array_equal(a["accuracy"], b["accuracy"])
    np.testing.assert_array_equal(a["robustness"], b["robustness"])
    np.testing.assert_array_equal(a["sequences"], b["sequences"])
    ca, cb = a["expected_overlaps"], b["expected_overlaps"]
    assert ca.shape == cb.shape
    assert (np.abs(ca.view(np.int32).astype(np.int64) - cb.view(np.int32).astype(np.int64)) <= 1).all()
    np.testing.assert_allclose(a["eao"], b["eao"], rtol=0, atol=1e-7)


def test_vot_queue_step_waits_only_to_admit_retire_or_reinit(sd):
    """Steps that neither admit, retire nor re-initialise streams run under torch's sync check set to raise, with CUDA
    frame lists.  A first run finds the re-initialising steps (the engine is deterministic)."""
    seqs = _vot_sequences()
    net = _net(sd, 8)
    first = _run_queue(smb.VotRunner(net, _params(), COMBOS), seqs)
    regions, _ = first.result()
    steps = schedule.plan([len(s[1]) for s in seqs], 3, 8)
    busy = {f for f, st in enumerate(steps) if st.admit or st.retire}
    for s in range(len(seqs) * 3):                     # a code 1 after frame 0 is a re-init at admission + t
        g, k = divmod(s, 3)
        busy |= {int(first._admit[s]) + t for t, x in enumerate(regions[g][k]) if t and isinstance(x, int) and x == 1}
    free = set(range(len(steps))) - busy
    assert len(free) > 10
    again = _run_queue(smb.VotRunner(net, _params(), COMBOS), seqs, sync_free_steps=free)
    r2, l2 = again.result()
    _, l1 = first.result()
    np.testing.assert_array_equal(l1, l2)
    assert all(_same_regions(regions[g][k], r2[g][k]) for g in range(len(seqs)) for k in range(3))


def test_vot_queue_rejects_bad_arguments(sd):
    seqs = _vot_sequences()[:2]
    runner = smb.VotRunner(_net(sd, 4), _params())
    with pytest.raises(ValueError):
        runner.open_queue([seqs[0][1], np.zeros((0, 8))])          # an empty sequence
    with pytest.raises(ValueError):
        runner.step([seqs[0][0][0]])                                # before open_queue
    runner.open_queue([s[1] for s in seqs])
    need = runner.needed()
    with pytest.raises(ValueError):
        runner.step([seqs[g][0][t] for g, t in need][:-1])          # one frame short
    with pytest.raises(ValueError):
        runner.frame([seqs[g][0][t] for g, t in need])              # frame() belongs to open()
    runner.step([seqs[g][0][t] for g, t in need])
    need = runner.needed()
    wrong = [seqs[g][0][t] for g, t in need]
    wrong[0] = torch.zeros(100, 120, 3, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        runner.step(wrong)                                          # not its sequence's frame-0 size
    while runner.pending:
        runner.step([seqs[g][0][t] for g, t in runner.needed()])
    with pytest.raises(ValueError):
        runner.step([seqs[0][0][0]])                                # the run has finished
    with pytest.raises(ValueError):
        runner.needed()


# ---------------------------------------------------------------------------------------------- 3. sweep queue
SWEEP_VIDEOS = [(9, (240, 320)), (5, (256, 352)), (12, (256, 352)), (3, (240, 320)), (7, (240, 320))]


def _sweep_videos():
    vids = []
    for g, (T, (H, W)) in enumerate(SWEEP_VIDEOS):
        frames, boxes = make_frames(n=T, h=H, w=W, seed=g + 3)
        annos = []
        for (x, y, w, h) in boxes:
            m = np.zeros((H, W), np.uint8)
            m[y:y + h, x:x + w] = 1
            m[y + 5:y + 9, x + 4:x + 40] = 0
            annos.append(torch.from_numpy(m).cuda())
        vids.append(([torch.from_numpy(f).cuda() for f in frames], boxes, annos))
    return vids


SWEEP_COMBOS = grid([0.0, 0.09], [0.3, 0.46], [0.8])


def test_sweep_queue_equals_per_video_runs_and_tune_vos(sd):
    vids = _sweep_videos()
    T = [len(v[0]) for v in vids]
    sweep = smb.ParamSweep(_net(sd, 6), _params(), SWEEP_COMBOS)
    sweep.open_queue([v[1][0] for v in vids], T)
    while sweep.pending:
        need = sweep.needed()
        sweep.step([vids[g][0][t] for g, t in need], [vids[g][2][t] if 0 < t < T[g] - 1 else None for g, t in need])
    iou_list, per_frame = sweep.result()
    assert iou_list.shape == (5, 4, 11) and [p.shape for p in per_frame] == [(t - 2, 4, 11) for t in T]
    net4, single = _net(sd, 4), _net(sd, 1)
    for g, (frames, boxes, annos) in enumerate(vids):
        ref = smb.ParamSweep(net4, _params(), SWEEP_COMBOS)
        ref.open(frames[0][None], [boxes[0]], num_frames=T[g])
        for f in range(1, T[g]):
            ref.frame(frames[f][None], annos[f][None] if f < T[g] - 1 else None)
        mean, rows = ref.result()
        np.testing.assert_array_equal(iou_list[g], mean[0], err_msg=f"video {g}")
        np.testing.assert_array_equal(per_frame[g], rows[:, 0], err_msg=f"video {g}")
        for k, (pk, wi, lr) in enumerate(SWEEP_COMBOS):
            hp = {**HP, "penalty_k": pk, "window_influence": wi, "lr": lr}
            iou, m, _ = tune_run(single, frames, [a.cpu().numpy() for a in annos], boxes[0], hp,
                                 np.arange(0.3, 0.81, 0.05))
            np.testing.assert_allclose(per_frame[g][:, k], iou, rtol=0, atol=1e-4, err_msg=f"video {g} combo {k}")
            np.testing.assert_allclose(iou_list[g, k], m, rtol=0, atol=1e-4, err_msg=f"video {g} combo {k}")
    assert all((p > 0).any() for p in per_frame)


def test_sweep_queue_step_waits_only_to_admit_or_retire(sd):
    vids = _sweep_videos()
    T = [len(v[0]) for v in vids]
    steps = schedule.plan(T, 4, 6)
    busy = {f for f, st in enumerate(steps) if st.admit or st.retire}
    sweep = smb.ParamSweep(_net(sd, 6), _params(), SWEEP_COMBOS)
    sweep.open_queue([v[1][0] for v in vids], T)
    f = 0
    while sweep.pending:
        need = sweep.needed()
        args = ([vids[g][0][t] for g, t in need], [vids[g][2][t] if 0 < t < T[g] - 1 else None for g, t in need])
        if f not in busy:
            torch.cuda.set_sync_debug_mode("error")
        try:
            sweep.step(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        f += 1
    assert len(set(range(len(steps))) - busy) > 3


def test_sweep_queue_rejects_bad_arguments(sd):
    vids = _sweep_videos()[:2]
    T = [len(v[0]) for v in vids]
    sweep = smb.ParamSweep(_net(sd, 4), _params(), SWEEP_COMBOS)
    with pytest.raises(ValueError):
        sweep.open_queue([v[1][0] for v in vids], [T[0], 2])        # too short to score a frame
    sweep.open_queue([v[1][0] for v in vids], T)
    need = sweep.needed()
    sweep.step([vids[g][0][t] for g, t in need], [None] * len(need))          # frame 0: nothing scored
    need = sweep.needed()
    fr = [vids[g][0][t] for g, t in need]
    with pytest.raises(ValueError):
        sweep.step(fr, [None] * len(need))                          # a scored frame without its annotation
    with pytest.raises(ValueError):
        sweep.step(fr[:-1], [vids[g][2][t] for g, t in need][:-1])
    with pytest.raises(ValueError):
        sweep.step(fr, [a[:10] for a in [vids[g][2][t] for g, t in need]])      # annotation of the wrong size
    while sweep.pending:
        need = sweep.needed()
        sweep.step([vids[g][0][t] for g, t in need], [vids[g][2][t] for g, t in need])
    with pytest.raises(ValueError):
        sweep.step([], [])
