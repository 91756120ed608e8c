"""A VOS dataset through one engine: `VideoSegmenter.open_queue` / `step` over videos of different lengths, frame sizes
and object counts, against per-video `open` runs (labels and `result()` bit for bit) and the track_vos / MultiBatchIouMeter
restatements, the host waits of a queue step, and the checks that reject bad input."""
import numpy as np
import pytest
import torch

import siammask_b200 as smb
from oracle.calibrate import calibrated_state_dict
from siammask_b200.tracker import TrackerParams
from siammask_b200.vos import VOS_THRESHOLDS, peak_width
from vos_reference import make_multi_frames, track_vos
from vos_score_reference import multi_batch_iou_meter

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}
SIZES = [(240, 320), (256, 352), (200, 296)]
# (length, size, objects (id, start, end, (x, y), (vx, vy), (cells w, cells h)))
VIDEOS = [
    (12, 0, [(1, 0, 11, (60.0, 70.0), (4.0, 1.0), (7, 6)), (2, 0, 11, (200.0, 90.0), (-4.0, 1.0), (6, 7))]),
    (30, 1, [(1, 0, 29, (50.0, 60.0), (3.0, 1.0), (7, 6)),
             (2, 3, 20, (220.0, 120.0), (-2.0, 1.0), (6, 6)),         # starts late, ends early
             (3, 21, 29, (150.0, 40.0), (1.0, 2.0), (6, 5)),          # starts the frame after object 2 ends
             (4, 5, 5, (100.0, 160.0), (2.0, -1.0), (5, 5))]),        # starts and ends on one frame
    (3, 2, [(1, 0, 2, (80.0, 60.0), (5.0, 3.0), (8, 7))]),
    (9, 0, [(2, 0, 8, (70.0, 80.0), (5.0, 2.0), (7, 7)),
            (5, 7, 8, (200.0, 140.0), (-3.0, -2.0), (6, 6))]),        # one frame after the last start
    (17, 1, [(1, 0, 16, (40.0, 50.0), (4.0, 2.0), (7, 6)), (2, 2, 16, (230.0, 60.0), (-3.0, 2.0), (6, 7)),
             (3, 4, 10, (120.0, 150.0), (2.0, -2.0), (6, 5)), (4, 6, 16, (180.0, 170.0), (-2.0, -3.0), (5, 6))]),
    (5, 2, [(3, 0, 4, (100.0, 80.0), (4.0, 3.0), (8, 8))]),
    (22, 0, [(1, 0, 21, (60.0, 60.0), (3.0, 2.0), (7, 6)), (2, 1, 12, (210.0, 130.0), (-3.0, -1.0), (6, 6))]),
]
MAX_BATCH = 5


def _params():
    return TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


def _net(sd, max_batch):
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch,
                      num_slots=max_batch).load_state_dict(sd).eval().to("cuda")


@pytest.fixture(scope="module")
def videos():
    out = []
    for g, (T, s, objs) in enumerate(VIDEOS):
        frames, annos, ol = make_multi_frames(n=T, h=SIZES[s][0], w=SIZES[s][1], seed=g, objects=objs)
        out.append(([torch.from_numpy(f).cuda() for f in frames], [torch.from_numpy(a).cuda() for a in annos], ol))
    return out


def _objects(videos):
    return [(g, oid, s, e) for g, (_, _, ol) in enumerate(videos) for (oid, s, e) in ol]


def _busy(seg):
    """Whether the pending step admits or retires a video or starts an object (the steps that may wait)."""
    st = seg._plan
    return bool(st.admit or st.retire) or any(seg.objects[k][2] == t for g, t in st.need for k in seg._members[g])


def _run_queue(sd, videos, score):
    seg = smb.VideoSegmenter(_net(sd, MAX_BATCH), _params())
    T = [len(v[0]) for v in videos]
    seg.open_queue(_objects(videos), T, score=score)
    labels, pos, n_free = {}, {}, 0
    while seg.pending:
        need, want = seg.needed(), seg.needs_anno()
        args = ([videos[g][0][t] for g, t in need], [videos[g][1][t] if w else None for (g, t), w in zip(need, want)])
        busy = _busy(seg)
        if not busy:
            torch.cuda.set_sync_debug_mode("error")
            n_free += 1
        try:
            out = seg.step(*args)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        st = seg.state()["target_pos"]
        for (g, t), lab in zip(need, out):
            labels[g, t] = lab.cpu().numpy()
            pos[g, t] = {k: st[k] for k, o in enumerate(seg.objects) if o[0] == g}
    return seg, labels, pos, n_free


def _run_single(sd, videos, score):
    net = _net(sd, 4)
    labels, res = {}, []
    for g, (frames, annos, ol) in enumerate(videos):
        seg = smb.VideoSegmenter(net, _params()).open([(0, oid, s, e) for (oid, s, e) in ol], num_frames=len(frames),
                                                      score=score)
        for t in range(len(frames)):
            labels[g, t] = seg.frame(frames[t][None], annos[t][None]).cpu().numpy()[0]
        if score is not None:
            res.append(seg.result()[0])
    return labels, res


class _NoSelect:
    """The engine behind the reference's plain model API only (numpy selection in ref_loop)."""
    def __init__(self, net):
        self._n = net
        self.anchors, self.anchor_num = net.anchors, net.anchor_num

    def template(self, z):
        return self._n.template(z)

    def track_mask(self, x):
        return self._n.track_mask(x)

    def track(self, x):
        return self._n.track(x)

    def track_refine(self, pos):
        return self._n.track_refine(pos)


@pytest.mark.parametrize("score", ["whole", "spans"])
def test_queue_equals_per_video_runs_and_track_vos(sd, videos, score):
    seg, labels, pos, n_free = _run_queue(sd, videos, score)
    widths = [peak_width([o[1] for o in ol], [o[2] for o in ol]) for _, _, ol in videos]
    assert sum(widths) > MAX_BATCH and max(widths) == 4 and seg.f < sum(len(v[0]) for v in videos)
    assert n_free > 10                                           # most steps ran with host waits forbidden
    single_labels, single_res = _run_single(sd, videos, score)
    assert set(labels) == set(single_labels) == {(g, t) for g, v in enumerate(videos) for t in range(len(v[0]))}
    for key, lab in labels.items():
        np.testing.assert_array_equal(lab, single_labels[key], err_msg=f"(video, frame) {key}")
    res = seg.result()
    assert len(res) == len(videos)
    for g in range(len(videos)):
        np.testing.assert_array_equal(res[g], single_res[g], err_msg=f"video {g}")        # NaN rows included
    if score == "spans":
        assert np.isnan(res[1][3]).all() and np.isnan(res[3][1]).all() and not np.isnan(res[4]).any()
    single = _NoSelect(_net(sd, 1))
    for g, (frames, annos, ol) in enumerate(videos):
        anp = [a.cpu().numpy() for a in annos]
        pred, _, rpos = track_vos(single, frames, [anp[s] for (_, s, _) in ol], [o[0] for o in ol],
                                  [o[1] for o in ol], [o[2] for o in ol], HP, HP["seg_thr"], device="cuda")
        ks = sorted(pos[g, 0])
        for t in range(len(frames)):
            for j, k in enumerate(ks):
                want, have = rpos[j, t], pos[g, t][k]
                assert np.isnan(want).all() == np.isnan(have).all(), (g, t, j)
                if not np.isnan(want).any():
                    np.testing.assert_allclose(have, want, rtol=0, atol=1e-5, err_msg=f"video {g} frame {t} obj {j}")
        if score == "whole":
            start = end = None
        else:
            start, end = {str(o[0]): o[1] for o in ol}, {str(o[0]): o[2] for o in ol}
        ref = multi_batch_iou_meter(VOS_THRESHOLDS, pred, anp, start=start, end=end)
        np.testing.assert_allclose(res[g], ref, rtol=0, atol=1e-4, err_msg=f"video {g}: result() vs track_vos")


def test_queue_rejects_bad_input(sd, videos):
    T = [len(v[0]) for v in videos]
    seg = smb.VideoSegmenter(_net(sd, MAX_BATCH), _params())
    with pytest.raises(ValueError, match="slots"):                   # video 4 has 4 objects at once
        smb.VideoSegmenter(_net(sd, 3), _params()).open_queue(_objects(videos), T)
    seg.open_queue(_objects(videos), T, score="whole")
    steps = 0
    while seg.pending:
        need, want = seg.needed(), seg.needs_anno()
        fr = [videos[g][0][t] for g, t in need]
        an = [videos[g][1][t] if w else None for (g, t), w in zip(need, want)]
        if steps == 1:
            with pytest.raises(ValueError, match="frames"):
                seg.step(fr[:-1], an)                                # one frame short
            wrong = list(fr)
            wrong[0] = torch.zeros(100, 120, 3, dtype=torch.uint8, device="cuda")
            with pytest.raises(ValueError, match="frame 0"):
                seg.step(wrong, an)                                  # not its video's frame-0 size
            missing = list(an)
            missing[want.index(True)] = None
            with pytest.raises(ValueError, match="required"):
                seg.step(fr, missing)
        seg.step(fr, an)
        steps += 1
    res = seg.result()
    clean, _, _, _ = _run_queue(sd, videos, "whole")
    for g, r in enumerate(clean.result()):                           # the rejected calls changed nothing
        np.testing.assert_array_equal(res[g], r)
    with pytest.raises(ValueError, match="pending"):
        seg.step([videos[0][0][0]], [None])
