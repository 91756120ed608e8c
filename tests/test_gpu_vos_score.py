"""Scoring multi-object VOS on the device: the fused label map + per-object IoU counts (sm_paste_labels_iou) against
sm_paste_labels and numpy counts over cv2.warpAffine / sm_warp_affine, and VideoSegmenter(score=...) against the
MultiBatchIouMeter restatement in tests/vos_score_reference.py."""
import cv2
import numpy as np
import pytest
import torch

import siammask_b200 as smb
from siammask_b200.ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED, _paste_labels_iou, paste_labels, paste_labels_iou, \
    warp_affine
from siammask_b200.tracker import TrackerParams
from siammask_b200.vos import VOS_THRESHOLDS, schedule
from oracle.calibrate import calibrated_state_dict
from vos_reference import make_multi_frames, track_vos
from vos_score_reference import count_frame, multi_batch_iou_meter

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}
SIDE = 127


def _params():
    return TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


def _net(sd, max_batch, num_slots):
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch, num_slots=num_slots).load_state_dict(sd).eval() \
        .to("cuda")


def _crop_back_map(cx, cy, s, W, H, side=SIDE):
    """The forward map of crop_back (tools/test.py:263-275) for a square sub-window of size s at (cx, cy)."""
    sub = [cx - s / 2, cy - s / 2, s, s]
    k = side / sub[2]
    back = [-sub[0] * k, -sub[1] * k, W * k, H * k]
    a, b = (W - 1) / back[2], (H - 1) / back[3]
    return np.array([a, 0, -a * back[0], 0, b, -b * back[1]], np.float64)


def _values(objects, masks, maps, anno_g, H, W, dev_warp):
    """float64 [K,H,W]: each entry's value (pred_masks of one video and frame), pasted by sm_warp_affine (dev_warp) or
    by cv2.warpAffine (dev_warp None)."""
    vals = []
    for kind, arg in objects:
        if kind == OBJ_TRACKED:
            v = dev_warp[arg] if dev_warp is not None else cv2.warpAffine(
                masks[arg], maps[arg].reshape(2, 3), (W, H), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                borderValue=-1)
        elif kind == OBJ_INIT:
            v = (anno_g == arg).astype(np.float64)
        else:
            v = np.full((H, W), -1.0)
        vals.append(np.asarray(v, np.float64))
    return np.stack(vals) if vals else np.zeros((0, H, W))


def _check_counts(objects, target_ids, masks, maps, anno, thrs, seg_thr, private=False):
    """Runs the fused kernel on objects (one list per video) and checks labels against sm_paste_labels and counts against
    count_frame over both warps.  Returns the counts."""
    G, H, W = anno.shape
    off = np.concatenate([[0], np.cumsum([len(o) for o in objects])])
    flat = [e for o in objects for e in o]
    md, mp, ad = torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda(), torch.from_numpy(anno).cuda()
    if private:                                          # thresholds the public checks reject (below -1)
        labels, counts = _paste_labels_iou(md, mp, ad, off, flat,
                                           torch.tensor(target_ids, dtype=torch.int32, device="cuda"), (H, W), seg_thr,
                                           torch.tensor(thrs, dtype=torch.float64, device="cuda"))
    else:
        labels, counts = paste_labels_iou(md, mp, ad, off, flat, target_ids, (H, W), seg_thr, thrs)
    want = paste_labels(md, mp, ad, off, flat, (H, W), seg_thr)
    torch.cuda.synchronize()
    assert torch.equal(labels, want)
    counts = counts.cpu().numpy()
    assert counts.shape == (len(flat), len(thrs), 2)
    dev_warp = warp_affine(md, mp, (W, H), -1.0).cpu().numpy()
    for use_dev in (False, True):
        for g in range(G):
            pred = _values(objects[g], masks, maps, anno[g], H, W, dev_warp if use_dev else None)
            ref = count_frame(pred, anno[g], target_ids[off[g]:off[g + 1]], thrs)
            np.testing.assert_array_equal(counts[off[g]:off[g + 1]], ref, err_msg=f"video {g} (device warp {use_dev})")
    return counts


def test_labels_and_counts_three_videos_with_0_4_and_70_objects():
    rng = np.random.RandomState(11)
    G, H, W = 3, 72, 104
    n = 76
    yy, xx = np.mgrid[0:SIDE, 0:SIDE]
    masks = []
    for r in range(n):                                    # blob-shaped sigmoid masks
        c = rng.rand(2) * 60 + 33
        d = np.sqrt((yy - c[0]) ** 2 + (xx - c[1]) ** 2)
        masks.append((1 / (1 + np.exp((d - rng.rand() * 30 - 15) / 6))).astype(np.float32))
    masks = np.stack(masks)
    masks[3, 50:70, 50:70] = np.nan                       # NaN values: np.max is NaN there, label 0
    maps = np.stack([_crop_back_map(rng.rand() * W, rng.rand() * H, rng.rand() * 60 + 20, W, H) for _ in range(n)])
    anno = rng.randint(0, 6, (G, H, W)).astype(np.uint8)
    anno[:, :, :30] = 0
    objects = [[],
               [(OBJ_TRACKED, 3), (OBJ_INIT, 2), (OBJ_IDLE, 0), (OBJ_TRACKED, 0)],
               [(OBJ_TRACKED, 4 + k) for k in range(70)]]
    objects[2][5] = (OBJ_INIT, 1)
    objects[2][66] = (OBJ_INIT, 3)                         # an init entry in the second chunk
    objects[2][67] = (OBJ_IDLE, 0)
    objects[2][10] = (OBJ_TRACKED, 3)                      # NaN mask in the big video too
    # video 1: ids 4 (present), 2, -1 (not scored), 9 (absent); video 2: a permutation with -1 entries, absent ids, and
    # scored entries in the second chunk
    ids2 = list(rng.permutation(np.arange(6, 200))[:70])   # 1..5 are placed below
    ids2[1], ids2[5], ids2[66], ids2[69] = -1, 1, 3, 5
    ids2[0] = 2
    target_ids = np.array([4, 2, -1, 9] + ids2, np.int64)
    thrs = [0.3, 0.35, 0.4, 0.45, -1.0]
    counts = _check_counts(objects, target_ids, masks, maps, anno, thrs, HP["seg_thr"])
    assert (counts[4 + 5, :, 0] > 0).all()                 # init entries scored against their own ids, in both chunks
    assert (counts[4 + 66, :, 0] > 0).all()


def test_counts_threshold_equal_to_a_pasted_value_and_below_minus_one():
    rng = np.random.RandomState(12)
    G, H, W = 2, 60, 90
    masks = (rng.rand(3, SIDE, SIDE) * 0.9 + 0.05).astype(np.float32)
    maps = np.stack([_crop_back_map(40, 30, 70, W, H), _crop_back_map(55, 35, 60, W, H),
                     _crop_back_map(-400, -400, 50, W, H)])                          # entirely off frame
    anno = rng.randint(0, 4, (G, H, W)).astype(np.uint8)
    dev_warp = warp_affine(torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda(), (W, H), -1.0).cpu().numpy()
    v = float(dev_warp[0, 30, 40])                       # a pasted value: pixels equal to it do not pass
    assert (dev_warp[0] == np.float32(v)).any()
    objects = [[(OBJ_TRACKED, 0), (OBJ_TRACKED, 1), (OBJ_TRACKED, 2)], [(OBJ_TRACKED, 0), (OBJ_INIT, 3)]]
    target_ids = np.array([1, 7, 3, -1, 3])              # 7 is absent from the annotation
    thrs = [0.3, v, -1.0, -1.5, 0.45]
    counts = _check_counts(objects, target_ids, masks, maps, anno, thrs, HP["seg_thr"], private=True)
    assert (counts[:, 3] == -1).all() and (counts[:, [0, 1, 2, 4]] >= 0).all()
    assert counts[1, 0, 0] == 0 and counts[1, 0, 1] > 0   # absent id: no intersection, the union is the prediction


def test_counts_255_objects_32_thresholds():
    rng = np.random.RandomState(13)
    H, W, n = 40, 56, 255
    masks = rng.rand(n, SIDE, SIDE).astype(np.float32)
    maps = np.stack([_crop_back_map(rng.rand() * W, rng.rand() * H, rng.rand() * 30 + 8, W, H) for _ in range(n)])
    anno = rng.randint(0, 230, (1, H, W)).astype(np.uint8)     # ids 230..255 are absent
    objects = [[(OBJ_TRACKED, k) for k in range(n)]]
    for k in (0, 100, 200, 254):
        objects[0][k] = (OBJ_INIT, int(anno[0, 5, 5 + k % 40]))
    objects[0][130] = (OBJ_IDLE, 0)
    target_ids = rng.permutation(np.arange(1, 256)).astype(np.int64)
    target_ids[::17] = -1
    thrs = list(np.linspace(-1.0, 1.0, 32))
    counts = _check_counts(objects, target_ids, masks, maps, anno, thrs, 0.5)
    assert (counts[:, :, 1] > 0).sum() > 1000


# ---------------------------------------------------------------------------------------------- VideoSegmenter
def _run(sd, videos, objs, T, score, thrs=VOS_THRESHOLDS):
    """Runs a VideoSegmenter over G videos; returns (labels per frame, pred_masks per video rebuilt from the segmenter's
    own pasted masks, result() or None)."""
    seg = smb.VideoSegmenter(_net(sd, 8, 8), _params()).open(objs, num_frames=T, score=score, thrs=thrs)
    G = len(videos)
    H, W = videos[0][1][0].shape
    per_video = [[k for k, o in enumerate(objs) if o[0] == g] for g in range(G)]
    pred = [np.full((len(p), T, H, W), -1.0) for p in per_video]
    starts, ends = np.array([o[2] for o in objs]), np.array([o[3] for o in objs])
    labels = []
    for f in range(T):
        fr = np.stack([v[0][f] for v in videos])
        an = np.stack([v[1][f] for v in videos])
        labels.append(seg.frame(fr, an).cpu().numpy())
        kinds = schedule(starts, ends, f)
        r = getattr(seg, "last", None)
        rows = {sid: i for i, sid in enumerate(r.extras["ids"])} if r is not None else {}
        pasted = warp_affine(r.extras["mask_prob"], r.extras["maps"], (W, H), -1.0).cpu().numpy() if rows else None
        for g in range(G):
            for j, k in enumerate(per_video[g]):
                if kinds[k] == OBJ_INIT:
                    pred[g][j, f] = (videos[g][1][f] == objs[k][1]).astype(np.float64)
                elif kinds[k] == OBJ_TRACKED:
                    pred[g][j, f] = pasted[rows[seg._sid[k]]]
        seg.last = None
    return labels, pred, (seg.result() if score else None)


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


def _check_segmenter(sd, videos, objs, T, score):
    labels, pred, res = _run(sd, videos, objs, T, score)
    plain, _, _ = _run(sd, videos, objs, T, None)
    for f in range(T):
        np.testing.assert_array_equal(labels[f], plain[f], err_msg=f"frame {f}: scoring changed the labels")
    single = _NoSelect(_net(sd, 1, 1))
    assert len(res) == len(videos)
    for g, (frames, annos, _) in enumerate(videos):
        ol = [o for o in objs if o[0] == g]
        if score == "whole":
            start = end = None
        else:
            start = {str(o[1]): o[2] for o in ol}
            end = {str(o[1]): o[3] for o in ol}
        want = multi_batch_iou_meter(VOS_THRESHOLDS, pred[g], annos, start=start, end=end)
        assert res[g].dtype == np.float32 and res[g].shape == (len(ol), len(VOS_THRESHOLDS))
        np.testing.assert_array_equal(res[g], want, err_msg=f"video {g}: result() vs the restatement")
        fdev = [torch.from_numpy(f).cuda() for f in frames]
        ref_pred, _, _ = track_vos(single, fdev, [annos[o[2]] for o in ol], [o[1] for o in ol], [o[2] for o in ol],
                                   [o[3] for o in ol], HP, HP["seg_thr"], device="cuda")
        ref = multi_batch_iou_meter(VOS_THRESHOLDS, ref_pred, annos, start=start, end=end)
        np.testing.assert_allclose(res[g], ref, rtol=0, atol=1e-4, err_msg=f"video {g}: result() vs track_vos")
    return res


def test_video_segmenter_score_whole(sd):
    T = 8
    # DAVIS 2016/2017 style: every object starts at frame 0; video 1's ids 2 and 5 are scored as 1 and 2 by position
    v0 = make_multi_frames(n=T, seed=0, objects=[(1, 0, T - 1, (60.0, 70.0), (9.0, 2.0), (7, 6)),
                                                 (2, 0, T - 1, (200.0, 90.0), (-9.0, 1.0), (6, 7))])
    v1 = make_multi_frames(n=T, seed=1, objects=[(5, 0, T - 1, (40.0, 40.0), (5.0, 4.0), (8, 7)),
                                                 (2, 0, T - 1, (220.0, 130.0), (-6.0, -2.0), (6, 6))])
    videos = [v0, v1]
    objs = [(g, oid, s, e) for g, (_, _, ol) in enumerate(videos) for (oid, s, e) in ol]
    res = _check_segmenter(sd, videos, objs, T, "whole")
    assert not np.isnan(np.concatenate(res)).any()


def test_video_segmenter_score_spans(sd):
    T = 8
    v0 = make_multi_frames(n=T, seed=0)                  # ids 1, 2, 3 joining at frames 0, 1, 2
    v1 = make_multi_frames(n=T, seed=1, objects=[(2, 0, 5, (40.0, 40.0), (5.0, 4.0), (8, 7)),
                                                 (4, 3, 4, (150.0, 100.0), (2.0, 1.0), (6, 6)),     # empty window
                                                 (1, 3, T - 1, (220.0, 130.0), (-6.0, -2.0), (6, 6))])
    videos = [v0, v1]
    objs = [(g, oid, s, e) for g, (_, _, ol) in enumerate(videos) for (oid, s, e) in ol]
    res = _check_segmenter(sd, videos, objs, T, "spans")
    assert np.isnan(res[1][1]).all() and not np.isnan(res[1][[0, 2]]).any() and not np.isnan(res[0]).any()
