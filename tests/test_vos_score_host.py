"""Host-side pieces of VideoSegmenter's scoring (MultiBatchIouMeter of tools/test.py:421-456) that need no GPU: the
restatement against the golden the reference's own meter produced, the reduction from integer counts, the scoring
windows and target ids of both branches, and the argument checks."""
import os

import numpy as np
import pytest
import torch

from siammask_b200.ops import OBJ_IDLE, paste_labels_iou
from siammask_b200.vos import VOS_THRESHOLDS, VideoSegmenter, score_row, score_windows
from vos_score_reference import count_frame, multi_batch_iou_meter

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "multi_iou.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _spans(z):
    ids = [str(i) for i in z["spans_ids"]]
    return dict(zip(ids, (int(v) for v in z["spans_start"]))), dict(zip(ids, (int(v) for v in z["spans_end"])))


def test_restatement_equals_reference_golden(golden):
    z = golden
    got = multi_batch_iou_meter(z["whole_thrs"], z["whole_outputs"], z["whole_targets"])
    np.testing.assert_array_equal(got, z["whole_res"])
    start, end = _spans(z)
    got = multi_batch_iou_meter(z["spans_thrs"], z["spans_outputs"], z["spans_targets"], start=start, end=end)
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got, z["spans_res"])                 # NaN positions included
    assert np.isnan(z["spans_res"][3]).all() and not np.isnan(z["spans_res"][:3]).any()
    assert np.allclose(VOS_THRESHOLDS, z["whole_thrs"], rtol=0, atol=0)


def _reduce(outputs, targets, thrs, objects, num_frames, score):
    """What VideoSegmenter.result computes: per-frame integer counts (the kernel's definition, in numpy), then score_row
    over each object's window.  objects: (video 0, id, start, end)."""
    ids, lo, hi = score_windows(objects, num_frames, score)
    counts = np.stack([count_frame(outputs[:, f], targets[f], ids, thrs) for f in range(num_frames)])
    return np.stack([score_row(counts[:, k], lo[k], hi[k]) for k in range(len(objects))])


def test_host_reduction_equals_restatement(golden):
    z = golden
    F = z["whole_targets"].shape[0]
    objs = [(0, oid, 0, F - 1) for oid in (2, 5, 7)]                     # tracked ids; scored by position
    got = _reduce(z["whole_outputs"], z["whole_targets"], z["whole_thrs"], objs, F, "whole")
    np.testing.assert_array_equal(got, z["whole_res"])
    start, end = _spans(z)
    objs = [(0, int(k), start[k], end[k]) for k in start]
    got = _reduce(z["spans_outputs"], z["spans_targets"], z["spans_thrs"], objs, F, "spans")
    np.testing.assert_array_equal(got, z["spans_res"])
    # more frames than numpy's pairwise-summation block, so the order of the mean's sum matters
    rng = np.random.RandomState(5)
    F, K, H, W = 23, 3, 9, 11
    out = rng.rand(K, F, H, W) * 2 - 1
    tgt = rng.randint(0, 4, (F, H, W)).astype(np.uint8)
    objs = [(0, 1, 0, F - 1), (0, 2, 0, F - 1), (0, 3, 0, F - 1)]
    np.testing.assert_array_equal(_reduce(out, tgt, VOS_THRESHOLDS, objs, F, "whole"),
                                  multi_batch_iou_meter(VOS_THRESHOLDS, out, tgt))


def test_score_row_empty_window_is_nan_without_warning():
    import warnings
    c = np.zeros((5, 3, 2), np.int32)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        r = score_row(c, 3, 3)
    assert r.dtype == np.float32 and np.isnan(r).all()
    np.testing.assert_array_equal(score_row(c, 0, 5), np.ones(3, np.float32))    # empty unions count as IoU 1


def test_score_windows_both_branches():
    objs = [(0, 3, 0, 9), (1, 2, 2, 7), (0, 5, 1, 9), (0, 9, 4, 5), (1, 8, 0, 9)]
    ids, lo, hi = score_windows(objs, 10, "whole")
    np.testing.assert_array_equal(ids, [1, 1, 2, 3, 2])                 # k-th object of its video -> k + 1
    np.testing.assert_array_equal(lo, [1] * 5)
    np.testing.assert_array_equal(hi, [9] * 5)
    ids, lo, hi = score_windows(objs, 10, "spans")
    np.testing.assert_array_equal(ids, [3, 2, 5, 9, 8])
    np.testing.assert_array_equal(lo, [1, 3, 2, 5, 1])
    np.testing.assert_array_equal(hi, [8, 6, 8, 4, 8])                  # (0, 9, 4, 5): empty window
    with pytest.raises(ValueError):
        score_windows(objs, 10, "frames")


def test_paste_labels_iou_checks_on_the_host():
    anno = torch.zeros(2, 4, 4, dtype=torch.uint8)                     # CPU: every check below fires before it matters
    obj = [(OBJ_IDLE, 0)] * 3
    off = [0, 2, 3]
    with pytest.raises(ValueError, match="thresholds"):
        paste_labels_iou(None, None, anno, off, obj, [1, 2, 1], (4, 4), 0.3, [])
    with pytest.raises(ValueError, match="thresholds"):
        paste_labels_iou(None, None, anno, off, obj, [1, 2, 1], (4, 4), 0.3, np.linspace(0, 1, 33))
    with pytest.raises(ValueError, match=">= -1"):
        paste_labels_iou(None, None, anno, off, obj, [1, 2, 1], (4, 4), 0.3, [0.3, -1.5])
    with pytest.raises(ValueError, match="unique"):
        paste_labels_iou(None, None, anno, off, obj, [4, 4, 1], (4, 4), 0.3, VOS_THRESHOLDS)
    for bad in ([0, 2, 1], [1, 256, 1], [-2, 1, 1]):
        with pytest.raises(ValueError, match="1..255"):
            paste_labels_iou(None, None, anno, off, obj, bad, (4, 4), 0.3, VOS_THRESHOLDS)
    with pytest.raises(ValueError, match="target_ids"):
        paste_labels_iou(None, None, anno, off, obj, [1, 2], (4, 4), 0.3, VOS_THRESHOLDS)
    with pytest.raises(ValueError, match="obj_offsets"):
        paste_labels_iou(None, None, anno, [0, 2], obj, [1, 2, 1], (4, 4), 0.3, VOS_THRESHOLDS)
    with pytest.raises(ValueError, match="anno"):                      # not CUDA
        paste_labels_iou(None, None, anno, off, obj, [1, -1, -1], (4, 4), 0.3, VOS_THRESHOLDS)
    with pytest.raises(ValueError, match="anno"):                      # wrong dtype / shape
        paste_labels_iou(None, None, anno.float(), off, obj, [1, 2, 1], (4, 4), 0.3, VOS_THRESHOLDS)


class _HostTracker:
    """Just enough of BatchTracker for the checks VideoSegmenter makes before any device work."""
    dev = torch.device("cpu")
    p = None

    def _clear(self):
        pass

    def _frames(self, frames):
        return torch.as_tensor(np.asarray(frames))


def _segmenter():
    seg = VideoSegmenter.__new__(VideoSegmenter)
    seg.tracker, seg.p, seg.dev, seg.objects, seg.score = _HostTracker(), None, torch.device("cpu"), [], None
    return seg


def test_video_segmenter_scoring_checks():
    seg = _segmenter()
    objs = [(0, 1, 0), (0, 2, 2), (1, 1, 0)]
    with pytest.raises(ValueError, match="num_frames"):
        seg.open(objs, score="whole")
    with pytest.raises(ValueError, match="score"):
        seg.open(objs, num_frames=6, score="all")
    with pytest.raises(ValueError, match="thresholds"):
        seg.open(objs, num_frames=6, score="whole", thrs=np.linspace(0, 1, 40))
    with pytest.raises(ValueError, match=">= -1"):
        seg.open(objs, num_frames=6, score="spans", thrs=[-2.0])
    with pytest.raises(ValueError, match="unique"):                    # the same id twice in one video
        seg.open([(0, 1, 0), (0, 1, 2)], num_frames=6, score="spans")
    seg.open([(0, 1, 0), (0, 1, 2)], num_frames=6, score="whole")      # positional ids 1, 2 are unique
    with pytest.raises(ValueError, match="end_frame"):
        seg.open([(0, 1, 0, 9)], num_frames=6, score="spans")
    seg.open([(0, 1, 0, 9)])                                          # without scoring nothing changes
    # a frame inside a window without annotations
    seg.open([(0, 1, 0, 5), (0, 2, 2, 5)], num_frames=6, score="spans")
    seg.f = 3                                                          # object 1's window is [1, 4)
    frames = np.zeros((1, 4, 4, 3), np.uint8)
    with pytest.raises(ValueError, match="scored"):
        seg.frame(frames)
    seg.open([(0, 1, 0, 5)], num_frames=6, score="whole")
    seg.f = 1
    with pytest.raises(ValueError, match="scored"):
        seg.frame(frames)
    seg.f = 6
    with pytest.raises(ValueError, match="num_frames"):
        seg.frame(frames)
    with pytest.raises(ValueError, match="score"):
        _segmenter().result()
