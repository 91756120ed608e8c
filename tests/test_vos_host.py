"""Host-side pieces of the multi-object VOS path that need no GPU: the track_vos fusion restatement on hand-built cases,
the label-box reduction against cv2.boundingRect, and the schedule function against the reference's conditions."""
import cv2
import numpy as np
import pytest

from siammask_b200.ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED
from siammask_b200.vos import schedule
from vos_reference import fuse_labels, label_box, make_multi_frames, schedule_ref


def test_fusion_hand_built_case():
    thr = 0.3
    H, W = 2, 4
    idle = np.full((H, W), -1.0)
    gt = np.array([[1, 0, 0, 1], [0, 0, 1, 1]], np.float64)              # init-frame GT mask (bool -> 1.0 / 0.0)
    soft = np.array([[0.2, 0.9, np.float32(0.3), 0.5],
                     [0.31, -1.0, 0.9, 1.0]], np.float64)                 # a pasted soft mask (border -1)
    pred = np.stack([idle, gt, soft, soft])                              # objects 3 and 4 tie everywhere
    got = fuse_labels(pred, thr)
    # float32(0.3) = 0.30000001192... > 0.3 in float64, although a float32 compare says no
    assert np.float64(np.float32(0.3)) > 0.3 and not np.float32(0.3) > np.float32(0.3)
    want = np.array([[2, 3, 3, 2],                                       # GT wins on 1.0; ties go to the lower index
                     [3, 0, 2, 2]], np.uint8)
    np.testing.assert_array_equal(got, want)
    # only idle objects: background; no objects at all: background
    np.testing.assert_array_equal(fuse_labels(np.stack([idle, idle]), thr), np.zeros((H, W), np.uint8))
    np.testing.assert_array_equal(fuse_labels(np.zeros((0, H, W)), thr), np.zeros((H, W), np.uint8))


def test_label_box_equals_cv2_bounding_rect():
    rng = np.random.RandomState(3)
    for trial in range(40):
        h, w = rng.randint(1, 40), rng.randint(1, 40)
        anno = (rng.rand(h, w) < rng.rand() * 0.2).astype(np.uint8) * rng.randint(1, 4, (h, w)).astype(np.uint8)
        if trial % 5 == 0:                           # objects touching every border
            anno[0, :] = anno[-1, :] = anno[:, 0] = anno[:, -1] = 2
        for oid in range(0, 5):
            want = cv2.boundingRect((anno == oid).astype(np.uint8))
            assert label_box(anno, oid) == tuple(want), (trial, oid)


@pytest.mark.parametrize("start,end", [(0, 7), (2, 5), (3, 3), (4, 2), (6, 100)])
def test_schedule_matches_reference_conditions(start, end):
    code = {"init": OBJ_INIT, "track": OBJ_TRACKED, "idle": OBJ_IDLE}
    for f in range(10):
        assert schedule([start], [end], f)[0] == code[schedule_ref(start, end, f)], f


def test_schedule_is_vectorised():
    starts, ends = [0, 2, 5], [4, 3, 9]
    got = np.stack([schedule(starts, ends, f) for f in range(8)])
    want = np.array([[code for code in
                      [{"init": OBJ_INIT, "track": OBJ_TRACKED, "idle": OBJ_IDLE}[schedule_ref(s, e, f)]
                       for s, e in zip(starts, ends)]] for f in range(8)])
    np.testing.assert_array_equal(got, want)


def test_multi_frames_overlap_and_lifetimes():
    frames, annos, objs = make_multi_frames()
    assert len(frames) == len(annos) == 8 and frames[0].dtype == np.uint8 and frames[0].shape == (240, 320, 3)
    for oid, s, e in objs:
        present = [bool((a == oid).any()) for a in annos]
        assert present == [s <= f <= e for f in range(len(annos))], oid
    # objects 1 and 2 overlap at some frame: their drawn boxes intersect, so one occludes the other
    def box(a, oid):
        return label_box(a, oid)
    overlapped = False
    for f, a in enumerate(annos):
        b1, b2 = box(a, 1), box(a, 2)
        if b1[2] and b2[2]:
            ix = min(b1[0] + b1[2], b2[0] + b2[2]) - max(b1[0], b2[0])
            iy = min(b1[1] + b1[3], b2[1] + b2[3]) - max(b1[1], b2[1])
            overlapped |= ix > 0 and iy > 0
    assert overlapped


def test_paste_labels_checks_offsets_on_the_host():
    from siammask_b200.ops import paste_labels
    many = [(OBJ_IDLE, 0)] * 256
    with pytest.raises(ValueError, match="255"):                  # labels are uint8
        paste_labels(None, None, None, [0, 256], many, (4, 4), 0.3)
    with pytest.raises(ValueError):                               # offsets must cover the objects
        paste_labels(None, None, None, [0, 2], [(OBJ_IDLE, 0)] * 3, (4, 4), 0.3)
    with pytest.raises(ValueError):                               # and rise monotonically
        paste_labels(None, None, None, [0, 2, 1, 3], [(OBJ_IDLE, 0)] * 3, (4, 4), 0.3)
