"""TEST INFRASTRUCTURE ONLY (checker) for VideoSegmenter's scoring (siammask_b200/vos.py).  Nothing under
`siammask_b200/` imports this module.

`multi_batch_iou_meter` restates MultiBatchIouMeter (tools/test.py:421-456) statement for statement, quirks included:
without a start dict the object ids are 1 .. num_objects by position, and with one each object's window is
range(start + 1, end - 1).  `count_frame` is the per-object (intersection, union) of one fused frame in numpy, the
definition `sm_paste_labels_iou` is checked against.
"""
from __future__ import annotations

import warnings

import numpy as np


def multi_batch_iou_meter(thrs, outputs, targets, start=None, end=None):
    targets = np.array(targets)
    outputs = np.array(outputs)

    num_frame = targets.shape[0]
    if start is None:
        object_ids = np.array(list(range(outputs.shape[0]))) + 1
    else:
        object_ids = [int(id) for id in start]

    num_object = len(object_ids)
    res = np.zeros((num_object, len(thrs)), dtype=np.float32)

    output_max_id = np.argmax(outputs, axis=0).astype('uint8') + 1
    outputs_max = np.max(outputs, axis=0)
    for k, thr in enumerate(thrs):
        output_thr = outputs_max > thr
        for j in range(num_object):
            target_j = targets == object_ids[j]

            if start is None:
                start_frame, end_frame = 1, num_frame - 1
            else:
                start_frame, end_frame = start[str(object_ids[j])] + 1, end[str(object_ids[j])] - 1
            iou = []
            for i in range(start_frame, end_frame):
                pred = (output_thr[i] * output_max_id[i]) == (j + 1)
                mask_sum = (pred == 1).astype(np.uint8) + (target_j[i] > 0).astype(np.uint8)
                intxn = np.sum(mask_sum == 2)
                union = np.sum(mask_sum > 0)
                if union > 0:
                    iou.append(intxn / union)
                elif union == 0 and intxn == 0:
                    iou.append(1)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", RuntimeWarning)        # np.mean of an empty window: NaN
                res[j, k] = np.mean(iou)
    return res


def count_frame(pred, anno, target_ids, thrs):
    """pred float64 [K,H,W] (one video's pred_masks at one frame), anno uint8 [H,W], target_ids int [K] (-1: matches no
    pixel) -> int64 [K,T,2] = (intersection, union) of (argmax + 1) * (max > thr) == k+1 and anno == target_ids[k]."""
    pred = np.asarray(pred, dtype=np.float64)
    K = pred.shape[0]
    out = np.zeros((K, len(thrs), 2), np.int64)
    if K == 0:
        return out
    max_id = np.argmax(pred, axis=0).astype(np.int64) + 1
    mx = np.max(pred, axis=0)
    for t, thr in enumerate(thrs):
        if thr < -1:
            out[:, t] = -1
            continue
        lab = (mx > thr) * max_id
        for k in range(K):
            p, g = lab == k + 1, anno.astype(np.int64) == target_ids[k]
            out[k, t] = (p & g).sum(), (p | g).sum()
    return out
