"""siammask_b200 — H100-native (sm_90a) implementation of SiamMask's per-frame inference hot path.

Public surface mirrors the reference's model object for that path:
    Custom.template / track / track_mask / track_refine   (experiments/siammask_sharp/custom.py:173-190)
    conv2d_dw_group                                       (models/rpn.py:32-38)
    VideoSegmenter (multi-object track_vos on the device)  (tools/test.py:459-542)
    ParamSweep (tune_vos's hyper-parameter grid search)    (tools/tune_vos.py)
    VotRunner (track_vot / tune_vot, VOT supervised protocol) (tools/test.py:318-418, tools/tune_vot.py)
    VotScore (tools/eval.py's VOT accuracy, robustness and EAO)  (utils/pysot/evaluation)
All compute lives in libsiammask_b200.so (C ABI: include/siammask_b200.h)."""
from .custom import Custom, DEFAULT_ANCHORS
from .ops import conv2d_dw_group, xcorr_depthwise, conv2d, crop_resize, warp_affine, paste_labels, label_boxes, \
    mask_iou, paste_labels_iou, vot_overlap
from .checkpoint import synthetic_state_dict, load_checkpoint, expected_keys
from .vos import VideoSegmenter, VOS_THRESHOLDS
from .tune import ParamSweep
from .vot import VotRunner, VotScore

__all__ = ["Custom", "DEFAULT_ANCHORS", "conv2d_dw_group", "xcorr_depthwise", "conv2d", "crop_resize", "warp_affine",
           "paste_labels", "label_boxes", "mask_iou", "paste_labels_iou", "VideoSegmenter", "VOS_THRESHOLDS",
           "ParamSweep", "VotRunner", "VotScore", "vot_overlap", "synthetic_state_dict", "load_checkpoint", "expected_keys"]
