"""Standalone operators of the hot path, bound to the C ABI (CUDA tensors in, CUDA tensors out).

`conv2d_dw_group` keeps the reference's name and argument order (models/rpn.py:32-38)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def conv2d_dw_group(x: torch.Tensor, kernel: torch.Tensor) -> torch.Tensor:
    """Depthwise cross-correlation: x f32[B,C,H,W], kernel f32[B,C,kh,kw] -> f32[B,C,H-kh+1,W-kw+1].
    Like the reference it requires paired batches (kernel.shape[:2] == x.shape[:2])."""
    if not (x.is_cuda and kernel.is_cuda):
        raise RuntimeError("siammask_b200 operators run on CUDA tensors only; there is no CPU path")
    if x.shape[:2] != kernel.shape[:2]:
        raise RuntimeError(f"paired batch required: x {tuple(x.shape)} vs kernel {tuple(kernel.shape)}")
    lib = _lib.load()
    x = x.to(torch.float32).contiguous()
    kernel = kernel.to(torch.float32).contiguous()
    B, Cn, H, W = x.shape
    kh, kw = kernel.shape[2:]
    out = torch.empty(B, Cn, H - kh + 1, W - kw + 1, device=x.device, dtype=torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(lib.sm_xcorr_depthwise(x.data_ptr(), kernel.data_ptr(), out.data_ptr(), B, Cn, H, W, kh, kw,
                                          _stream(x.device)))
    return out


xcorr_depthwise = conv2d_dw_group


CONV_ROUTES = {_lib.SM_CONV_ROUTE_SIMT: "simt", _lib.SM_CONV_ROUTE_GEMM_TILED: "gemm_tiled",
               _lib.SM_CONV_ROUTE_GEMM_IM2COL: "gemm_im2col", _lib.SM_CONV_ROUTE_PATCH: "patch"}


def conv2d_route(x_shape, w_shape, stride=1, padding=0, dilation=1, backend="tensor", precision="exact") -> str:
    """The kernel `conv2d` runs for these shapes (C ABI `sm_conv2d_route`, no device needed): 'simt', 'gemm_tiled',
    'gemm_im2col' or 'patch'.  Raises RuntimeError for the arguments `conv2d` rejects."""
    if len(x_shape) != 4 or len(w_shape) != 4 or int(w_shape[1]) != int(x_shape[1]):
        raise RuntimeError(f"conv2d needs x [B,Cin,H,W] and weight [Cout,Cin,KH,KW], got {tuple(x_shape)} and "
                           f"{tuple(w_shape)}")
    be = {"tensor": _lib.SM_BACKEND_TENSOR, "simt": _lib.SM_BACKEND_SIMT}[backend]
    pr = {"exact": _lib.SM_PRECISION_EXACT, "fast": _lib.SM_PRECISION_FAST}[precision]
    B, Cin, H, W = (int(v) for v in x_shape)
    Cout, _, KH, KW = (int(v) for v in w_shape)
    route = C.c_int32(-1)
    _lib.check(_lib.load().sm_conv2d_route(B, Cin, H, W, Cout, KH, KW, int(stride), int(padding), int(dilation), be, pr,
                                           C.byref(route)))
    return CONV_ROUTES[route.value]


def conv2d(x, weight, scale=None, shift=None, stride=1, padding=0, dilation=1, relu=False, backend="tensor",
           precision="exact", out=None):
    """F.conv2d(x, weight) * scale[c] + shift[c] (+ReLU) through the engine's convolution kernels.
    x f32[B,Cin,H,W] NCHW, weight f32[Cout,Cin,KH,KW]; returns f32 NCHW, written into `out` when given (a contiguous
    f32 tensor of the output's shape on x's device).  The geometry is checked first (`conv2d_route`)."""
    conv2d_route(x.shape, weight.shape, stride, padding, dilation, backend, precision)
    for name, t in (("scale", scale), ("shift", shift)):
        if t is not None and t.numel() != weight.shape[0]:
            raise RuntimeError(f"{name} must have one entry per output channel ({weight.shape[0]})")
    if not x.is_cuda:
        raise RuntimeError("siammask_b200 operators run on CUDA tensors only; there is no CPU path")
    lib = _lib.load()
    dev = x.device
    x = x.to(torch.float32).contiguous()
    weight = weight.to(dev, torch.float32).contiguous()
    B, Cin, H, W = x.shape
    Cout, _, KH, KW = weight.shape
    Ho = (H + 2 * padding - dilation * (KH - 1) - 1) // stride + 1
    Wo = (W + 2 * padding - dilation * (KW - 1) - 1) // stride + 1
    if out is None:
        out = torch.empty(B, Cout, Ho, Wo, device=dev, dtype=torch.float32)
    elif (tuple(out.shape) != (B, Cout, Ho, Wo) or out.dtype != torch.float32 or out.device != dev
          or not out.is_contiguous()):
        raise RuntimeError(f"out must be a contiguous float32 tensor of shape {(B, Cout, Ho, Wo)} on {dev}")
    sc = scale.to(dev, torch.float32).contiguous() if scale is not None else None
    sh = shift.to(dev, torch.float32).contiguous() if shift is not None else None
    be = {"tensor": _lib.SM_BACKEND_TENSOR, "simt": _lib.SM_BACKEND_SIMT}[backend]
    pr = {"exact": _lib.SM_PRECISION_EXACT, "fast": _lib.SM_PRECISION_FAST}[precision]
    with torch.cuda.device(dev):
        _lib.check(lib.sm_conv2d(x.data_ptr(), weight.data_ptr(), sc.data_ptr() if sc is not None else None,
                                 sh.data_ptr() if sh is not None else None, out.data_ptr(), B, Cin, H, W, Cout, KH, KW,
                                 stride, padding, dilation, int(relu), be, pr, _stream(dev)))
    return out


def crop_resize(frames: torch.Tensor, boxes, model_size: int) -> torch.Tensor:
    """Device form of get_subwindow_tracking (tools/test.py:67-110).  frames: uint8 CUDA tensor [H,W,3] (shared by all
    boxes) or [B,H,W,3]; boxes: int [B,6] = (context_xmin, context_ymin, original_sz, avg0, avg1, avg2) in frame
    coordinates before padding.  Returns f32 [B,3,model,model], bit-identical to the cv2 path."""
    if not frames.is_cuda or frames.dtype != torch.uint8:
        raise RuntimeError("crop_resize expects uint8 CUDA frames; there is no CPU path")
    lib = _lib.load()
    dev = frames.device
    frames = frames.contiguous()
    bx = torch.as_tensor(boxes, dtype=torch.int32).reshape(-1, 6)
    B = bx.shape[0]
    full = torch.zeros(B, 8, dtype=torch.int32)
    full[:, :6] = bx
    full = full.to(dev)
    if frames.dim() == 3:
        H, W, stride = frames.shape[0], frames.shape[1], 0
    else:
        if frames.shape[0] != B:
            raise ValueError("one frame per box expected")
        H, W, stride = frames.shape[1], frames.shape[2], frames.shape[1] * frames.shape[2] * 3
    out = torch.empty(B, 3, model_size, model_size, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_crop_resize(frames.data_ptr(), stride, H, W, full.data_ptr(), B, model_size, out.data_ptr(),
                                      _stream(dev)))
    return out


def warp_affine(src: torch.Tensor, maps, dsize, border_value: float = -1.0) -> torch.Tensor:
    """cv2.warpAffine(src, M, dsize, INTER_LINEAR, BORDER_CONSTANT, border_value) on the device (crop_back,
    tools/test.py:263-275).  src f32 CUDA [h,w] or [B,h,w]; maps: forward 2x3 map(s); dsize = (width, height)."""
    if not src.is_cuda:
        raise RuntimeError("warp_affine expects a CUDA tensor; there is no CPU path")
    lib = _lib.load()
    dev = src.device
    squeeze = src.dim() == 2
    s3 = (src.unsqueeze(0) if squeeze else src).to(torch.float32).contiguous()
    B, sh, sw = s3.shape
    m = torch.as_tensor(maps, dtype=torch.float64).reshape(-1, 6)
    if m.shape[0] != B:
        raise ValueError("one 2x3 map per image expected")
    m = m.to(dev).contiguous()
    dw, dh = int(dsize[0]), int(dsize[1])
    out = torch.empty(B, dh, dw, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_warp_affine(s3.data_ptr(), sh, sw, m.data_ptr(), out.data_ptr(), dh, dw, float(border_value), B,
                                      _stream(dev)))
    return out[0] if squeeze else out


OBJ_IDLE, OBJ_TRACKED, OBJ_INIT = 0, 1, 2          # SM_OBJ_* of include/siammask_b200.h


def paste_labels(masks, maps, anno, obj_offsets, objects, size, seg_thr: float) -> torch.Tensor:
    """Fused paste-back + multi-object label map of track_vos (tools/test.py:480-523, C ABI `sm_paste_labels`).
    masks f32 CUDA [rows,side,side] (sigmoid masks) and maps f64 [rows,6] (forward paste-back maps) of the tracked
    objects, or None when no object is tracked; anno uint8 CUDA [G,H,W] (or None when no object is initialised);
    obj_offsets int32 [G+1]: the objects of video g are entries obj_offsets[g]..obj_offsets[g+1]-1 of objects int32
    [n,2] = (kind, arg) with kind OBJ_TRACKED (arg = row), OBJ_INIT (arg = label id) or OBJ_IDLE; size = (H, W).
    Returns labels uint8 [G,H,W] = (first argmax over the video's objects + 1) * (max > seg_thr) in float64.
    The offsets are checked on the host (one D2H copy if they live on the device): non-decreasing, covering `objects`,
    at most 255 objects per video (labels are uint8)."""
    _check_offsets(obj_offsets, _num_entries(objects))
    return _paste_labels(masks, maps, anno, obj_offsets, objects, size, seg_thr)


def _paste_labels(masks, maps, anno, obj_offsets, objects, size, seg_thr: float, ragged=None) -> torch.Tensor:
    """`paste_labels` without the host-side check of the offsets (callers that validated their tables once).
    ragged = (desc, total): videos of different sizes (`sm_paste_labels_ragged`): desc the device sm_image_desc table of
    the G videos, total the packed label buffer's length; anno (if given) is that packed uint8 buffer, size = (max_h,
    max_w), and the packed labels uint8 [total] are returned."""
    off = torch.as_tensor(obj_offsets, dtype=torch.int32).reshape(-1)
    G = off.numel() - 1
    H, W = int(size[0]), int(size[1])
    ref = masks if masks is not None else anno
    dev = ref.device if ref is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise RuntimeError("paste_labels expects CUDA tensors; there is no CPU path")
    lib = _lib.load()
    off = off.to(dev).contiguous()
    obj = torch.as_tensor(objects, dtype=torch.int32).reshape(-1, 2)
    obj = (obj if obj.numel() else torch.zeros(1, 2, dtype=torch.int32)).to(dev).contiguous()
    side = 1
    if masks is not None:
        masks = masks.to(dev, torch.float32).contiguous()
        side = int(masks.shape[-1])
        maps = torch.as_tensor(maps, dtype=torch.float64).reshape(-1, 6).to(dev).contiguous()
    shape = (G, H, W) if ragged is None else (int(ragged[1]),)
    if anno is not None:
        anno = anno.to(dev).contiguous()
        if anno.dtype != torch.uint8 or tuple(anno.shape) != shape:
            raise ValueError(f"anno must be uint8 {list(shape)}")
    out = torch.empty(shape, dtype=torch.uint8, device=dev)

    def ptr(t):
        return t.data_ptr() if t is not None else None
    with torch.cuda.device(dev):
        if ragged is None:
            _lib.check(lib.sm_paste_labels(ptr(masks), side, ptr(maps) if masks is not None else None, ptr(anno),
                                           off.data_ptr(), obj.data_ptr(), G, H, W, float(seg_thr), out.data_ptr(),
                                           _stream(dev)))
        else:
            _lib.check(lib.sm_paste_labels_ragged(ptr(masks), side, ptr(maps) if masks is not None else None, ptr(anno),
                                                  off.data_ptr(), obj.data_ptr(), ragged[0].data_ptr(), G, H, W,
                                                  float(seg_thr), out.data_ptr(), _stream(dev)))
    return out


def _num_entries(objects) -> int:
    return int(np.prod(objects.shape[:-1])) if torch.is_tensor(objects) else len(np.asarray(objects).reshape(-1, 2))


def _check_offsets(obj_offsets, n: int) -> np.ndarray:
    off = np.asarray(obj_offsets.cpu() if torch.is_tensor(obj_offsets) else obj_offsets, dtype=np.int64).reshape(-1)
    if off.size < 2 or off[0] != 0 or off[-1] != n or (np.diff(off) < 0).any():
        raise ValueError(f"obj_offsets must rise from 0 to the number of objects ({n})")
    if (np.diff(off) > 255).any():
        raise ValueError("at most 255 objects per video (labels are uint8)")
    return off


def paste_labels_iou(masks, maps, anno, obj_offsets, objects, target_ids, size, seg_thr: float, thrs):
    """`paste_labels` fused with the per-object IoU counts of the reference's MultiBatchIouMeter (tools/test.py:421-456)
    for one frame (C ABI `sm_paste_labels_iou`).  The arguments of `paste_labels` mean the same, but anno uint8 CUDA
    [G,H,W] is required; target_ids int [n]: the annotation value entry i is scored against (1..255, unique within its
    video) or -1 (not scored: it matches no pixel); thrs: 1..32 thresholds >= -1.  Returns (labels uint8 [G,H,W], equal
    to `paste_labels` bit for bit, counts int32 [n,T,2]) where counts[i,t] = (intersection, union) of
    label_t == k+1 and anno[g] == target_ids[i], label_t = (first argmax + 1) * (max > thrs[t]) in float64 and k the
    entry's position within its video g.  The checks read the offsets, target_ids and thrs on the host."""
    from .tune import _check_thresholds
    n = _num_entries(objects)
    off = _check_offsets(obj_offsets, n)
    t = _check_thresholds(thrs.cpu() if torch.is_tensor(thrs) else thrs)
    ids = np.asarray(target_ids.cpu() if torch.is_tensor(target_ids) else target_ids).reshape(-1)
    if ids.size != n or (n and not np.issubdtype(ids.dtype, np.integer)):
        raise ValueError(f"target_ids must be an integer array [{n}]")
    if ((ids != -1) & ((ids < 1) | (ids > 255))).any():
        raise ValueError("target_ids must lie in 1..255, or be -1 for an entry that is not scored")
    for g in range(off.size - 1):
        v = ids[off[g]:off[g + 1]]
        v = v[v != -1]
        if np.unique(v).size != v.size:
            raise ValueError(f"video {g}: target_ids must be unique within a video")
    G, H, W = off.size - 1, int(size[0]), int(size[1])
    if not (torch.is_tensor(anno) and anno.is_cuda and anno.dtype == torch.uint8 and tuple(anno.shape) == (G, H, W)):
        raise ValueError(f"anno must be a uint8 CUDA tensor [{G},{H},{W}]")
    dev = anno.device
    return _paste_labels_iou(masks, maps, anno, obj_offsets, objects,
                             torch.as_tensor(ids.astype(np.int32), device=dev), size, seg_thr,
                             torch.as_tensor(t, device=dev))


def _paste_labels_iou(masks, maps, anno, obj_offsets, objects, target_ids, size, seg_thr: float, thrs, counts=None,
                      ragged=None):
    """`paste_labels_iou` without the host-side checks (callers that validated their tables once): anno uint8, target_ids
    int32 and thrs float64 are CUDA tensors.  counts (optional): a contiguous int32 CUDA tensor [n,T,2] to write into.
    ragged = (desc, total) as in `_paste_labels` (`sm_paste_labels_iou_ragged`): anno and the returned labels are packed
    uint8 [total], size = (max_h, max_w)."""
    off = torch.as_tensor(obj_offsets, dtype=torch.int32).reshape(-1)
    G = off.numel() - 1
    H, W = int(size[0]), int(size[1])
    dev = anno.device
    anno = anno.contiguous()
    lib = _lib.load()
    off = off.to(dev).contiguous()
    obj = torch.as_tensor(objects, dtype=torch.int32).reshape(-1, 2)
    n, T = int(obj.shape[0]), int(thrs.numel())
    obj = (obj if obj.numel() else torch.zeros(1, 2, dtype=torch.int32)).to(dev).contiguous()
    tid = target_ids if n else torch.full((1,), -1, dtype=torch.int32, device=dev)
    side = 1
    if masks is not None:
        masks = masks.to(dev, torch.float32).contiguous()
        side = int(masks.shape[-1])
        maps = torch.as_tensor(maps, dtype=torch.float64).reshape(-1, 6).to(dev).contiguous()
    if counts is None:
        counts = torch.empty(n, T, 2, dtype=torch.int32, device=dev)
    cnt = counts if n else torch.empty(1, T, 2, dtype=torch.int32, device=dev)
    labels = torch.empty((G, H, W) if ragged is None else (int(ragged[1]),), dtype=torch.uint8, device=dev)
    mp = masks.data_ptr() if masks is not None else None
    mpp = maps.data_ptr() if masks is not None else None
    with torch.cuda.device(dev):
        if ragged is None:
            _lib.check(lib.sm_paste_labels_iou(mp, side, mpp, anno.data_ptr(), off.data_ptr(), obj.data_ptr(),
                                               tid.contiguous().data_ptr(), G, H, W, float(seg_thr), labels.data_ptr(),
                                               thrs.contiguous().data_ptr(), T, cnt.data_ptr(), _stream(dev)))
        else:
            _lib.check(lib.sm_paste_labels_iou_ragged(mp, side, mpp, anno.data_ptr(), off.data_ptr(), obj.data_ptr(),
                                                      tid.contiguous().data_ptr(), ragged[0].data_ptr(), G, H, W,
                                                      float(seg_thr), labels.data_ptr(), thrs.contiguous().data_ptr(),
                                                      T, cnt.data_ptr(), _stream(dev)))
    return labels, counts


def label_boxes(anno: torch.Tensor, queries) -> torch.Tensor:
    """cv2.boundingRect(anno[g] == id) for every query (g, id) on the device (init boxes of track_vos,
    tools/test.py:483-496, C ABI `sm_label_boxes`).  anno uint8 CUDA [G,H,W]; queries int [Q,2].  Returns int32 [Q,4]
    x, y, w, h ((0, 0, 0, 0) where no pixel carries the id)."""
    if not anno.is_cuda or anno.dtype != torch.uint8 or anno.dim() != 3:
        raise RuntimeError("label_boxes expects a uint8 CUDA tensor [G,H,W]; there is no CPU path")
    lib = _lib.load()
    dev = anno.device
    anno = anno.contiguous()
    q = torch.as_tensor(queries, dtype=torch.int32).reshape(-1, 2).to(dev).contiguous()
    out = torch.zeros(q.shape[0], 4, dtype=torch.int32, device=dev)
    if q.shape[0] == 0:
        return out
    G, H, W = anno.shape
    with torch.cuda.device(dev):
        _lib.check(lib.sm_label_boxes(anno.data_ptr(), G, H, W, q.data_ptr(), q.shape[0], out.data_ptr(), _stream(dev)))
    return out


def _label_boxes_ragged(anno: torch.Tensor, desc: torch.Tensor, G: int, queries) -> torch.Tensor:
    """`label_boxes` for G videos of different sizes (C ABI `sm_label_boxes_ragged`): anno the packed uint8 CUDA buffer
    and desc its device sm_image_desc table; queries int [Q,2] (g, id).  No host-side checks."""
    lib = _lib.load()
    dev = anno.device
    q = torch.as_tensor(queries, dtype=torch.int32).reshape(-1, 2).to(dev).contiguous()
    out = torch.zeros(q.shape[0], 4, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_label_boxes_ragged(anno.contiguous().data_ptr(), desc.data_ptr(), int(G), q.data_ptr(),
                                             q.shape[0], out.data_ptr(), _stream(dev)))
    return out


def _crop_resize_ragged(frames: torch.Tensor, desc: torch.Tensor, frame_idx: torch.Tensor, boxes: torch.Tensor,
                        model_size: int) -> torch.Tensor:
    """`crop_resize` over a packed uint8 CUDA frame buffer (C ABI `sm_crop_resize_ragged`): stream b crops frame
    desc[frame_idx[b]]; frame_idx int32 CUDA [B]; boxes int32 CUDA [B,8] whose first 6 columns are `crop_resize`'s
    boxes.  No host-side checks and no host staging."""
    lib = _lib.load()
    dev = frames.device
    B = int(boxes.shape[0])
    out = torch.empty(B, 3, model_size, model_size, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_crop_resize_ragged(frames.contiguous().data_ptr(), desc.data_ptr(),
                                             frame_idx.contiguous().data_ptr(), boxes.contiguous().data_ptr(), B,
                                             model_size, out.data_ptr(), _stream(dev)))
    return out


def _warp_affine_ragged(src: torch.Tensor, maps, desc: torch.Tensor, max_hw, total: int,
                        border_value: float = -1.0) -> torch.Tensor:
    """`warp_affine` of B square masks src f32 CUDA [B,side,side] into destinations of different sizes (C ABI
    `sm_warp_affine_ragged`): desc the device sm_image_desc table of the B destinations in a packed f32 buffer of
    `total` elements, max_hw = (max_h, max_w).  Returns that buffer (elements outside every image are left as they
    were allocated).  No host-side checks."""
    lib = _lib.load()
    dev = src.device
    s3 = src.to(torch.float32).contiguous()
    m = torch.as_tensor(maps, dtype=torch.float64).reshape(-1, 6).to(dev).contiguous()
    out = torch.empty(int(total), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_warp_affine_ragged(s3.data_ptr(), int(s3.shape[-1]), m.data_ptr(), out.data_ptr(),
                                             desc.data_ptr(), int(s3.shape[0]), int(max_hw[0]), int(max_hw[1]),
                                             float(border_value), _stream(dev)))
    return out


def mask_iou(masks, maps, anno, video, thrs) -> torch.Tensor:
    """Fused paste-back + IoU counts of the reference's IouMeter.add (utils/average_meter_helper.py:71-113), as
    tools/tune_vos.py scores each frame (C ABI `sm_mask_iou`).  masks f32 CUDA [B,side,side] (sigmoid masks) and maps
    f64 [B,6] (forward paste-back maps) of B streams; anno uint8 CUDA [G,H,W] annotations; video int [B]: the video in
    [0, G) stream b is scored against; thrs: 1..32 thresholds >= -1.  Returns int32 [B,T,2] = (intersection, union) of
    pred = v > thrs[t] (compared in float64) and target = anno > 0, where v is the cv2.warpAffine(INTER_LINEAR,
    BORDER_CONSTANT, -1) value of the mask, bit for bit with `warp_affine`.  The checks read `video` and `thrs` on the
    host (one D2H copy each if they live on the device)."""
    if not (torch.is_tensor(masks) and masks.is_cuda and masks.dtype == torch.float32 and masks.dim() == 3
            and masks.shape[1] == masks.shape[2]):
        raise ValueError("masks must be a float32 CUDA tensor [B, side, side]")
    if not (torch.is_tensor(anno) and anno.is_cuda and anno.dtype == torch.uint8 and anno.dim() == 3):
        raise ValueError("anno must be a uint8 CUDA tensor [G, H, W]")
    B, G = int(masks.shape[0]), int(anno.shape[0])
    m = torch.as_tensor(maps)
    if m.dtype != torch.float64 or tuple(m.shape) != (B, 6):
        raise ValueError(f"maps must be float64 [{B}, 6]")
    v = np.asarray(video.cpu() if torch.is_tensor(video) else video)
    if v.shape != (B,) or not np.issubdtype(v.dtype, np.integer):
        raise ValueError(f"video must be an integer array [{B}]")
    if B and ((v < 0) | (v >= G)).any():
        raise ValueError(f"video entries must lie in [0, {G})")
    t = np.asarray(thrs.cpu() if torch.is_tensor(thrs) else thrs, dtype=np.float64).reshape(-1)
    if not 1 <= t.size <= 32:
        raise ValueError("1 to 32 thresholds expected")
    if not (t >= -1.0).all():
        raise ValueError("thresholds must be >= -1 (pixels the mask misses have the value -1)")
    if B == 0:
        return torch.zeros(0, t.size, 2, dtype=torch.int32, device=masks.device)
    dev = masks.device
    return _mask_iou(masks, m.to(dev), anno, torch.as_tensor(v.astype(np.int32), device=dev),
                     torch.as_tensor(t, device=dev))


def _mask_iou(masks, maps, anno, video, thrs) -> torch.Tensor:
    """`mask_iou` without the host-side checks (callers that validated `video` and `thrs` once); every argument is a
    CUDA tensor of the documented dtype."""
    lib = _lib.load()
    dev = masks.device
    masks, maps, anno, video, thrs = (t.contiguous() for t in (masks, maps, anno, video, thrs))
    B, side = int(masks.shape[0]), int(masks.shape[-1])
    _, H, W = anno.shape
    T = int(thrs.numel())
    out = torch.empty(B, T, 2, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_mask_iou(masks.data_ptr(), side, maps.data_ptr(), anno.data_ptr(), video.data_ptr(), B, H, W,
                                   thrs.data_ptr(), T, out.data_ptr(), _stream(dev)))
    return out


def mask_iou_ragged(masks, maps, anno, table, video, thrs) -> torch.Tensor:
    """`mask_iou` against annotations of different sizes (C ABI `sm_mask_iou_ragged`): anno a flat uint8 CUDA buffer
    holding the annotation images back to back, table their host sm_image_desc rows (`tracker.IMAGE_DESC`: offset, h,
    w per image), video int [B]: the image stream b is scored against.  Each stream's counts equal `mask_iou` on its
    image alone.  The checks read `table`, `video` and `thrs` on the host: every image inside the buffer, every image
    a stream reads at least 1 x 1."""
    from .tracker import IMAGE_DESC
    if not (torch.is_tensor(masks) and masks.is_cuda and masks.dtype == torch.float32 and masks.dim() == 3
            and masks.shape[1] == masks.shape[2]):
        raise ValueError("masks must be a float32 CUDA tensor [B, side, side]")
    if not (torch.is_tensor(anno) and anno.is_cuda and anno.dtype == torch.uint8 and anno.dim() == 1):
        raise ValueError("anno must be a flat uint8 CUDA tensor (the packed annotation images)")
    B = int(masks.shape[0])
    m = torch.as_tensor(maps)
    if m.dtype != torch.float64 or tuple(m.shape) != (B, 6):
        raise ValueError(f"maps must be float64 [{B}, 6]")
    tb = np.asarray(table)
    if tb.dtype != IMAGE_DESC or tb.ndim != 1 or tb.size == 0:
        raise ValueError("table must be a non-empty 1-D array of sm_image_desc rows (tracker.IMAGE_DESC)")
    off, h, w = tb["offset"].astype(np.int64), tb["h"].astype(np.int64), tb["w"].astype(np.int64)
    if (off < 0).any() or (h < 0).any() or (w < 0).any() or (off + h * w > anno.numel()).any():
        raise ValueError(f"every image must lie inside the {anno.numel()}-byte buffer with h, w >= 0")
    if (h * w > 2 ** 31 - 1).any():
        raise ValueError("image too large for int32 counts")
    v = np.asarray(video.cpu() if torch.is_tensor(video) else video)
    if v.shape != (B,) or not np.issubdtype(v.dtype, np.integer):
        raise ValueError(f"video must be an integer array [{B}]")
    if B and ((v < 0) | (v >= tb.size)).any():
        raise ValueError(f"video entries must lie in [0, {tb.size})")
    if B and ((h[v] < 1) | (w[v] < 1)).any():
        raise ValueError("a stream reads an empty image")
    t = np.asarray(thrs.cpu() if torch.is_tensor(thrs) else thrs, dtype=np.float64).reshape(-1)
    if not 1 <= t.size <= 32:
        raise ValueError("1 to 32 thresholds expected")
    if not (t >= -1.0).all():
        raise ValueError("thresholds must be >= -1 (pixels the mask misses have the value -1)")
    dev = masks.device
    if B == 0:
        return torch.zeros(0, t.size, 2, dtype=torch.int32, device=dev)
    desc = torch.from_numpy(tb.view(np.uint8).copy()).to(dev)
    return _mask_iou_ragged(masks, m.to(dev), anno, desc, torch.as_tensor(v.astype(np.int32), device=dev),
                            (int(h.max()), int(w.max())), torch.as_tensor(t, device=dev))


def _mask_iou_ragged(masks, maps, anno, desc, video, max_hw, thrs) -> torch.Tensor:
    """`mask_iou_ragged` without the host-side checks: anno the packed uint8 CUDA buffer, desc its device sm_image_desc
    table, video int32 CUDA [B], max_hw = (max_h, max_w) bounding every image a stream reads, thrs float64 CUDA."""
    lib = _lib.load()
    dev = masks.device
    masks, maps, video, thrs = (t.contiguous() for t in (masks, maps, video, thrs))
    B, side = int(masks.shape[0]), int(masks.shape[-1])
    T = int(thrs.numel())
    out = torch.empty(B, T, 2, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_mask_iou_ragged(masks.data_ptr(), side, maps.data_ptr(), anno.contiguous().data_ptr(),
                                          desc.data_ptr(), video.data_ptr(), B, int(max_hw[0]), int(max_hw[1]),
                                          thrs.data_ptr(), T, out.data_ptr(), _stream(dev)))
    return out


VOT_COORD_LIMIT = 2.0 ** 20       # |coordinate| bound of sm_vot_overlap's precondition


def vot_overlap(poly_a, poly_b, size) -> torch.Tensor:
    """Region overlap of the VOT supervised protocol (tools/test.py:341-354, C ABI `sm_vot_overlap`): pyvotkit's
    vot_overlap(poly_a[b], poly_b[b], (W, H)) for B pairs, bit for bit.  poly_a, poly_b: float32 CUDA [B,8] 4-point
    polygons x0, y0, .. x3, y3; size = (H, W), or an int array [B,2] of per-pair (H, W) (`sm_vot_overlap_sized`).
    Returns float32 [B]; NaN where both rasterised polygons are empty inside the frame (the protocol does not count that
    as a loss).  The checks read both polygon tensors on the host: shapes, dtype, device, and every coordinate finite and
    within +-2^20 px."""
    for name, p in (("poly_a", poly_a), ("poly_b", poly_b)):
        if not (torch.is_tensor(p) and p.is_cuda and p.dtype == torch.float32 and p.dim() == 2 and p.shape[1] == 8):
            raise ValueError(f"{name} must be a float32 CUDA tensor [B, 8]")
    if poly_a.shape != poly_b.shape or poly_a.device != poly_b.device:
        raise ValueError("poly_a and poly_b must have the same shape and device")
    sz = np.asarray(size.cpu() if torch.is_tensor(size) else size)
    per_pair = sz.ndim == 2
    if per_pair and (sz.shape != (poly_a.shape[0], 2) or not np.issubdtype(sz.dtype, np.integer)):
        raise ValueError(f"per-pair sizes must be an int array [{poly_a.shape[0]}, 2] of (H, W)")
    hw = sz.reshape(-1, 2).astype(np.int64) if per_pair else np.array([[int(size[0]), int(size[1])]], np.int64)
    H, W = hw[:, 0], hw[:, 1]
    if (H < 1).any() or (W < 1).any() or ((W + 1) * (H + 1) > 2 ** 31 - 1).any():
        raise ValueError("size must be (H, W) with H, W >= 1 and (W+1)*(H+1) < 2^31")
    for name, p in (("poly_a", poly_a), ("poly_b", poly_b)):
        v = p.cpu().numpy()
        if not (np.isfinite(v).all() and (np.abs(v) <= VOT_COORD_LIMIT).all()):
            raise ValueError(f"{name}: coordinates must be finite and within +-2^20 px")
    if poly_a.shape[0] == 0:
        return torch.empty(0, dtype=torch.float32, device=poly_a.device)
    if per_pair:
        wh = torch.as_tensor(np.stack([W, H], 1).astype(np.int32), device=poly_a.device)
        return _vot_overlap_sized(poly_a, poly_b, wh)
    return _vot_overlap(poly_a, poly_b, (int(H[0]), int(W[0])))


def _vot_overlap(poly_a, poly_b, size, out=None) -> torch.Tensor:
    """`vot_overlap` without the host-side checks: poly_a, poly_b float32 CUDA [B,8] with B >= 1 inside the
    precondition.  out (optional): a contiguous float32 CUDA tensor [B] to write into."""
    lib = _lib.load()
    dev = poly_a.device
    poly_a, poly_b = poly_a.contiguous(), poly_b.contiguous()
    B = int(poly_a.shape[0])
    if out is None:
        out = torch.empty(B, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_vot_overlap(poly_a.data_ptr(), poly_b.data_ptr(), B, int(size[1]), int(size[0]),
                                      out.data_ptr(), _stream(dev)))
    return out


def _vot_overlap_sized(poly_a, poly_b, wh, out=None) -> torch.Tensor:
    """`_vot_overlap` with per-pair bounds (C ABI `sm_vot_overlap_sized`): wh int32 CUDA [B,2] = (W, H) of each pair,
    inside the precondition.  No host-side checks."""
    lib = _lib.load()
    dev = poly_a.device
    poly_a, poly_b = poly_a.contiguous(), poly_b.contiguous()
    B = int(poly_a.shape[0])
    if out is None:
        out = torch.empty(B, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_vot_overlap_sized(poly_a.data_ptr(), poly_b.data_ptr(), B, wh.contiguous().data_ptr(),
                                            out.data_ptr(), _stream(dev)))
    return out


def _vot_trajectory_overlap(rec, T: int, S: int, gt, seq, wh, lengths, poly=None):
    """C ABI `sm_vot_trajectory_overlap` without host-side checks: rec float64 CUDA [>= T, S, 5] (a `VotRunner` record),
    gt float32 CUDA [G, >= T, 8], seq / lengths int32 CUDA [S], wh int32 CUDA [S, 2] = (W, H), all inside the
    precondition.  Returns (acc, eao) float32 [T, S]: pysot's per-frame overlaps with bounds (W, H) and burn-in 10, and
    with bounds (W-1, H-1).  With poly float64 CUDA [>= T, S, 8] (a mask-mode record's polygons), a location entry is
    that polygon (`sm_vot_trajectory_overlap_poly`) and rec supplies the entry codes only."""
    lib = _lib.load()
    dev = rec.device
    acc = torch.empty(T, S, dtype=torch.float32, device=dev)
    eao = torch.empty(T, S, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        if poly is None:
            _lib.check(lib.sm_vot_trajectory_overlap(rec.data_ptr(), T, S, gt.data_ptr(), int(gt.shape[1]),
                                                     seq.data_ptr(), wh.data_ptr(), lengths.data_ptr(), acc.data_ptr(),
                                                     eao.data_ptr(), _stream(dev)))
        else:
            _lib.check(lib.sm_vot_trajectory_overlap_poly(rec.data_ptr(), poly.data_ptr(), T, S, gt.data_ptr(),
                                                          int(gt.shape[1]), seq.data_ptr(), wh.data_ptr(),
                                                          lengths.data_ptr(), acc.data_ptr(), eao.data_ptr(),
                                                          _stream(dev)))
    return acc, eao


def _vot_eao_accumulate(eao, acc, rec, lengths, combo, tail_from, tail_in, tail_out, num, den, stats):
    """C ABI `sm_vot_eao_accumulate` without host-side checks: adds the streams of the planes eao / acc float32 CUDA
    [T, S] into the score rows combo[s] of num / den float64 [R, cap], tail_out float64 [R, 2] (from tail_in) and stats
    float64 [R, 4].  The workspace comes from torch's caching allocator."""
    lib = _lib.load()
    dev = eao.device
    T, S = int(eao.shape[0]), int(eao.shape[1])
    R, cap = int(num.shape[0]), int(num.shape[1])
    nbytes = int(lib.sm_vot_eao_workspace_size(T, S))
    ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sm_vot_eao_accumulate(eao.data_ptr(), acc.data_ptr(), rec.data_ptr(), T, S, lengths.data_ptr(),
                                             combo.data_ptr(), R, cap, int(tail_from), tail_in.data_ptr(),
                                             tail_out.data_ptr(), num.data_ptr(), den.data_ptr(), stats.data_ptr(),
                                             ws.data_ptr(), ws.numel() * 8, _stream(dev)))


RBOX_MAX_SIDE = 32767             # frame side bound of sm_rotated_box_ragged


def rotated_box(masks, fallback_cxcywh):
    """SiamMask's rotated box (tools/test.py:284-303, C ABI `sm_rotated_box_ragged`) for N thresholded masks: the
    minimum-area rectangle of the largest outer contour if its area is over 100, else the rectangle of the fallback
    state.  masks: a bool (or uint8, nonzero = foreground) CUDA tensor [N,H,W], or a list of N CUDA tensors [H_i,W_i]
    (as `BatchTracker.track(mask=True, paste=True)` returns them); fallback_cxcywh: float64 [N,4] = target_pos,
    target_sz before the clamps (host or device).  Returns (poly float64 [N,8] in cv2.boxPoints' vertex order, or the
    fallback's 4 corners; flag int32 [N], 1 contour / 0 fallback; area2 int64 [N], twice the largest contour area),
    all on the masks' device, without a host sync.  Contour areas, selection and fallback equal cv2's exactly; the
    rectangle is a deterministic float64 rule (include/siammask_b200.h) that may differ from cv2's minAreaRect where
    two orientations give nearly equal areas."""
    if torch.is_tensor(masks):
        if masks.dim() != 3:
            raise ValueError(f"masks must be [N,H,W] or a list of [H,W] tensors, got {tuple(masks.shape)}")
        masks = list(masks.unbind(0))
    if not isinstance(masks, (list, tuple)):
        raise ValueError("masks must be a CUDA tensor [N,H,W] or a list of CUDA tensors [H,W]")
    N = len(masks)
    for i, m in enumerate(masks):
        if not (torch.is_tensor(m) and m.is_cuda and m.dim() == 2 and m.dtype in (torch.bool, torch.uint8)):
            raise ValueError(f"masks[{i}] must be a bool or uint8 CUDA tensor [H,W]")
        if not 1 <= min(m.shape) or max(m.shape) > RBOX_MAX_SIDE:
            raise ValueError(f"masks[{i}]: sides must lie in [1, {RBOX_MAX_SIDE}], got {tuple(m.shape)}")
    if not 1 <= N <= 65535:
        raise ValueError(f"1 <= N <= 65535 masks expected, got {N}")
    dev = masks[0].device
    if any(m.device != dev for m in masks):
        raise ValueError("masks must all be on one device")
    fb = fallback_cxcywh if torch.is_tensor(fallback_cxcywh) else torch.as_tensor(np.asarray(fallback_cxcywh,
                                                                                                np.float64))
    if tuple(fb.shape) != (N, 4):
        raise ValueError(f"fallback_cxcywh must be [{N}, 4] (cx, cy, w, h), got {tuple(fb.shape)}")
    from .tracker import FramePacker
    packed = FramePacker(dev).pack([m.to(torch.uint8) if m.dtype != torch.uint8 else m for m in masks], 1)
    hs, ws = zip(*packed.shapes)
    return _rotated_box(packed.data, packed.desc, N, (max(hs), max(ws)), fb.to(dev, torch.float64))


def _rotated_box(data, desc, N: int, max_hw, fallback):
    """`rotated_box` without host-side checks: data the packed mask buffer (bool or uint8, CUDA), desc its device
    sm_image_desc table of N masks, max_hw bounds of their sides, fallback float64 CUDA [N,4].  The workspace comes
    from torch's caching allocator."""
    lib = _lib.load()
    dev = data.device
    total = int(data.numel())
    nbytes = int(lib.sm_rotated_box_workspace_size(total, N, int(max_hw[0])))
    ws = torch.empty((nbytes + 15) // 16 * 2, dtype=torch.float64, device=dev)
    poly = torch.empty(N, 8, dtype=torch.float64, device=dev)
    flag = torch.empty(N, dtype=torch.int32, device=dev)
    area2 = torch.empty(N, dtype=torch.int64, device=dev)
    fallback = fallback.contiguous()
    with torch.cuda.device(dev):
        _lib.check(lib.sm_rotated_box_ragged(data.data_ptr(), desc.data_ptr(), N, int(max_hw[0]), int(max_hw[1]), total,
                                             fallback.data_ptr(), ws.data_ptr(), ws.numel() * 8, poly.data_ptr(),
                                             flag.data_ptr(), area2.data_ptr(), _stream(dev)))
    return poly, flag, area2
