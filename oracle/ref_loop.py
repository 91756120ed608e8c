"""TEST INFRASTRUCTURE ONLY (checker).  Nothing under `siammask_b200/` imports this module.

Host restatement of the reference tracker loop, kept next to the other oracles because its integer / float64
arithmetic has to match the reference statement for statement: it pins the product's batched device tracker
(`siammask_b200/tracker.py`, kernels `tracker_prepare_kernel` / `tracker_update_kernel`) and the device crop / select /
paste-back operators to the golden trajectory that the reference's OWN `siamese_init` / `siamese_track` produced
(`oracle/make_golden.py::tracker_loop_golden`).

A restatement of
`generate_anchor`, `siamese_init` and `siamese_track` (tools/test.py:113-315) that drives a `net` exposing the
reference's model API.  With a siammask_b200 engine the score/box post-processing + argmax between `track_mask`
and `track_refine` (tools/test.py:205-254) runs on the device (`Custom.select`, C ABI `sm_select`), so the only
host round trip per frame is 8 floats per stream; with any other `net` (e.g. the CPU oracle in the tests) the same
arithmetic runs in numpy as in the reference.  Frames may be numpy arrays (crop + cv2.resize on the host, as in the
reference, :67-110) or uint8 CUDA tensors (the crop + a bit-exact restatement of cv2's 8-bit INTER_LINEAR resize run on
the device, `ops.crop_resize` / C ABI `sm_crop_resize`).  Mask paste-back (crop_back :263-282) runs with cv2 on the
host as in the reference, or on the device (`device_paste=True`, `ops.warp_affine` / `sm_warp_affine`); contour
extraction and minAreaRect (:285-303) stay on the host.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

try:  # cv2 is only needed for the image-facing half of the loop
    import cv2
except Exception:  # pragma: no cover
    cv2 = None


class TrackerConfig:
    """utils/tracker_config.py:10-47 (defaults of SiamMask) + experiments/siammask_sharp/config_davis.json hp."""
    penalty_k = 0.09
    window_influence = 0.39
    lr = 0.38
    seg_thr = 0.3
    windowing = "cosine"
    exemplar_size = 127
    instance_size = 255
    total_stride = 8
    out_size = 63
    base_size = 8
    context_amount = 0.5
    ratios = [0.33, 0.5, 1, 2, 3]
    scales = [8]
    round_dight = 0

    def update(self, newparam=None, anchors=None):
        for k, v in (newparam or {}).items():
            setattr(self, k, v)
        if anchors is not None:
            self.total_stride = anchors.get("stride", self.total_stride)
            self.ratios = anchors.get("ratios", self.ratios)
            self.scales = anchors.get("scales", self.scales)
            self.round_dight = anchors.get("round_dight", self.round_dight)
        self.renew()

    def renew(self):
        self.score_size = (self.instance_size - self.exemplar_size) // self.total_stride + 1 + self.base_size
        self.anchor_num = len(self.ratios) * len(self.scales)


def base_anchors(cfg: dict) -> np.ndarray:
    """Anchors.generate_anchors, utils/anchors.py:26-48 (anchor_density 1): (A,4) x1,y1,x2,y2 float32."""
    stride, ratios, scales = cfg.get("stride", 8), cfg["ratios"], cfg["scales"]
    rd = cfg.get("round_dight", 0)
    out = np.zeros((len(ratios) * len(scales), 4), dtype=np.float32)
    size = stride * stride
    i = 0
    for r in ratios:
        if rd > 0:
            ws = round(math.sqrt(size * 1.0 / r), rd)
            hs = round(ws * r, rd)
        else:
            ws = int(math.sqrt(size * 1.0 / r))
            hs = int(ws * r)
        for s in scales:
            w, h = ws * s, hs * s
            out[i] = [-w * 0.5, -h * 0.5, w * 0.5, h * 0.5]
            i += 1
    return out


def generate_anchor(cfg: dict, score_size: int) -> np.ndarray:
    """tools/test.py:113-129 -> (A*S*S, 4) cx,cy,w,h float32, ordered (anchor, y, x)."""
    a = base_anchors(cfg)
    x1, y1, x2, y2 = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    anchor = np.stack([(x1 + x2) * 0.5, (y1 + y2) * 0.5, x2 - x1, y2 - y1], 1)
    stride = cfg.get("stride", 8)
    n = anchor.shape[0]
    anchor = np.tile(anchor, score_size * score_size).reshape((-1, 4))
    ori = -(score_size // 2) * stride
    xx, yy = np.meshgrid([ori + stride * dx for dx in range(score_size)],
                         [ori + stride * dy for dy in range(score_size)])
    xx, yy = np.tile(xx.flatten(), (n, 1)).flatten(), np.tile(yy.flatten(), (n, 1)).flatten()
    anchor[:, 0], anchor[:, 1] = xx.astype(np.float32), yy.astype(np.float32)
    return anchor


def subwindow_box(pos, original_sz, avg_chans):
    """The integers get_subwindow_tracking derives before touching pixels (tools/test.py:71-76,89-100):
    (context_xmin, context_ymin, original_sz, uint8(avg_chans))."""
    c = (original_sz + 1) / 2
    a = np.asarray(avg_chans, dtype=np.float64).astype(np.uint8)      # numpy assignment into a uint8 image truncates
    return [int(round(pos[0] - c)), int(round(pos[1] - c)), int(original_sz), int(a[0]), int(a[1]), int(a[2])]


def get_subwindow_tracking(im, pos, model_sz, original_sz, avg_chans):
    """tools/test.py:67-110: crop a square window around pos (padding with the frame's mean colour), resize to
    model_sz with cv2.resize, return a float CHW tensor of raw 0..255 pixels."""
    if isinstance(im, torch.Tensor):         # frame already on the GPU: crop + cv2-exact resize on the device
        from siammask_b200.ops import crop_resize
        return crop_resize(im, [subwindow_box(pos, original_sz, avg_chans)], int(model_sz))[0]
    sz = original_sz
    im_sz = im.shape
    c = (original_sz + 1) / 2
    context_xmin = round(pos[0] - c)
    context_xmax = context_xmin + sz - 1
    context_ymin = round(pos[1] - c)
    context_ymax = context_ymin + sz - 1
    left_pad = int(max(0.0, -context_xmin))
    top_pad = int(max(0.0, -context_ymin))
    right_pad = int(max(0.0, context_xmax - im_sz[1] + 1))
    bottom_pad = int(max(0.0, context_ymax - im_sz[0] + 1))
    context_xmin += left_pad
    context_xmax += left_pad
    context_ymin += top_pad
    context_ymax += top_pad
    r, cc, k = im.shape
    if any([top_pad, bottom_pad, left_pad, right_pad]):
        te = np.zeros((r + top_pad + bottom_pad, cc + left_pad + right_pad, k), np.uint8)
        te[top_pad:top_pad + r, left_pad:left_pad + cc, :] = im
        if top_pad:
            te[0:top_pad, left_pad:left_pad + cc, :] = avg_chans
        if bottom_pad:
            te[r + top_pad:, left_pad:left_pad + cc, :] = avg_chans
        if left_pad:
            te[:, 0:left_pad, :] = avg_chans
        if right_pad:
            te[:, cc + left_pad:, :] = avg_chans
        patch = te[int(context_ymin):int(context_ymax + 1), int(context_xmin):int(context_xmax + 1), :]
    else:
        patch = im[int(context_ymin):int(context_ymax + 1), int(context_xmin):int(context_xmax + 1), :]
    if model_sz != original_sz:
        patch = cv2.resize(patch, (model_sz, model_sz))
    return torch.from_numpy(np.ascontiguousarray(np.transpose(patch, (2, 0, 1)))).float()


def select_numpy(score_t: torch.Tensor, delta_t: torch.Tensor, anchor: np.ndarray, window: np.ndarray,
                 target_sz_in_crop: np.ndarray, penalty_k: float, window_influence: float):
    """tools/test.py:205-237 for ONE stream, in numpy exactly as the reference does it.
    Returns (best_id, decoded box (4,) in crop units, score, penalty, pscore)."""
    delta = delta_t.permute(1, 2, 3, 0).contiguous().view(4, -1).data.cpu().numpy()
    score = F.softmax(score_t.permute(1, 2, 3, 0).contiguous().view(2, -1).permute(1, 0), dim=1).data[:, 1].cpu().numpy()
    delta[0, :] = delta[0, :] * anchor[:, 2] + anchor[:, 0]
    delta[1, :] = delta[1, :] * anchor[:, 3] + anchor[:, 1]
    delta[2, :] = np.exp(delta[2, :]) * anchor[:, 2]
    delta[3, :] = np.exp(delta[3, :]) * anchor[:, 3]

    def change(r):
        return np.maximum(r, 1.0 / r)

    def sz(w, h):
        pad = (w + h) * 0.5
        return np.sqrt((w + pad) * (h + pad))

    s_c = change(sz(delta[2, :], delta[3, :]) / sz(target_sz_in_crop[0], target_sz_in_crop[1]))
    r_c = change((target_sz_in_crop[0] / target_sz_in_crop[1]) / (delta[2, :] / delta[3, :]))
    penalty = np.exp(-(r_c * s_c - 1) * penalty_k)
    pscore = penalty * score
    pscore = pscore * (1 - window_influence) + window * window_influence
    best = int(np.argmax(pscore))
    return best, delta[:, best].copy(), float(score[best]), float(penalty[best]), float(pscore[best])


def siamese_init(im, target_pos, target_sz, model, hp=None, device="cuda"):
    """tools/test.py:132-169."""
    state = {"im_h": im.shape[0], "im_w": im.shape[1]}
    p = TrackerConfig()
    p.update(hp, model.anchors)
    p.renew()
    p.scales = model.anchors["scales"]
    p.ratios = model.anchors["ratios"]
    p.anchor_num = model.anchor_num
    p.anchor = generate_anchor(model.anchors, p.score_size)
    avg_chans = im.double().mean(dim=(0, 1)).cpu().numpy() if isinstance(im, torch.Tensor) else np.mean(im, axis=(0, 1))
    wc_z = target_sz[0] + p.context_amount * sum(target_sz)
    hc_z = target_sz[1] + p.context_amount * sum(target_sz)
    s_z = round(np.sqrt(wc_z * hc_z))
    z_crop = get_subwindow_tracking(im, target_pos, p.exemplar_size, s_z, avg_chans)
    model.template(z_crop.unsqueeze(0).to(device))
    if p.windowing == "cosine":
        window = np.outer(np.hanning(p.score_size), np.hanning(p.score_size))
    else:
        window = np.ones((p.score_size, p.score_size))
    window = np.tile(window.flatten(), p.anchor_num)
    state.update(p=p, net=model, avg_chans=avg_chans, window=window,
                 target_pos=np.asarray(target_pos, dtype=np.float64), target_sz=np.asarray(target_sz, dtype=np.float64))
    if hasattr(model, "select"):      # device copies for the on-device post-processing
        state["anchor_dev"] = torch.from_numpy(p.anchor).to(device)
        state["window_dev"] = torch.from_numpy(window).to(device)
    return state


def siamese_track(state, im, mask_enable=False, refine_enable=False, device="cuda", device_paste=False):
    """tools/test.py:172-315.  device_paste=True keeps the 127x127 mask on the GPU and pastes it back into the frame
    with `ops.warp_affine` (bit-exact restatement of the cv2.warpAffine in crop_back); only the thresholded uint8 mask
    travels to the host for the contour / minAreaRect step."""
    p, net = state["p"], state["net"]
    avg_chans, window = state["avg_chans"], state["window"]
    target_pos, target_sz = state["target_pos"], state["target_sz"]
    wc_x = target_sz[1] + p.context_amount * sum(target_sz)
    hc_x = target_sz[0] + p.context_amount * sum(target_sz)
    s_x = np.sqrt(wc_x * hc_x)
    scale_x = p.exemplar_size / s_x
    d_search = (p.instance_size - p.exemplar_size) / 2
    pad = d_search / scale_x
    s_x = s_x + 2 * pad
    crop_box = [target_pos[0] - round(s_x) / 2, target_pos[1] - round(s_x) / 2, round(s_x), round(s_x)]
    x_crop = get_subwindow_tracking(im, target_pos, p.instance_size, round(s_x), avg_chans).unsqueeze(0).to(device)
    mask = None
    if mask_enable:
        if hasattr(net, "select") and refine_enable:
            score, delta, mask = net.track_mask(x_crop, mask_head=False)   # 3969-channel head is dead under --refine
        else:
            score, delta, mask = net.track_mask(x_crop)
    else:
        score, delta = net.track(x_crop)
    tsz_crop = target_sz * scale_x
    pos_dev = None
    if hasattr(net, "select"):
        best_t, pos_dev, rec = net.select(score, delta, state["anchor_dev"], state["window_dev"],
                                          torch.tensor(tsz_crop[None], dtype=torch.float64), p.penalty_k,
                                          p.window_influence)
        rec = rec[0].cpu().numpy()        # the one host round trip of the frame (8 floats; rec[7] = best index)
        best_id, box, best_score, best_pen = int(rec[7]), rec[:4].astype(np.float64), float(rec[4]), float(rec[5])
    else:
        best_id, box, best_score, best_pen, _ = select_numpy(score, delta, p.anchor, window, tsz_crop, p.penalty_k,
                                                             p.window_influence)
    pred_in_crop = box / scale_x
    lr = best_pen * best_score * p.lr
    res_x = pred_in_crop[0] + target_pos[0]
    res_y = pred_in_crop[1] + target_pos[1]
    res_w = target_sz[0] * (1 - lr) + pred_in_crop[2] * lr
    res_h = target_sz[1] * (1 - lr) + pred_in_crop[3] * lr
    target_pos = np.array([res_x, res_y])
    target_sz = np.array([res_w, res_h])
    mask_in_img, rbox = [], []
    if mask_enable:
        _, delta_y, delta_x = np.unravel_index(best_id, (p.anchor_num, p.score_size, p.score_size))
        if refine_enable:
            m = net.track_refine(pos_dev if pos_dev is not None else (delta_y, delta_x))
            m = m.sigmoid().squeeze().view(p.out_size, p.out_size)
        else:
            m = mask[0, :, delta_y, delta_x].sigmoid().squeeze().view(p.out_size, p.out_size)
        on_dev = device_paste and m.is_cuda
        if not on_dev:
            m = m.cpu().data.numpy()

        def crop_back(image, bbox, out_sz, padding=-1):          # tools/test.py:263-275
            a = (out_sz[0] - 1) / bbox[2]
            b = (out_sz[1] - 1) / bbox[3]
            mapping = np.array([[a, 0, -a * bbox[0]], [0, b, -b * bbox[1]]]).astype(float)
            if on_dev:
                from siammask_b200.ops import warp_affine
                return warp_affine(image, mapping, (out_sz[0], out_sz[1]), padding)
            return cv2.warpAffine(image, mapping, (out_sz[0], out_sz[1]), flags=cv2.INTER_LINEAR,
                                  borderMode=cv2.BORDER_CONSTANT, borderValue=padding)

        s = crop_box[2] / p.instance_size
        sub_box = [crop_box[0] + (delta_x - p.base_size / 2) * p.total_stride * s,
                   crop_box[1] + (delta_y - p.base_size / 2) * p.total_stride * s,
                   s * p.exemplar_size, s * p.exemplar_size]
        s = p.out_size / sub_box[2]
        back_box = [-sub_box[0] * s, -sub_box[1] * s, state["im_w"] * s, state["im_h"] * s]
        mask_in_img = crop_back(m, back_box, (state["im_w"], state["im_h"]))
        if on_dev:
            target_mask = (mask_in_img > p.seg_thr).to(torch.uint8).cpu().numpy()
        else:
            target_mask = (mask_in_img > p.seg_thr).astype(np.uint8)
        contours = cv2.findContours(target_mask, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_NONE)[-2]
        cnt_area = [cv2.contourArea(cnt) for cnt in contours]
        if len(contours) != 0 and np.max(cnt_area) > 100:
            polygon = contours[int(np.argmax(cnt_area))].reshape(-1, 2)
            rbox = cv2.boxPoints(cv2.minAreaRect(polygon))
        else:
            x0, y0 = target_pos[0] - target_sz[0] / 2, target_pos[1] - target_sz[1] / 2
            rbox = np.array([[x0, y0], [x0 + target_sz[0], y0], [x0 + target_sz[0], y0 + target_sz[1]],
                             [x0, y0 + target_sz[1]]])
    target_pos[0] = max(0, min(state["im_w"], target_pos[0]))
    target_pos[1] = max(0, min(state["im_h"], target_pos[1]))
    target_sz[0] = max(10, min(state["im_w"], target_sz[0]))
    target_sz[1] = max(10, min(state["im_h"], target_sz[1]))
    state.update(target_pos=target_pos, target_sz=target_sz, score=best_score, mask=mask_in_img, ploygon=rbox,
                 best_id=best_id)
    return state
