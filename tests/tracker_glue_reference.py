"""Host restatement of the tracker's per-frame glue around the network, in the reference's numpy order of operations
(tools/test.py:180-198, 205-249, 263-282), batched over streams: the selection (softmax score -> decode -> scale /
ratio penalty -> pscore with the float64 cosine window -> np.argmax), the search-window arithmetic of the next frame
and the lr-smoothed state update with crop_back's forward map.  `tests/test_gpu_tracker_glue.py` holds the device
kernels to it bit for bit; `tests/test_tracker_glue_host.py` pins it to `oracle/ref_loop.py` and shows that its
assertions reject the arithmetic variants a kernel could silently fall into (keyword switches below).

It also builds the constructed inputs both files use: pairs of score-map positions whose float64 window values differ
but round to the same float32, and select inputs where only chosen candidates can win."""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from oracle import ref_loop


def fma(a: float, b: float, c: float) -> float:
    """a * b + c rounded once (float64), exactly: Python 3.12 has no math.fma."""
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return float(a) * float(b) + float(c)
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def window(R: int, A: int, dtype=np.float64) -> np.ndarray:
    """tools/test.py:157-161: the tiled outer product of two Hanning windows (float64 in the reference)."""
    w = np.tile(np.outer(np.hanning(R), np.hanning(R)).flatten(), A)
    return w.astype(dtype).astype(np.float64)


def window_tie_pairs(R: int):
    """Score-map positions (p, q), p < q, whose float64 window values differ while their float32 roundings are equal:
    with the same cls / loc, numpy ranks the two candidates and a float32 window makes them an exact tie."""
    w = np.outer(np.hanning(R), np.hanning(R)).flatten()
    f = w.astype(np.float32)
    pairs = []
    for v in np.unique(f):
        pos = np.flatnonzero(f == v)
        for i in range(len(pos)):
            for j in range(i + 1, len(pos)):
                if w[pos[i]] != w[pos[j]]:
                    pairs.append((int(pos[i]), int(pos[j])))
    return pairs


def expf_cr(x: np.ndarray) -> np.ndarray:
    """Correctly rounded float32 exp (a mutation: numpy's float32 np.exp is not correctly rounded)."""
    with np.errstate(over="ignore", under="ignore"):
        return np.exp(np.asarray(x, np.float32).astype(np.float64)).astype(np.float32)


def select(score, loc, anchor, win, tsz, pk, wi, *, window32=False, fused=None, exp32=None):
    """tools/test.py:205-237 for B streams at once.  score f32 [B,n] = softmax(cls)[:, 1] in (anchor, y, x) order (the
    reference runs F.softmax on the device, :206-207); loc f32 [B,4,n]; anchor f32 [n,4]; win f64 [n]; tsz f64 [B,2];
    pk, wi: scalars or f64 [B].  Returns (best int [B], box f32 [B,4,n], penalty f64 [B,n], pscore f64 [B,n]).
    Mutations: window32 rounds the window to float32; fused = "window" or "score" evaluates pscore with one fused
    multiply-add (window * wi + P, or P * (1 - wi) + window * wi), exactly; exp32 replaces numpy's float32 exp."""
    B = score.shape[0]
    ex = exp32 if exp32 is not None else np.exp
    pk = np.broadcast_to(np.asarray(pk, np.float64), (B,))[:, None]
    wi = np.broadcast_to(np.asarray(wi, np.float64), (B,))[:, None]
    tw, th = tsz[:, 0:1].astype(np.float64), tsz[:, 1:2].astype(np.float64)
    a = anchor.astype(np.float32)
    with np.errstate(all="ignore"):
        box = np.empty((B, 4, loc.shape[2]), np.float32)
        box[:, 0] = loc[:, 0] * a[:, 2] + a[:, 0]
        box[:, 1] = loc[:, 1] * a[:, 3] + a[:, 1]
        box[:, 2] = ex(loc[:, 2]) * a[:, 2]
        box[:, 3] = ex(loc[:, 3]) * a[:, 3]
        w, h = box[:, 2], box[:, 3]

        def sz(w_, h_):
            pad = (w_ + h_) * 0.5
            return np.sqrt((w_ + pad) * (h_ + pad))

        def change(r):
            return np.maximum(r, 1.0 / r)
        s_c = change(sz(w, h) / sz(tw, th))
        r_c = change((tw / th) / (w / h))
        penalty = np.exp(-(r_c * s_c - 1) * pk)
        ps = penalty * score
        win = win.astype(np.float32).astype(np.float64) if window32 else win
        if fused is None:
            ps = ps * (1 - wi) + win * wi
        else:
            ps = _fused_pscore(ps, win, wi, fused)
    return np.argmax(ps, axis=1), box, penalty, ps


def _fused_pscore(p, win, wi, form):
    """pscore with one exact FMA.  Only the candidates that can matter (within 1e-12 of each stream's unfused maximum,
    and every NaN) are evaluated with exact rationals; the rest keep the unfused value."""
    out = p * (1 - wi) + win * wi
    top = np.nanmax(np.where(np.isnan(out), -np.inf, out), axis=1, keepdims=True)
    for b, i in zip(*np.nonzero((out >= top - 1e-12 * np.abs(top)) & np.isfinite(out))):
        q, c = float(p[b, i]), float(1 - wi[b, 0])
        out[b, i] = fma(win[i], wi[b, 0], q * c) if form == "window" else fma(q, c, win[i] * wi[b, 0])
    return out


def prepare(state, context_amount=0.5, exemplar=127, instance=255, trunc=False):
    """tools/test.py:180-198 + get_subwindow_tracking :71-76 per stream with Python floats, as the reference runs
    them.  state f64 [B,4] = (x, y, w, h).  Returns (boxes int [B,3] = xmin, ymin, round(s_x), tsz f64 [B,2],
    aux f64 [B,4] = scale_x, round(s_x), crop_box x0, y0).  trunc: the mutation that truncates instead of rounding."""
    rnd = (lambda v: float(int(v))) if trunc else (lambda v: float(round(v)))
    boxes, tsz, aux = [], [], []
    for px, py, sw, sh in np.asarray(state, np.float64):
        target_sz = np.array([sw, sh])
        wc_x = target_sz[1] + context_amount * sum(target_sz)
        hc_x = target_sz[0] + context_amount * sum(target_sz)
        s_x = np.sqrt(wc_x * hc_x)
        scale_x = exemplar / s_x
        d_search = (instance - exemplar) / 2
        pad = d_search / scale_x
        s_x = s_x + 2 * pad
        sxr = rnd(s_x)
        c = (sxr + 1) / 2
        boxes.append([int(rnd(px - c)), int(rnd(py - c)), int(sxr)])
        tsz.append(target_sz * scale_x)
        aux.append([scale_x, sxr, px - sxr / 2, py - sxr / 2])
    return np.array(boxes, np.int64), np.array(tsz), np.array(aux)


def update(state, rec, aux, im_wh, pk, lr_hp, R, exemplar=127, instance=255, base=8, stride=8, out_size=127,
           fused_subbox=False):
    """tools/test.py:226-249 (the winner's penalty re-evaluated in float64), crop_back's map :263-282 and the clamps
    :305-308, per stream.  rec f32 [B,8] as sm_select writes it; pk, lr_hp: scalars or [B].  Returns (state f64 [B,4],
    maps f64 [B,6]).  fused_subbox: the mutation that evaluates crop_back's sub-box corner with one exact FMA."""
    B = len(state)
    pk = np.broadcast_to(np.asarray(pk, np.float64), (B,))
    lr_hp = np.broadcast_to(np.asarray(lr_hp, np.float64), (B,))
    new, maps = [], []
    for b in range(B):
        px, py, sw, sh = (float(v) for v in state[b])
        target_pos, target_sz = np.array([px, py]), np.array([sw, sh])
        scale_x, sxr, cx0, cy0 = (float(v) for v in aux[b])
        im_w, im_h = int(im_wh[b][0]), int(im_wh[b][1])
        tsz_crop = target_sz * scale_x
        r = rec[b]
        w, h = r[2:3], r[3:4]                          # float32 arrays, as the reference's delta rows
        with np.errstate(all="ignore"):
            def sz(w_, h_):
                pad = (w_ + h_) * 0.5
                return np.sqrt((w_ + pad) * (h_ + pad))
            s_c = np.maximum(sz(w, h) / sz(tsz_crop[0], tsz_crop[1]), 1.0 / (sz(w, h) / sz(tsz_crop[0], tsz_crop[1])))
            rr = (tsz_crop[0] / tsz_crop[1]) / (w / h)
            r_c = np.maximum(rr, 1.0 / rr)
            penalty = float(np.exp(-(r_c * s_c - 1) * pk[b])[0])
        pred = r[:4].astype(np.float64) / scale_x
        lr = penalty * float(r[4]) * lr_hp[b]
        res_x, res_y = pred[0] + target_pos[0], pred[1] + target_pos[1]
        res_w = target_sz[0] * (1 - lr) + pred[2] * lr
        res_h = target_sz[1] * (1 - lr) + pred[3] * lr
        best_id = int(r[7])
        delta_y, delta_x = (best_id % (R * R)) // R, best_id % R       # np.unravel_index(best_id, (A, R, R))[1:]
        s = sxr / instance
        if fused_subbox:
            sub0 = fma((delta_x - base / 2) * stride, s, cx0)
            sub1 = fma((delta_y - base / 2) * stride, s, cy0)
        else:
            sub0 = cx0 + (delta_x - base / 2) * stride * s
            sub1 = cy0 + (delta_y - base / 2) * stride * s
        sub_box = [sub0, sub1, s * exemplar, s * exemplar]
        s = out_size / sub_box[2]
        back_box = [-sub_box[0] * s, -sub_box[1] * s, im_w * s, im_h * s]
        a = (im_w - 1) / back_box[2]
        bq = (im_h - 1) / back_box[3]
        maps.append([a, 0.0, -a * back_box[0], 0.0, bq, -bq * back_box[1]])
        new.append([max(0, min(im_w, res_x)), max(0, min(im_h, res_y)), max(10, min(im_w, res_w)),
                    max(10, min(im_h, res_h))])
    return np.array(new, np.float64), np.array(maps, np.float64)


def crop(frame, box, model):
    """get_subwindow_tracking (tools/test.py:67-110) on the host with cv2, from a crop box (xmin, ymin, sz, avg*3)."""
    xmin, ymin, sz = box[:3]
    c = (sz + 1) / 2
    # a position whose round(pos - c) is xmin, ymin: pos = xmin + c (exact in float64 for these integers and halves)
    return ref_loop.get_subwindow_tracking(frame, [xmin + c, ymin + c], model, sz, np.asarray(box[3:6], np.float64))
