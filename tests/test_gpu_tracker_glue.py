"""The tracker's per-frame glue kernels against the host restatement of the reference's numpy / OpenCV arithmetic
(tests/tracker_glue_reference.py), bit for bit, on constructed inputs: the selection (sm_select, and once through
sm_step_slots_hp), numpy's float32 exp inside it, the search-window and state-update kernels (sm_tracker_prepare,
sm_tracker_update(_hp)), the crop (sm_crop_resize, _indexed, _ragged) and the paste-back of the maps the update
writes (sm_warp_affine, _ragged).  Each frame's output feeds the next frame's crop, so an ulp here compounds."""
import ctypes as C

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

import siammask_b200 as smb
import tracker_glue_reference as ref
from siammask_b200 import _lib, ops
from siammask_b200.tracker import IMAGE_DESC
from oracle import ref_loop
from test_tracker_glue_host import edge_states, expf_sweep, numpy_expf_is_simd, tie_inputs, update_inputs

pytestmark = pytest.mark.gpu
ANCHORS = {"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8]}
# The penalty's float64 exp (device libm against numpy's) may differ by an ulp; with pscore <= ~2 that moves it by
# < 1e-15.  Only streams whose restated top two are closer than this (relative) may pick the other one.
MARGIN = 1e-13
_ENGINES = {}


def _engine(R):
    if R not in _ENGINES:
        _ENGINES[R] = smb.Custom(anchors=smb.DEFAULT_ANCHORS, search_size=(R - 9) * 8 + 127).to("cuda")
    return _ENGINES[R]


def _device_select(R, cls, loc, tsz, pk, wi):
    """cls f32 [B,2,n], loc f32 [B,4,n] in (anchor, y, x) order -> sm_select's (best, rec) and torch.softmax's score."""
    B = cls.shape[0]
    c = torch.from_numpy(cls).cuda().reshape(B, 10, R, R)
    lo = torch.from_numpy(loc).cuda().reshape(B, 20, R, R)
    anchor = ref_loop.generate_anchor(ANCHORS, R)
    best, _, rec = _engine(R).select(c, lo, torch.from_numpy(anchor), torch.from_numpy(ref.window(R, 5)),
                                     torch.from_numpy(tsz), pk, wi)
    score = torch.softmax(torch.from_numpy(cls).cuda(), dim=1)[:, 1].cpu().numpy()     # tools/test.py:206-207
    return best.cpu().numpy(), rec.cpu().numpy(), score, anchor


def _same(a, b):
    """Bit-equal, or NaN on both sides (the device's NaN payload is its own)."""
    return (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))


def _check_select(R, cls, loc, tsz, pk, wi, exact=True):
    best, rec, score, anchor = _device_select(R, cls, loc, tsz, pk, wi)
    want, box, pen, ps = ref.select(score, loc, anchor, ref.window(R, 5), tsz, pk, wi)
    B = len(best)
    bad = np.flatnonzero(best != want)
    if not exact and bad.size:
        top2 = np.sort(np.where(np.isnan(ps), np.inf, ps), axis=1)[:, -2:]
        close = np.abs(top2[:, 1] - top2[:, 0]) <= MARGIN * np.abs(top2[:, 1])
        bad = bad[~close[bad]]
    assert bad.size == 0, f"{bad.size}/{B} winners differ, e.g. stream {bad[0]}: device {best[bad[0]]} numpy {want[bad[0]]}"
    assert np.array_equal(rec[:, 7], best.astype(np.float32))
    b = np.arange(B)
    k = best
    assert _same(rec[:, 0:4], box[b, :, k]).all(), "decoded box not bit-equal"
    # the kernel's softmax (expf of the difference, one division) against torch.softmax on the device
    u = np.abs(rec[:, 4].view(np.int32).astype(np.int64) - score[b, k].view(np.int32).astype(np.int64))
    assert ((u <= 1) | (np.isnan(rec[:, 4]) & np.isnan(score[b, k]))).all(), f"score differs from torch.softmax by {u.max()} ulp"
    fin = np.isfinite(pen[b, k])
    pu = np.abs(rec[fin, 5].view(np.int32).astype(np.int64) - pen[b, k][fin].astype(np.float32).view(np.int32))
    assert (pu <= 1).all(), "penalty"
    return best, rec, score


@pytest.mark.parametrize("R", [25, 41])
@pytest.mark.parametrize("B", [1, 3, 64, 256])
def test_select_random(R, B):
    g = np.random.RandomState(R * 1000 + B)
    n = 5 * R * R
    cls = (g.randn(B, 2, n) * 3).astype(np.float32)
    loc = (g.randn(B, 4, n) * 0.5).astype(np.float32)
    tsz = g.rand(B, 2) * 80 + 10
    for pk, wi in ((0.04, 0.4), (0.0, 0.4), (0.09, 0.0), (0.09, 1.0)):
        _check_select(R, cls, loc, tsz, pk, wi, exact=pk == 0.0 or wi == 1.0)


@pytest.mark.parametrize("R", [25, 41])
def test_select_exact_ties_pick_the_lowest_index(R):
    B, n = 4, 5 * R * R
    cls = np.zeros((B, 2, n), np.float32)
    loc = np.zeros((B, 4, n), np.float32)
    tsz = np.full((B, 2), 64.0)
    best, _, _ = _check_select(R, cls, loc, tsz, 0.04, 0.0)          # equal scores: the ratio-1 anchor's penalty wins
    assert (best == 2 * R * R).all()
    best, _, _ = _check_select(R, cls, loc, tsz, 0.0, 0.0)           # penalty 1: every pscore equal
    assert (best == 0).all()
    best, _, _ = _check_select(R, cls, loc, tsz, 0.04, 1.0)          # the window alone: its maximum in every anchor
    assert (best == (R * R) // 2).all()


def test_select_window_ties():
    """Candidate pairs with equal cls / loc whose float64 window values round to the same float32: numpy ranks them,
    a float32 window cannot.  2048 streams, scores spread over [0.63, 1)."""
    R, B = 25, 2048
    cls, loc = tie_inputs(R, B)
    best, _, _ = _check_select(R, cls, loc, np.full((B, 2), 40.0), 0.0, 0.4)
    firsts = [p for p, _ in ref.window_tie_pairs(R)]
    assert (~np.isin(best % 625, firsts)).any()


@pytest.mark.parametrize("R", [25, 41])
def test_select_near_ties(R):
    """Two candidates near the window's centre, all others with a negligible score; window_influence solved so that
    their pscores differ by a relative margin of 1e-12 .. 1e-6, either way round."""
    n, RR, c = 5 * R * R, R * R, (R * R) // 2
    win = ref.window(R, 5)
    for m in (1e-12, 1e-10, 1e-8, 1e-6):
        for sign in (1, -1):
            i, j = 2 * RR + c, 3 * RR + c + 1
            cls = np.zeros((1, 2, n), np.float32)
            cls[0, 1] = -20
            cls[0, 1, i], cls[0, 1, j] = 2.0, 3.0
            loc = np.zeros((1, 4, n), np.float32)
            s = torch.softmax(torch.from_numpy(cls).cuda(), dim=1)[0, 1].cpu().numpy().astype(np.float64)
            ds, dw = s[i] - s[j], win[i] - win[j]
            wi0 = ds / (ds - dw)
            wi = wi0 + sign * m * (s[i] * (1 - wi0) + win[i] * wi0) / (dw - ds)
            best, _, _ = _check_select(R, cls, loc, np.full((1, 2), 40.0), 0.0, wi)
            assert best[0] == (i if sign > 0 else j)


@pytest.mark.parametrize("R", [25, 41])
def test_select_non_finite(R):
    """NaN in cls (the first NaN wins, as with np.argmax); NaN, +-inf, huge and tiny loc values (w = inf, w = 0,
    w = h = 0 and a NaN ratio)."""
    g = np.random.RandomState(9)
    n = 5 * R * R
    B = 8
    cls = (g.randn(B, 2, n) * 2).astype(np.float32)
    loc = (g.randn(B, 4, n) * 0.3).astype(np.float32)
    cls[0, 1, [700, 90]] = np.nan
    cls[1, 0, 33] = np.nan
    for b, vals in ((2, [np.nan]), (3, [np.inf, -np.inf]), (4, [1e30, -1e30]), (5, [1e-30, -1e-30]), (6, [200.0, -200.0])):
        idx = g.choice(n, 50, replace=False)
        for k, v in enumerate(vals):
            loc[b, 2 + k % 2, idx] = v
            loc[b, k % 2, idx[::2]] = v
    loc[7, 2:4, g.choice(n, 50, replace=False)] = -200.0                  # w = h = 0: w / h is NaN
    tsz = g.rand(B, 2) * 80 + 10
    for pk, wi in ((0.04, 0.4), (0.0, 0.0), (0.0, 1.0)):
        best, _, _ = _check_select(R, cls, loc, tsz, pk, wi, exact=pk == 0.0)
        assert best[0] == 90 and best[1] == 33


def test_select_expf_sweep():
    """w = np.exp(loc[2]) * anchor_w and h likewise (float32, tools/test.py:211-212) for ~10^6 arguments, read back
    from the records of streams whose winner carries them."""
    if not numpy_expf_is_simd():
        pytest.skip("this numpy's float32 exp is correctly rounded, not the SIMD algorithm the device restates")
    R, B = 25, 8192
    n, k = 5 * R * R, 2 * 625 + 312                      # winner: anchor 2 (ratio 1, 64 x 64), the centre
    x = expf_sweep()
    x = np.concatenate([x, np.zeros((-len(x)) % (2 * B), np.float32)])
    cls = np.zeros((B, 2, n), np.float32)
    cls[:, 1] = -30
    cls[:, 1, k] = 30
    anchor = ref_loop.generate_anchor(ANCHORS, R)
    aw = anchor[k, 2]
    got = []
    for s in range(0, len(x), 2 * B):
        loc = np.zeros((B, 4, n), np.float32)
        loc[:, 2, k], loc[:, 3, k] = x[s:s + B], x[s + B:s + 2 * B]
        best, rec, _, _ = _device_select(R, cls, loc, np.full((B, 2), 64.0), 0.0, 0.0)
        assert (best == k).all()
        got.append(np.concatenate([rec[:, 2], rec[:, 3]]))
    got = np.concatenate(got)
    with np.errstate(over="ignore", under="ignore"):
        want = np.exp(x) * aw
    same = _same(got, want)
    assert same.all(), f"{(~same).sum()} of {len(x)} differ, e.g. x = {x[~same][:4]}"


def test_step_slots_hp_matches_restatement(calib_sd):
    """One frame through sm_step_slots_hp: per-stream (penalty_k, window_influence) rows give the restatement's
    winners and records on the frame's own cls / loc."""
    from oracle.calibrate import synthetic_inputs
    B, R = 6, 25
    m = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=B).load_state_dict(calib_sd).eval().to("cuda")
    z, x = synthetic_inputs(41, B)
    m.template(z.cuda())
    rows = np.array([[0.04, 0.4, 1.0], [0.0, 0.4, 1.0], [0.09, 0.0, 1.0], [0.0, 1.0, 1.0], [0.02, 0.3, 1.0],
                     [0.1, 0.5, 1.0]])
    tsz = np.random.RandomState(2).rand(B, 2) * 60 + 30
    anchor = ref_loop.generate_anchor(ANCHORS, R)
    out = m.step(x.cuda(), torch.from_numpy(anchor), torch.from_numpy(ref.window(R, 5)), torch.from_numpy(tsz), 0.0, 0.0,
                 refine=False, hp=torch.from_numpy(rows).cuda())
    loc = out["loc"].reshape(B, 4, -1).cpu().numpy()
    score = torch.softmax(out["cls"].reshape(B, 2, -1), dim=1)[:, 1].cpu().numpy()
    want, box, _, _ = ref.select(score, loc, anchor, ref.window(R, 5), tsz, rows[:, 0], rows[:, 1])
    best, rec = out["best"].cpu().numpy(), out["records"].cpu().numpy()
    assert np.array_equal(best, want)
    assert _same(rec[:, 0:4], box[np.arange(B), :, best]).all()


# ------------------------------------------------------------------------------------------------ tracker state
def _prepare(st, ctx):
    lib = _lib.load()
    B = len(st)
    hp = _lib.SmTrackerHp(ctx, 0.04, 0.4, 1.0, 127, 255, 8, 8, 127, 0)
    avg = np.tile(np.int32([7, 80, 200]), (B, 1))
    sd, ad = torch.from_numpy(st.copy()).cuda(), torch.from_numpy(avg).cuda()
    boxes = torch.zeros(B, 8, dtype=torch.int32, device="cuda")
    tsz = torch.zeros(B, 2, dtype=torch.float64, device="cuda")
    aux = torch.zeros(B, 4, dtype=torch.float64, device="cuda")
    _lib.check(lib.sm_tracker_prepare(B, sd.data_ptr(), ad.data_ptr(), C.byref(hp), boxes.data_ptr(), tsz.data_ptr(),
                                      aux.data_ptr(), None))
    return boxes.cpu().numpy(), tsz.cpu().numpy(), aux.cpu().numpy()


@pytest.mark.parametrize("ctx", [0.5, 0.45])
def test_tracker_prepare_bit_exact(ctx):
    st = edge_states()
    boxes, tsz, aux = _prepare(st, ctx)
    wb, wt, wa = ref.prepare(st, ctx)
    assert np.array_equal(boxes[:, :3], wb)
    assert np.array_equal(tsz.view(np.int64), wt.view(np.int64)), "target_sz_in_crop"
    assert np.array_equal(aux.view(np.int64), wa.view(np.int64)), "aux"


def _update(st, rec, aux, im, R, out_size, pk, lr, hp_rows=None):
    lib = _lib.load()
    B = len(st)
    hp = _lib.SmTrackerHp(0.45, pk, 0.4, lr, 127, 255, 8, 8, out_size, 0)
    sd = torch.from_numpy(st.copy()).cuda()
    rd, ad = torch.from_numpy(rec).cuda(), torch.from_numpy(aux).cuda()
    imd = torch.from_numpy(im.astype(np.int32)).cuda()
    maps = torch.zeros(B, 6, dtype=torch.float64, device="cuda")
    if hp_rows is None:
        _lib.check(lib.sm_tracker_update(B, sd.data_ptr(), rd.data_ptr(), ad.data_ptr(), imd.data_ptr(), C.byref(hp), 5, R,
                                         maps.data_ptr(), None, None))
    else:
        h = torch.from_numpy(hp_rows).cuda()
        _lib.check(lib.sm_tracker_update_hp(B, sd.data_ptr(), rd.data_ptr(), ad.data_ptr(), imd.data_ptr(), C.byref(hp),
                                            h.data_ptr(), 5, R, maps.data_ptr(), None, None))
    return sd.cpu().numpy(), maps.cpu().numpy()


def _update_cases(R):
    st, aux, rec = update_inputs(R, 1000)
    B = len(st)
    g = np.random.RandomState(R)
    im = np.stack([g.randint(1, 700, B), g.randint(1, 500, B)], 1)
    im[:4] = [[320, 240], [1920, 1080], [1, 1], [17, 3]]
    return st, aux, rec, im


@pytest.mark.parametrize("R", [25, 41])
@pytest.mark.parametrize("out_size", [127, 63])
def test_tracker_update_bit_exact(R, out_size):
    st, aux, rec, im = _update_cases(R)
    B = len(st)
    for pk in (0.0, 0.04):
        for lr in (0.0, 1.0, 0.38):
            got, maps = _update(st, rec, aux, im, R, out_size, pk, lr)
            want, wmaps = ref.update(st, rec, aux, im, pk, lr, R, out_size=out_size)
            assert np.array_equal(maps.view(np.int64), wmaps.view(np.int64)), "crop_back map"
            assert np.array_equal(got[:, :2].view(np.int64), want[:, :2].view(np.int64)), "position"
            if pk == 0.0:
                assert np.array_equal(got[:, 2:].view(np.int64), want[:, 2:].view(np.int64)), f"size lr={lr}"
            else:      # the penalty's float64 exp may differ by an ulp, which reaches w, h through lr
                np.testing.assert_allclose(got[:, 2:], want[:, 2:], rtol=4e-16, atol=0)
    # both sides of every clamp were reached
    for c, lim in ((0, im[:, 0]), (1, im[:, 1]), (2, im[:, 0]), (3, im[:, 1])):
        assert (want[:, c] == (0 if c < 2 else 10)).any() and (want[:, c] == lim).any(), f"clamp {c}"
    # per-stream rows: the same arithmetic, row by row
    rows = np.stack([np.where(np.arange(B) % 2, 0.0, 0.04), np.full(B, 0.4), np.linspace(0, 1, B)], 1)
    got, maps = _update(st, rec, aux, im, R, out_size, 0.5, 0.5, rows)
    want, wmaps = ref.update(st, rec, aux, im, rows[:, 0], rows[:, 2], R, out_size=out_size)
    assert np.array_equal(maps.view(np.int64), wmaps.view(np.int64))
    z = rows[:, 0] == 0
    assert np.array_equal(got[z].view(np.int64), want[z].view(np.int64))


# ------------------------------------------------------------------------------------------------ crop
def _frames():
    g = np.random.RandomState(4)
    return [g.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((1, 1), (1, 57), (97, 131), (1080, 1920))]


def _crop_boxes(frame, sizes, g):
    H, W = frame.shape[:2]
    out = []
    for sz in sizes:
        for xmin, ymin in ((W // 2 - sz // 2, H // 2 - sz // 2), (-sz // 2, -sz // 2), (W - sz // 2, H - sz // 2),
                           (W + 3, -sz - 2), (int(g.randint(-sz, W + 1)), int(g.randint(-sz, H + 1)))):
            out.append([xmin, ymin, sz, 17, 140, 251])
    return np.array(out)


@pytest.mark.parametrize("model", [127, 255, 383])
def test_crop_sweep_bit_exact(model):
    """Every sz from 1 to 1024 (and a sample up to the ~6000 px windows of a 1920 x 1080 frame), windows inside,
    straddling edges and corners, outside and larger than the frame, on 1x1, 1xW, odd-sized and 1920x1080 frames;
    sm_crop_resize, _indexed and _ragged against the cv2 path."""
    g = np.random.RandomState(model)
    frames = _frames()
    lib = _lib.load()
    plan = [(frames[0], list(range(1, 40))), (frames[1], list(range(1, 80, 3))), (frames[2], list(range(1, 1025))),
            (frames[3], [1, 3, 5, 15, 17, 255, 383] + list(g.randint(1025, 6001, 6)))]
    packed = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).cuda()
    desc = np.zeros(len(frames), IMAGE_DESC)
    off = 0
    for i, f in enumerate(frames):
        desc[i] = (off, f.shape[0], f.shape[1])
        off += f.size
    desc_d = torch.from_numpy(desc.view(np.uint8).copy()).cuda()
    for fi, (frame, sizes) in enumerate(plan):
        boxes = _crop_boxes(frame, sizes, g)
        fd = torch.from_numpy(frame).cuda()
        for s in range(0, len(boxes), 128):
            bx = boxes[s:s + 128]
            got = ops.crop_resize(fd, bx, model).cpu().numpy()
            full = torch.zeros(len(bx), 8, dtype=torch.int32)
            full[:, :6] = torch.from_numpy(bx.astype(np.int32))
            full = full.cuda()
            idx = torch.full((len(bx),), fi, dtype=torch.int32, device="cuda")
            rag = ops._crop_resize_ragged(packed, desc_d, idx, full, model).cpu().numpy()
            fstack = torch.from_numpy(np.stack([frame, frame])).cuda()     # frame 1 of a 2-frame batch
            ind = torch.empty(len(bx), 3, model, model, device="cuda")
            one = torch.ones(len(bx), dtype=torch.int32, device="cuda")
            _lib.check(lib.sm_crop_resize_indexed(fstack.data_ptr(), frame.size, frame.shape[0], frame.shape[1],
                                                  one.data_ptr(), full.data_ptr(), len(bx), model, ind.data_ptr(), None))
            ind = ind.cpu().numpy()
            for k, b in enumerate(bx):
                want = ref.crop(frame, [int(v) for v in b], model).numpy()
                for name, arr in (("crop_resize", got), ("ragged", rag), ("indexed", ind)):
                    assert np.array_equal(arr[k], want), f"{name} frame {frame.shape} box {b} -> {model}"


# ------------------------------------------------------------------------------------------------ paste-back
@pytest.mark.parametrize("R,out_size", [(25, 127), (41, 63)])
def test_paste_back_of_update_maps_bit_exact(R, out_size):
    st, aux, rec, im = _update_cases(R)
    sel = np.r_[0:4, 6:40]
    st, aux, rec, im = st[sel], aux[sel], rec[sel], im[sel]
    _, maps = _update(st, rec, aux, im, R, out_size, 0.04, 0.38)
    _, wmaps = ref.update(st, rec, aux, im, 0.04, 0.38, R, out_size=out_size)
    B = len(st)
    src = np.random.RandomState(1).rand(B, out_size, out_size).astype(np.float32)
    desc = np.zeros(B, IMAGE_DESC)
    off = 0
    for b in range(B):
        desc[b] = (off, im[b, 1], im[b, 0])
        off += int(im[b, 0] * im[b, 1])
    rag = ops._warp_affine_ragged(torch.from_numpy(src).cuda(), torch.from_numpy(maps).cuda(),
                                  torch.from_numpy(desc.view(np.uint8).copy()).cuda(),
                                  (int(im[:, 1].max()), int(im[:, 0].max())), off).cpu().numpy()
    for b in range(B):
        W, H = int(im[b, 0]), int(im[b, 1])
        want = cv2.warpAffine(src[b], wmaps[b].reshape(2, 3), (W, H), flags=cv2.INTER_LINEAR,
                              borderMode=cv2.BORDER_CONSTANT, borderValue=-1)
        got = ops.warp_affine(torch.from_numpy(src[b]).cuda(), maps[b], (W, H)).cpu().numpy()
        assert np.array_equal(got, want), f"stream {b}: warp_affine"
        assert np.array_equal(rag[desc[b]["offset"]:desc[b]["offset"] + W * H].reshape(H, W), want), f"stream {b}: ragged"
