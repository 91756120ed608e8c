"""Hyper-parameter sweeps on the device: the per-stream hyper-parameter table (sm_step_slots_hp /
sm_tracker_update_hp), the graph key of sm_step / sm_step_slots, BatchTracker with per-stream hp, the fused paste-back +
IoU counts (sm_mask_iou), and ParamSweep end to end against the tune_vos restatement in tests/sweep_reference.py."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

import siammask_b200 as smb
from siammask_b200 import _lib, ops
from siammask_b200.ops import mask_iou, warp_affine
from siammask_b200.tracker import BatchTracker, TrackerParams
from siammask_b200.tune import grid
from oracle import ref_loop
from oracle.calibrate import calibrated_state_dict, synthetic_inputs
from oracle.synthetic_video import make_frames
from sweep_reference import tune_run

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}
STEP_KEYS = ("cls", "loc", "best", "pos", "records", "refine")


def _params():
    return TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


def _net(sd, max_batch, num_slots, graphs=False):
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch, num_slots=num_slots,
                      graphs=graphs).load_state_dict(sd).eval().to("cuda")


def _table(rows):
    return torch.tensor(np.asarray(rows, np.float64).reshape(-1, 3), dtype=torch.float64, device="cuda")


def _step(net, x, bt, tsz, pk=0.04, wi=0.4, slots=None, hp=None):
    out = net.step(x, bt.anchors, bt.window, tsz, pk, wi, refine=True, slots=slots, hp=hp)
    return {k: out[k].clone() for k in STEP_KEYS}


def _setup(sd, B, graphs=False, seed=5):
    net = _net(sd, max_batch=17, num_slots=24, graphs=graphs)
    bt = BatchTracker(net, _params())                  # anchors / window only
    z, x = synthetic_inputs(seed, B)
    z, x = z.cuda(), x.cuda()
    slots = torch.tensor(np.random.RandomState(B).permutation(24)[:B], dtype=torch.int32, device="cuda")
    net.template(z, slot0=0)                           # slots 0..B-1 for the calls without a table
    net.template(z, slots=slots)
    tsz = torch.rand(B, 2, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(B)) * 60 + 20
    return net, bt, x, tsz, slots


# ---------------------------------------------------------------------------------------------- 1. uniform table
@pytest.mark.parametrize("B", [3, 17])
def test_uniform_hp_table_equals_scalars(sd, B):
    net, bt, x, tsz, slots = _setup(sd, B)
    want = _step(net, x, bt, tsz, slots=slots)
    got = _step(net, x, bt, tsz, pk=9.0, wi=9.0, slots=slots, hp=_table([[0.04, 0.4, 1.0]] * B))  # scalars ignored
    torch.cuda.synchronize()
    for k in STEP_KEYS:
        assert torch.equal(got[k], want[k]), k


def test_tracker_update_hp_uniform_table_equals_struct():
    lib = _lib.load()
    B, A, R = 9, 5, 25
    rng = np.random.RandomState(0)
    state = torch.from_numpy(np.c_[rng.rand(B, 2) * 300 + 50, rng.rand(B, 2) * 80 + 20]).cuda()
    rec = np.zeros((B, 8), np.float32)
    rec[:, :2] = rng.randn(B, 2) * 10
    rec[:, 2:4] = rng.rand(B, 2) * 60 + 30
    rec[:, 4] = rng.rand(B)
    rec[:, 7] = rng.randint(0, A * R * R, B)
    rec = torch.from_numpy(rec).cuda()
    aux = torch.from_numpy(np.c_[rng.rand(B) + 0.5, rng.randint(200, 400, B), rng.rand(B, 2) * 100]).cuda()
    imwh = torch.tensor([[640, 480]] * B, dtype=torch.int32, device="cuda")
    p = TrackerParams(penalty_k=0.07, lr=0.85)
    hp = p.c_struct()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    outs = []
    for table in (None, _table([[0.07, 0.4, 0.85]] * B)):
        s, maps, out = state.clone(), torch.zeros(B, 6, dtype=torch.float64, device="cuda"), \
            torch.zeros(B, 8, dtype=torch.float64, device="cuda")
        if table is None:
            _lib.check(lib.sm_tracker_update(B, s.data_ptr(), rec.data_ptr(), aux.data_ptr(), imwh.data_ptr(),
                                             C.byref(hp), A, R, maps.data_ptr(), out.data_ptr(), st))
        else:
            _lib.check(lib.sm_tracker_update_hp(B, s.data_ptr(), rec.data_ptr(), aux.data_ptr(), imwh.data_ptr(),
                                                C.byref(hp), table.data_ptr(), A, R, maps.data_ptr(), out.data_ptr(), st))
        outs.append((s, maps, out))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    # distinct rows: stream b follows the struct run with row b's penalty_k / lr
    rows = np.c_[rng.rand(B) * 0.1, rng.rand(B), rng.rand(B) * 0.5 + 0.5]
    s, out = state.clone(), torch.zeros(B, 8, dtype=torch.float64, device="cuda")
    _lib.check(lib.sm_tracker_update_hp(B, s.data_ptr(), rec.data_ptr(), aux.data_ptr(), imwh.data_ptr(), C.byref(hp),
                                        _table(rows).data_ptr(), A, R, None, out.data_ptr(), st))
    for b in range(B):
        hb = TrackerParams(penalty_k=rows[b, 0], window_influence=rows[b, 1], lr=rows[b, 2]).c_struct()
        sb, ob = state.clone(), torch.zeros(B, 8, dtype=torch.float64, device="cuda")
        _lib.check(lib.sm_tracker_update(B, sb.data_ptr(), rec.data_ptr(), aux.data_ptr(), imwh.data_ptr(), C.byref(hb),
                                         A, R, None, ob.data_ptr(), st))
        torch.cuda.synchronize()
        assert torch.equal(s[b], sb[b]) and torch.equal(out[b], ob[b]), b


# ---------------------------------------------------------------------------------------------- 2. distinct rows
def test_distinct_rows_equal_uniform_runs_eager_and_replayed(sd):
    B = 5
    rows = np.c_[np.linspace(0.0, 0.09, B), np.linspace(0.3, 0.46, B), np.linspace(0.8, 1.0, B)]
    net, bt, x, tsz, slots = _setup(sd, B)
    got = _step(net, x, bt, tsz, slots=slots, hp=_table(rows))
    for b in range(B):
        one = _step(net, x, bt, tsz, slots=slots, hp=_table([rows[b]] * B))
        torch.cuda.synchronize()
        for k in STEP_KEYS:
            assert torch.equal(got[k][b], one[k][b]), (b, k)
    assert len({float(v) for v in got["records"][:, 5].cpu()}) > 1          # the rows do change the penalties
    # graph replay reads the table's current contents
    gnet, gbt, gx, gtsz, gslots = _setup(sd, B, graphs=True)
    table = _table(rows)
    for r in (rows, rows, rows, rows[::-1].copy(), rows[[2, 2, 0, 4, 1]]):       # eager, capture, replay, replays
        table.copy_(_table(r))
        want = _step(net, x, bt, tsz, slots=slots, hp=table)
        have = _step(gnet, gx, gbt, gtsz, slots=gslots, hp=table)
        torch.cuda.synchronize()
        for k in STEP_KEYS:
            assert torch.equal(have[k], want[k]), k


# ---------------------------------------------------------------------------------------------- 3. graph key
@pytest.mark.parametrize("with_slots", [False, True])
def test_graph_replay_uses_the_scalars_of_each_call(sd, with_slots):
    B = 3
    eager, bt, x, tsz, slots = _setup(sd, B)
    graph, gbt, gx, gtsz, gslots = _setup(sd, B, graphs=True)
    calls = [(0.04, 0.4), (0.09, 0.4), (0.09, 0.2), (0.0, 0.46), (0.09, 0.2), (0.09, 0.2), (0.04, 0.4)]
    for pk, wi in calls:
        want = _step(eager, x, bt, tsz, pk, wi, slots=slots if with_slots else None)
        have = _step(graph, gx, gbt, gtsz, pk, wi, slots=gslots if with_slots else None)
        torch.cuda.synchronize()
        for k in STEP_KEYS:
            assert torch.equal(have[k], want[k]), ((pk, wi), k)


# ---------------------------------------------------------------------------------------------- 4. BatchTracker
def _ref_run(sd, frames, box, start, stop, hp):
    net = _net(sd, 1, 1)
    x, y, w, h = box
    state = ref_loop.siamese_init(torch.from_numpy(frames[start]).cuda(), np.array([x + w / 2, y + h / 2]),
                                  np.array([w, h], np.float64), net, {**HP, **hp})
    out = {}
    for t in range(start + 1, stop):
        state = ref_loop.siamese_track(state, torch.from_numpy(frames[t]).cuda(), True, True, device_paste=True)
        out[t] = (state["target_pos"].copy(), state["target_sz"].copy())
    return out


def test_batch_tracker_per_stream_hp_follows_single_stream_runs(sd):
    T = 6
    vids = [make_frames(n=T, seed=s) for s in range(3)]
    frames = [np.stack([v[0][t] for v in vids], 0) for t in range(T)]
    hps = [{"penalty_k": 0.0, "window_influence": 0.3, "lr": 0.8}, {"penalty_k": 0.09, "window_influence": 0.46,
                                                                     "lr": 1.0},
           {"penalty_k": 0.03, "window_influence": 0.34, "lr": 0.9}]
    row = [[h["penalty_k"], h["window_influence"], h["lr"]] for h in hps]
    bt = BatchTracker(_net(sd, 4, 4), _params())
    ids = {}
    ids[0], ids[1] = bt.add(frames[0], [vids[0][1][0], vids[1][1][0]], frame_index=[0, 1], hp=row[:2])
    got = {0: {}, 1: {}, 2: {}}
    for t in range(1, T):
        if t == 3:
            bt.remove([ids[0]])
        r = bt.track(frames[t])
        s = r.state.cpu().numpy()
        for v, sid in ids.items():
            if sid in r.extras["ids"]:
                got[v][t] = s[r.extras["ids"].index(sid)]
        if t == 2:
            ids[2], = bt.add(frames[t], [vids[2][1][t]], frame_index=[2], hp=row[2:])
    spans = {0: (0, 3), 1: (0, T), 2: (2, T)}
    for v, (s0, e) in spans.items():
        ref = _ref_run(sd, vids[v][0], vids[v][1][s0], s0, e, hps[v])
        assert sorted(got[v]) == sorted(ref), v
        for t, st in got[v].items():
            np.testing.assert_allclose(st[0:2], ref[t][0], rtol=0, atol=1e-5, err_msg=f"stream {v} frame {t}")
            np.testing.assert_allclose(st[2:4], ref[t][1], rtol=0, atol=1e-5, err_msg=f"stream {v} frame {t}")


def _scalar_track(bt, frames):
    """One frame of BatchTracker.track through the scalar entry points (sm_step_slots, sm_tracker_update): the path the
    tracker took before it carried a per-stream table."""
    p, N, lib = bt.p, bt.N, bt.lib
    fr = bt._input(frames)
    st = bt._stream()
    _lib.check(lib.sm_tracker_prepare(N, bt.state.data_ptr(), bt.avg.data_ptr(), C.byref(bt.hp), bt.boxes.data_ptr(),
                                      bt.tsz.data_ptr(), bt.aux.data_ptr(), st))
    x = ops._crop_resize_ragged(fr.data, fr.desc, bt._fidx_dev, bt.boxes, p.instance_size)
    out = bt.net._step(x, bt.anchors, bt.window, bt.tsz, p.penalty_k, p.window_influence, refine=True,
                       slots=bt._slots_dev)
    res = torch.empty(N, 8, dtype=torch.float64, device="cuda")
    _lib.check(lib.sm_tracker_update(N, bt.state.data_ptr(), out["records"].data_ptr(), bt.aux.data_ptr(),
                                     bt.imsize.data_ptr(), C.byref(bt.hp), bt.net.anchor_num, p.score_size,
                                     bt.maps.data_ptr(), res.data_ptr(), st))
    m = out["refine"].sigmoid().view(N, 127, 127).contiguous()
    return res, m


def test_batch_tracker_without_hp_is_unchanged(sd):
    T = 5
    vids = [make_frames(n=T, seed=s) for s in range(3)]
    frames = [np.stack([v[0][t] for v in vids], 0) for t in range(T)]
    boxes = [v[1][0] for v in vids]
    a = BatchTracker(_net(sd, 3, 3), _params()).init(frames[0], boxes)
    b = BatchTracker(_net(sd, 3, 3), _params()).init(frames[0], boxes)
    for t in range(1, T):
        ra = a.track(frames[t], paste=False)
        sb, mb = _scalar_track(b, frames[t])
        torch.cuda.synchronize()
        assert torch.equal(ra.state, sb), t
        assert torch.equal(ra.extras["mask_prob"], mb), t
        assert torch.equal(a.maps, b.maps), t


# ---------------------------------------------------------------------------------------------- 5. sm_mask_iou
def _crop_back_map(cx, cy, s, W, H, side=127):
    """The forward map of crop_back (tools/test.py:263-275) for a square sub-window of size s at (cx, cy)."""
    sub = [cx - s / 2, cy - s / 2, s, s]
    k = side / sub[2]
    back = [-sub[0] * k, -sub[1] * k, W * k, H * k]
    a, b = (W - 1) / back[2], (H - 1) / back[3]
    return np.array([a, 0, -a * back[0], 0, b, -b * back[1]], np.float64)


def _counts(pasted, anno, thrs):
    """IouMeter.add's intersection / union in numpy: pred compared in float64, as NumPy 2 compares a float32 array
    with an np.float64 threshold."""
    out = np.zeros((len(thrs), 2), np.int64)
    tgt = anno > 0
    for i, t in enumerate(thrs):
        pred = pasted.astype(np.float64) > t
        out[i] = (pred & tgt).sum(), (pred | tgt).sum()
    return out


def test_mask_iou_equals_counts_over_warp_affine():
    rng = np.random.RandomState(3)
    G, H, W, side = 3, 150, 260, 127
    yy, xx = np.mgrid[0:side, 0:side]
    masks = []
    for r in range(7):                                   # smooth blob-shaped sigmoid masks, values across 0..1
        c = rng.rand(2) * 60 + 33
        d = np.sqrt((yy - c[0]) ** 2 + (xx - c[1]) ** 2)
        masks.append((1 / (1 + np.exp((d - 30) / 6))).astype(np.float32))
    masks[4][50:56, 40:70] = np.nan                      # NaN values compare false
    masks = np.stack(masks)
    maps = np.stack([_crop_back_map(70, 60, 90, W, H), _crop_back_map(240, 20, 110, W, H),     # partly off frame
                     _crop_back_map(-500, -400, 60, W, H),                                      # wholly off frame
                     _crop_back_map(130, 75, 140, W, H), _crop_back_map(100, 90, 80, W, H),
                     _crop_back_map(-500, 900, 60, W, H),                                       # wholly off frame
                     _crop_back_map(10, 140, 200, W, H)])
    video = np.array([0, 0, 1, 2, 0, 2, 1], np.int32)    # several streams share a video
    anno = np.zeros((G, H, W), np.uint8)
    anno[0, 30:100, 40:120] = 1
    anno[0, 110:140, 200:250] = 2
    anno[1] = rng.randint(0, 3, (H, W)) * (rng.rand(H, W) < 0.3)
    # video 2: empty target; stream 5 is wholly off frame on it, so its union is empty (IoU 1)
    md, mp = torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda()
    ad = torch.from_numpy(anno).cuda()
    dev_warp = warp_affine(md, mp, (W, H), -1.0).cpu().numpy()
    present = float(dev_warp[0][(dev_warp[0] > 0.4) & (dev_warp[0] < 0.6)][0])       # a value of a pasted mask
    thrs = np.r_[np.arange(0.3, 0.81, 0.05), present, -1.0, np.float64(np.float32(0.35)), 0.999]
    got = mask_iou(md, mp, ad, torch.from_numpy(video).cuda(), thrs).cpu().numpy()
    assert got.shape == (len(masks), len(thrs), 2)
    for b in range(len(masks)):
        cvw = cv2.warpAffine(masks[b], maps[b].reshape(2, 3), (W, H), flags=cv2.INTER_LINEAR,
                             borderMode=cv2.BORDER_CONSTANT, borderValue=-1)
        np.testing.assert_array_equal(got[b], _counts(cvw, anno[video[b]], thrs), err_msg=f"stream {b} (cv2)")
        np.testing.assert_array_equal(got[b], _counts(dev_warp[b], anno[video[b]], thrs), err_msg=f"stream {b}")
    assert (got[5] == 0).all()                           # empty target, empty prediction
    assert got[0, 0, 0] > 0 and got[1, 0, 1] > got[1, 0, 0]
    assert (dev_warp[0] == np.float32(present)).any()


def test_mask_iou_rejects_bad_arguments():
    masks = torch.rand(2, 127, 127, device="cuda")
    maps = torch.from_numpy(np.stack([_crop_back_map(50, 50, 60, 100, 80)] * 2)).cuda()
    anno = torch.zeros(2, 80, 100, dtype=torch.uint8, device="cuda")
    ok = mask_iou(masks, maps, anno, [0, 1], [0.5])
    assert ok.shape == (2, 1, 2)
    for thrs in ([-1.5], [0.5, float("nan")], [], list(np.linspace(0, 1, 33))):
        with pytest.raises(ValueError):
            mask_iou(masks, maps, anno, [0, 1], thrs)
    for video in ([0, 2], [-1, 0], [0], [0.0, 1.0]):
        with pytest.raises(ValueError):
            mask_iou(masks, maps, anno, video, [0.5])
    with pytest.raises(ValueError):
        mask_iou(masks.double(), maps, anno, [0, 1], [0.5])
    with pytest.raises(ValueError):
        mask_iou(masks, maps.float(), anno, [0, 1], [0.5])


def test_hp_tables_are_checked(sd):
    net, bt, x, tsz, slots = _setup(sd, 3)
    for bad in (torch.zeros(3, 3, device="cuda"), torch.zeros(3, 3, dtype=torch.float64),
                torch.zeros(2, 3, dtype=torch.float64, device="cuda"),
                torch.tensor([[0.0, 0.4, 1.0]] * 2 + [[float("inf"), 0.4, 1.0]], dtype=torch.float64, device="cuda")):
        with pytest.raises(ValueError):
            net.step(x, bt.anchors, bt.window, tsz, 0.04, 0.4, slots=slots, hp=bad)
    frames, boxes = make_frames(n=1)
    t = BatchTracker(_net(sd, 2, 2), _params())
    with pytest.raises(ValueError):
        t.add(frames[0], [boxes[0]], hp=[[0.04, 0.4]])
    with pytest.raises(ValueError):
        t.add(frames[0], [boxes[0]], hp=[[0.04, np.nan, 1.0]])


# ---------------------------------------------------------------------------------------------- 6. ParamSweep
def test_param_sweep_equals_tune_vos(sd):
    T, G = 8, 2
    vids = [make_frames(n=T, seed=s + 3) for s in range(G)]
    annos = []
    for frames, boxes in vids:
        a = []
        for (x, y, w, h) in boxes:
            m = np.zeros(frames[0].shape[:2], np.uint8)
            m[y:y + h, x:x + w] = 1
            a.append(m)
        annos.append(a)
    combos = grid([0.0, 0.09], [0.3, 0.46, 0.38], [0.8])
    assert combos.shape == (6, 3)
    net = _net(sd, G * 6, G * 6)
    sweep = smb.ParamSweep(net, _params(), combos)
    sweep.open(np.stack([v[0][0] for v in vids]), [v[1][0] for v in vids], num_frames=T)
    pos = np.zeros((T, G * 6, 2))
    for f in range(1, T):
        r = sweep.frame(np.stack([v[0][f] for v in vids]), np.stack([a[f] for a in annos]) if f < T - 1 else None)
        pos[f] = r.state[:, 0:2].cpu().numpy()
    iou_list, per_frame = sweep.result()
    assert iou_list.shape == (G, 6, 11) and per_frame.shape == (T - 2, G, 6, 11)
    single = _net(sd, 1, 1)
    for g, (frames, boxes) in enumerate(vids):
        fdev = [torch.from_numpy(f).cuda() for f in frames]
        for k, (pk, wi, lr) in enumerate(combos):
            hp = {**HP, "penalty_k": pk, "window_influence": wi, "lr": lr}
            iou, mean, rpos = tune_run(single, fdev, annos[g], boxes[0], hp, np.arange(0.3, 0.81, 0.05))
            np.testing.assert_allclose(pos[1:, g * 6 + k], rpos[1:], rtol=0, atol=1e-5, err_msg=f"video {g} combo {k}")
            np.testing.assert_allclose(per_frame[:, g, k], iou, rtol=0, atol=1e-4, err_msg=f"video {g} combo {k}")
            np.testing.assert_allclose(iou_list[g, k], mean, rtol=0, atol=1e-4, err_msg=f"video {g} combo {k}")
    assert (per_frame > 0).any() and len({tuple(np.round(p, 6)) for p in pos[-1]}) > G   # the combinations differ


def test_param_sweep_rejects_too_many_streams(sd):
    net = _net(sd, 4, 4)
    frames, boxes = make_frames(n=3)
    sweep = smb.ParamSweep(net, _params(), grid([0.0, 0.1], [0.4], [1.0, 0.9]))      # 4 combinations
    with pytest.raises(ValueError):
        sweep.open(np.stack([frames[0]] * 2), [boxes[0]] * 2, num_frames=3)
    sweep.open(frames[0][None], [boxes[0]], num_frames=3)
    with pytest.raises(ValueError):
        sweep.frame(frames[1][None])                    # frame 1 of 3 is scored: annotations required
