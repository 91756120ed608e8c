"""Frames of different sizes in one batch on the device: the *_ragged / *_sized entry points against the uniform ones
run per size group (bit for bit), and BatchTracker, VotRunner and VideoSegmenter over mixed sizes against the same
streams run in per-size runners, the single-stream reference loop and the track_vot restatement."""
import os

import numpy as np
import pytest
import torch

import siammask_b200 as smb
import vot_reference
from conftest import GOLDEN
from oracle import ref_loop
from oracle.calibrate import calibrated_state_dict
from oracle.cv_resize import resize_linear_u8
from oracle.synthetic_video import make_frames
from siammask_b200 import ops
from siammask_b200.ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED
from siammask_b200.tracker import BatchTracker, FramePacker, TrackerParams
from siammask_b200.tune import grid
from vos_reference import make_multi_frames

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}
SIZES = [(240, 320), (480, 854), (720, 1280), (97, 131)]
TRACK_SIZES = [(240, 320), (480, 854), (171, 217)]          # make_frames needs room for its drifting rectangle


def _params():
    return TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


def _net(sd, max_batch, num_slots=None, mask=True):
    if not mask:
        sd = {k: v for k, v in sd.items() if not k.startswith(("mask_model", "refine_model"))}
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch, num_slots=num_slots or max_batch,
                      mask=mask).load_state_dict(sd).eval().to("cuda")


def _noise(h, w, seed, c=3):
    return np.random.RandomState(seed).randint(0, 256, (h, w, c) if c else (h, w)).astype(np.uint8)


def _bits(t):
    return np.asarray(t.cpu().numpy() if torch.is_tensor(t) else t, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------- 1. crop
def test_crop_ragged_equals_indexed_crop_per_size_group():
    frames = [_noise(h, w, i) for i, (h, w) in enumerate(SIZES)]
    rng = np.random.RandomState(3)
    boxes, fidx = [], []
    for g, (h, w) in enumerate(SIZES):
        for sz in (255, 97, 600, 31):                               # copy path, up- and down-scaling
            for x0, y0 in ((w // 3, h // 4), (-sz // 2, h - sz // 3), (-sz - 40, -sz - 10), (w + 5, h + 5)):
                boxes.append((x0, y0, sz, *rng.randint(0, 256, 3)))     # inside, partly and wholly outside
                fidx.append(g)
    order = rng.permutation(len(boxes))                             # sizes interleaved in the batch
    boxes, fidx = np.array(boxes)[order], np.array(fidx)[order]
    pk = FramePacker("cuda").pack(frames, 3)
    table = torch.zeros(len(boxes), 8, dtype=torch.int32)                # the tracker's [B,8] box table
    table[:, :6] = torch.from_numpy(boxes)
    got = ops._crop_resize_ragged(pk.data, pk.desc, torch.from_numpy(fidx).int().cuda(), table.cuda(), 255)
    dev = [torch.from_numpy(f).cuda() for f in frames]
    for g in range(len(SIZES)):
        sel = np.nonzero(fidx == g)[0]
        want = ops.crop_resize(dev[g], boxes[sel], 255)
        assert torch.equal(got[torch.from_numpy(sel).cuda()], want), SIZES[g]
    for i in range(0, len(boxes), 13):                                 # a few streams against the cv2 host path
        x0, y0, sz, a0, a1, a2 = (int(v) for v in boxes[i])
        h, w = SIZES[fidx[i]]
        pad = np.empty((sz, sz, 3), np.uint8)
        pad[:] = (a0, a1, a2)
        ys, xs = np.arange(y0, y0 + sz), np.arange(x0, x0 + sz)
        iy, ix = (ys >= 0) & (ys < h), (xs >= 0) & (xs < w)
        pad[np.ix_(iy, ix)] = frames[fidx[i]][np.ix_(ys[iy], xs[ix])]
        ref = pad if sz == 255 else resize_linear_u8(pad, (255, 255))
        np.testing.assert_array_equal(got[i].permute(1, 2, 0).cpu().numpy(), ref.astype(np.float32))


# ---------------------------------------------------------------------------------------------- 2. paste-back
def _maps(rng, n, h, w):
    out = []
    for i in range(n):
        s = rng.uniform(30, 400)
        cx, cy = (rng.uniform(-s, w + s), rng.uniform(-s, h + s)) if i % 3 == 2 else (rng.uniform(0, w), rng.uniform(0, h))
        k = 127 / s
        back = [-(cx - s / 2) * k, -(cy - s / 2) * k, w * k, h * k]
        a, b = (w - 1) / back[2] if w > 1 else 0.5, (h - 1) / back[3] if h > 1 else 0.5
        out.append([a, 0, -a * back[0], 0, b, -b * back[1]])
    return np.array(out, np.float64)


def test_warp_affine_ragged_equals_per_stream_warp():
    sizes = SIZES + [(1, 300)]                                      # a 1-pixel-high frame
    rng = np.random.RandomState(4)
    src = torch.rand(len(sizes) * 3, 127, 127, device="cuda")
    shapes = [s for s in sizes for _ in range(3)]
    maps = np.concatenate([_maps(rng, 3, h, w) for h, w in sizes])
    desc, table = FramePacker("cuda").table(shapes, 1)
    total = int(table["offset"][-1]) + shapes[-1][0] * shapes[-1][1]
    got = ops._warp_affine_ragged(src, maps, desc, (720, 1280), total)
    for b, (h, w) in enumerate(shapes):
        want = ops.warp_affine(src[b], maps[b], (w, h), -1.0)
        o = int(table["offset"][b])
        np.testing.assert_array_equal(_bits(got[o:o + h * w].view(h, w)), _bits(want), err_msg=f"stream {b} {h}x{w}")


# ---------------------------------------------------------------------------------------------- 3. overlap
def test_vot_overlap_sized_equals_golden_in_one_call():
    g = dict(np.load(os.path.join(GOLDEN, "vot_overlap.npz")))
    a, b = torch.from_numpy(g["poly_a"]).cuda(), torch.from_numpy(g["poly_b"]).cuda()
    hw = g["size"][:, ::-1].astype(np.int64)                          # golden sizes are (W, H)
    got = ops.vot_overlap(a, b, hw)
    np.testing.assert_array_equal(_bits(got), g["overlap_bits"])
    assert np.isnan(got.cpu().numpy()).any()
    W, H = 1280, 720
    uniform = ops._vot_overlap_sized(a, b, torch.tensor([[W, H]] * a.shape[0], dtype=torch.int32, device="cuda"))
    np.testing.assert_array_equal(_bits(uniform), _bits(ops.vot_overlap(a, b, (H, W))))


def test_vot_overlap_per_pair_size_checks():
    a = torch.zeros(2, 8, device="cuda")
    for size in (np.array([[10, 10]]), np.array([[10, 10], [0, 5]]), np.array([[10.0, 10.0], [5.0, 5.0]]),
                 np.array([[70000, 70000], [5, 5]])):
        with pytest.raises(ValueError):
            ops.vot_overlap(a, a, size)


# ---------------------------------------------------------------------------------------------- 4. labels
def _label_case(seed):
    """Videos of several sizes: 70 objects (the chunked case), none, one smaller than a 32x8 block, and a mixed one."""
    rng = np.random.RandomState(seed)
    sizes = [(240, 320), (97, 131), (5, 7), (480, 854)]
    kinds = [70, 0, 3, 9]
    annos = [rng.randint(0, 6, (h, w)).astype(np.uint8) for h, w in sizes]
    objects, rows_hw = [], []
    for g, ((h, w), n) in enumerate(zip(sizes, kinds)):
        ob = []
        for k in range(n):
            kind = (OBJ_TRACKED, OBJ_INIT, OBJ_IDLE)[k % 3]
            if kind == OBJ_TRACKED:
                ob.append((kind, len(rows_hw)))
                rows_hw.append((h, w))
            else:
                ob.append((kind, 1 + k % 5))
        objects.append(ob)
    maps = np.concatenate([_maps(rng, 1, h, w) for h, w in rows_hw])
    masks = torch.rand(len(rows_hw), 127, 127, device="cuda")
    return sizes, annos, objects, masks, torch.from_numpy(maps).cuda()


def _per_video(objects, g):
    """Video g's entries with their rows unchanged (masks / maps are shared)."""
    return [0, len(objects[g])], objects[g]


def test_paste_labels_ragged_equals_uniform_per_video():
    sizes, annos, objects, masks, maps = _label_case(7)
    pk = FramePacker("cuda").pack(annos, 1)
    off = np.concatenate([[0], np.cumsum([len(o) for o in objects])])
    flat = [e for o in objects for e in o]
    H, W = max(s[0] for s in sizes), max(s[1] for s in sizes)
    total = pk.data.numel()
    thrs = torch.tensor([0.2, 0.35, 0.5, 0.9], dtype=torch.float64, device="cuda")
    tid = [(k % 7) + 1 if k % 4 else -1 for k in range(len(flat))]
    for g, o in enumerate(objects):                                  # unique within a video
        seen = set()
        for i in range(off[g], off[g + 1]):
            if tid[i] in seen:
                tid[i] = -1
            seen.add(tid[i])
    tid_dev = torch.tensor(tid, dtype=torch.int32, device="cuda")
    got = ops._paste_labels(masks, maps, pk.data, off, flat, (H, W), 0.35, ragged=(pk.desc, total))
    got_iou, cnt = ops._paste_labels_iou(masks, maps, pk.data, off, flat, tid_dev, (H, W), 0.35, thrs,
                                         ragged=(pk.desc, total))
    queries = [(g, i) for g in range(len(sizes)) for i in range(0, 7)]
    boxes = ops._label_boxes_ragged(pk.data, pk.desc, len(sizes), queries)
    assert torch.equal(got, got_iou)
    for g, (h, w) in enumerate(sizes):
        o = int(pk.table[g]["offset"])
        a = torch.from_numpy(annos[g]).cuda().unsqueeze(0)
        want = ops._paste_labels(masks, maps, a, *_per_video(objects, g), (h, w), 0.35)
        assert torch.equal(got[o:o + h * w].view(1, h, w), want), (g, h, w)
        want_l, want_c = ops._paste_labels_iou(masks, maps, a, *_per_video(objects, g),
                                               tid_dev[off[g]:off[g + 1]].contiguous(), (h, w), 0.35, thrs)
        assert torch.equal(want_l, want)
        assert torch.equal(cnt[off[g]:off[g + 1]], want_c), (g, h, w)
        want_b = ops.label_boxes(a, [(0, i) for i in range(0, 7)])
        assert torch.equal(boxes[7 * g:7 * g + 7], want_b)


# ---------------------------------------------------------------------------------------------- 5. BatchTracker
def _video(size, seed, n=8):
    return make_frames(n=n, h=size[0], w=size[1], seed=seed)


def test_batch_tracker_mixed_sizes_equal_per_size_trackers(sd):
    T = 7
    vids = {(g, s): _video(TRACK_SIZES[g], 10 * g + s, T) for g in range(3) for s in range(2)}
    late = _video((300, 410), 99, T)                                  # joins at frame 2 with a fourth size
    net = _net(sd, 8)
    bt = BatchTracker(net, _params())
    keys = sorted(vids)
    ids = bt.add([vids[k][0][0] for k in keys], [vids[k][1][0] for k in keys])
    per = {g: BatchTracker(_net(sd, 2), _params()) for g in range(3)}
    for g in range(3):
        per[g].add([vids[(g, s)][0][0] for s in range(2)], [vids[(g, s)][1][0] for s in range(2)])
    per[3] = BatchTracker(_net(sd, 1), _params())
    key_of = dict(zip(ids, keys))
    for t in range(1, T):
        if t == 2:
            new = bt.add([vids[k][0][1] for k in keys] + [late[0][1]], [late[1][1]], frame_index=[len(keys)])
            per[3].add([late[0][1]], [late[1][1]])
            key_of[new[0]] = (3, 0)
        if t == 3:
            bt.remove([ids[1]])                                        # (0, 1) leaves
            per[0].remove([per[0].ids[1]])
        if t == 4:
            pos, sz = np.array([[150.25, 110.5]]), np.array([[60.0, 50.5]])
            rid = ids[4]                                               # (2, 0) restarts
            frames_now = [vids[k][0][t - 1] for k in keys] + [late[0][t - 1]]
            bt.reinit([rid], frames_now, pos, sz)
            per[2].reinit([per[2].ids[0]], [vids[(2, 0)][0][t - 1], vids[(2, 1)][0][t - 1]], pos, sz)
        frames = [vids[k][0][t] for k in keys] + [late[0][t]]
        r = bt.track(frames, mask=True)
        assert isinstance(r.mask, list) and len(r.mask) == bt.N
        rs = {g: per[g].track([vids[(g, s)][0][t] for s in range(2)] if g < 3 else [late[0][t]], mask=True)
              for g in per if not (t < 2 and g == 3)}
        for row, i in enumerate(bt.ids):
            g, s = key_of[i]
            prow = 0 if g == 3 or (g == 0 and t >= 3) else s
            np.testing.assert_array_equal(r.state[row].cpu().numpy(), rs[g].state[prow].cpu().numpy(),
                                          err_msg=f"frame {t} stream {(g, s)}")
            assert r.mask[row].shape == (TRACK_SIZES + [(300, 410)])[g]
            assert torch.equal(r.mask[row], rs[g].mask[prow]), (t, g, s)


def test_batch_tracker_mixed_sizes_equal_reference_loop(sd):
    vids = [_video(s, i, 6) for i, s in enumerate(TRACK_SIZES)]
    bt = BatchTracker(_net(sd, 3), _params())
    bt.init([v[0][0] for v in vids], [v[1][0] for v in vids])
    got = [bt.track([v[0][t] for v in vids]).cpu() for t in range(1, 6)]
    single = _net(sd, 1)

    class _NoSelect:
        def __init__(self, n):
            self._n, self.anchors, self.anchor_num = n, n.anchors, n.anchor_num

        def __getattr__(self, k):
            return getattr(self._n, k)
    for b, (fs, bx) in enumerate(vids):
        fdev = [torch.from_numpy(f).cuda() for f in fs]
        x, y, w, h = bx[0]
        st = ref_loop.siamese_init(fdev[0], np.array([x + w / 2, y + h / 2]), np.array([w, h]), _NoSelect(single), HP,
                                   device="cuda")
        for t, f in enumerate(fdev[1:]):
            st = ref_loop.siamese_track(st, f, mask_enable=True, refine_enable=True, device="cuda", device_paste=True)
            np.testing.assert_allclose(got[t]["target_pos"][b], st["target_pos"], rtol=0, atol=1e-5)
            np.testing.assert_allclose(got[t]["target_sz"][b], st["target_sz"], rtol=1e-6, atol=1e-5)


def test_batch_tracker_rejects_a_frame_of_another_size(sd):
    a, b = _video((240, 320), 0, 2), _video((151, 217), 1, 2)
    bt = BatchTracker(_net(sd, 2), _params())
    bt.add([a[0][0], b[0][0]], [a[1][0], b[1][0]])
    with pytest.raises(ValueError):
        bt.track([b[0][1], a[0][1]])                                    # swapped sizes
    with pytest.raises(ValueError):
        bt.track([a[0][1]])                                             # stream 1 has no frame
    with pytest.raises(ValueError):
        bt.track(np.stack([a[0][1], a[0][1]]))                          # one tensor for two sizes
    with pytest.raises(ValueError):
        bt.reinit(bt.ids[:1], [b[0][1], b[0][1]], [[100.0, 100.0]], [[40.0, 40.0]])


# ---------------------------------------------------------------------------------------------- 6. VotRunner
FAR = np.array([0.0, 0.0, 10.0, 0.0, 10.0, 10.0, 0.0, 10.0])


def _sequence(size, seed, T, fail_at=()):
    frames, boxes = make_frames(n=T, h=size[0], w=size[1], seed=seed)
    gt = np.asarray([[x, y, x + w, y, x + w, y + h, x, y + h] for (x, y, w, h) in boxes], np.float64)
    gt[0] += np.array([0.5, 0.25, -0.5, 0.25, -0.5, -0.75, 0.5, -0.75])
    for f in fail_at:
        gt[f] = FAR
    return frames, gt


def _run(runner, seqs, cuda=False):
    T = max(len(s[0]) for s in seqs)

    def frame(f):
        out = [s[0][f] if f < len(s[0]) else None for s in seqs]
        return [None if x is None else torch.from_numpy(x).cuda() for x in out] if cuda else out
    runner.open(frame(0), [s[1] for s in seqs])
    for f in range(1, T):
        runner.frame(frame(f))
    return runner.result()


def test_vot_runner_mixed_sizes_equal_per_size_runners_and_reference(sd):
    combos = grid([0.04, 0.2], [0.4], [1.0])                          # K = 2
    seqs = [_sequence(TRACK_SIZES[0], 0, 14, fail_at=(1, 9)), _sequence(TRACK_SIZES[1], 1, 9, fail_at=(3,)),
            _sequence(TRACK_SIZES[2], 2, 6), _sequence(TRACK_SIZES[0], 3, 11, fail_at=(7,))]
    regions, lost = _run(smb.VotRunner(_net(sd, 8), _params(), combos), seqs)
    groups = {}
    for i, s in enumerate(seqs):
        groups.setdefault(s[0][0].shape[:2], []).append(i)
    for size, members in groups.items():
        sub = [seqs[i] for i in members]
        r2, l2 = _run(smb.VotRunner(_net(sd, 2 * len(sub)), _params(), combos), sub)
        for j, i in enumerate(members):
            np.testing.assert_array_equal(lost[i], l2[j])
            for k in range(2):
                a, b = regions[i][k], r2[j][k]
                assert [x if isinstance(x, int) else 3 for x in a] == [x if isinstance(x, int) else 3 for x in b]
                for x, y in zip(a, b):
                    if not isinstance(x, int):
                        np.testing.assert_array_equal(x, y)
    ref_net = _net(sd, 1)
    for g, (frames, gt) in enumerate(seqs):
        fdev = [torch.from_numpy(f).cuda() for f in frames]
        for k, (pk, wi, lr) in enumerate(combos):
            want, want_lost = vot_reference.track_vot(ref_net, fdev, gt, {**HP, "penalty_k": pk, "window_influence": wi,
                                                                          "lr": lr})
            got = regions[g][k]
            assert [r if isinstance(r, int) else 3 for r in got] == [r if isinstance(r, int) else 3 for r in want]
            assert lost[g, k] == want_lost
            for x, y in zip(got, want):
                if not isinstance(x, int):
                    np.testing.assert_allclose(x, y, rtol=0, atol=1e-5)


def test_vot_runner_ragged_frames_do_not_wait_for_the_device(sd):
    seqs = [_sequence(TRACK_SIZES[g], g, 9, fail_at=(2,)) for g in range(3)]
    seqs[2] = (seqs[2][0][:4], seqs[2][1][:4])                        # ends at frame 3: retired, then None
    frames = [[torch.from_numpy(s[0][f]).cuda() if f < len(s[0]) else None for s in seqs] for f in range(9)]
    runner = smb.VotRunner(_net(sd, 3), _params())
    runner.open(frames[0], [s[1] for s in seqs])
    torch.cuda.synchronize()
    quiet = (1, 2, 4, 5)                                               # frame 3 retires sequence 2
    for f in range(1, 9):
        if f in quiet:
            torch.cuda.set_sync_debug_mode("error")
        try:
            runner.frame(frames[f])
        finally:
            torch.cuda.set_sync_debug_mode("default")
    regions, lost = runner.result()
    assert lost[0, 0] >= 1 and lost[1, 0] >= 1


def test_vot_runner_rejects_bad_lists(sd):
    seqs = [_sequence(TRACK_SIZES[g], g, 4) for g in range(2)]
    runner = smb.VotRunner(_net(sd, 2), _params())
    runner.open([s[0][0] for s in seqs], [s[1] for s in seqs])
    with pytest.raises(ValueError):
        runner.frame([seqs[0][0][1]])                                   # G = 2
    with pytest.raises(ValueError):
        runner.frame([seqs[1][0][1], seqs[0][0][1]])                    # swapped sizes


# ---------------------------------------------------------------------------------------------- 7. VideoSegmenter
@pytest.mark.parametrize("score", ["whole", "spans"])
def test_video_segmenter_mixed_sizes_equal_per_size_segmenters(sd, score):
    T = 6
    sizes = [(240, 320), (288, 400), (240, 320)]
    vids = [make_multi_frames(n=T, h=h, w=w, seed=g) for g, (h, w) in enumerate(sizes)]
    objs = [(g, oid, s, e) if score == "spans" else (g, oid, s) for g, v in enumerate(vids) for (oid, s, e) in v[2]]
    seg = smb.VideoSegmenter(_net(sd, 9), _params()).open(objs, num_frames=T, score=score)
    got = [seg.frame([v[0][f] for v in vids], [v[1][f] for v in vids]) for f in range(T)]
    res = seg.result()
    groups = {}
    for g, s in enumerate(sizes):
        groups.setdefault(s, []).append(g)
    for size, members in groups.items():
        sub = [(members.index(o[0]),) + tuple(o[1:]) for o in objs if o[0] in members]
        one = smb.VideoSegmenter(_net(sd, 3 * len(members)), _params()).open(sub, num_frames=T, score=score)
        for f in range(T):
            want = one.frame(np.stack([vids[g][0][f] for g in members]), np.stack([vids[g][1][f] for g in members]))
            for j, g in enumerate(members):
                assert got[f][g].shape == size
                assert torch.equal(got[f][g], want[j]), (score, f, g)
        r1 = one.result()
        for j, g in enumerate(members):
            np.testing.assert_array_equal(res[g], r1[j])


def test_video_segmenter_rejects_mismatched_lists(sd):
    vids = [make_multi_frames(n=2, h=h, w=w, seed=g) for g, (h, w) in enumerate([(240, 320), (288, 400)])]
    seg = smb.VideoSegmenter(_net(sd, 6), _params()).open([(g, o, s) for g, v in enumerate(vids) for (o, s, _) in v[2]])
    with pytest.raises(ValueError):
        seg.frame([vids[0][0][0]], [vids[0][1][0]])                     # G = 2
    with pytest.raises(ValueError):
        seg.frame([v[0][0] for v in vids], [vids[1][1][0], vids[0][1][0]])   # anno sizes swapped
    with pytest.raises(ValueError):
        seg.frame([v[0][0] for v in vids], [vids[0][1][0]])
