"""Multi-object VOS and the stream lifecycle on the device: slot tables (sm_template_slots / sm_step_slots), the indexed
crop, the fused paste-back + label map (sm_paste_labels), label boxes (sm_label_boxes), BatchTracker.add / remove, and
VideoSegmenter end to end against the track_vos restatement in tests/vos_reference.py."""
import cv2
import numpy as np
import pytest
import torch

import siammask_b200 as smb
from siammask_b200 import _lib
from siammask_b200.ops import OBJ_IDLE, OBJ_INIT, OBJ_TRACKED, paste_labels, label_boxes, warp_affine, crop_resize
from siammask_b200.tracker import BatchTracker, TrackerParams
from oracle import ref_loop
from oracle.calibrate import calibrated_state_dict, synthetic_inputs
from oracle.synthetic_video import make_frames
from vos_reference import make_multi_frames, track_vos

pytestmark = pytest.mark.gpu
HP = {"instance_size": 255, "base_size": 8, "out_size": 127, "seg_thr": 0.35, "penalty_k": 0.04,
      "window_influence": 0.4, "lr": 1.0}


def _params():
    return TrackerParams(instance_size=255, out_size=127, seg_thr=HP["seg_thr"], penalty_k=HP["penalty_k"],
                         window_influence=HP["window_influence"], lr=HP["lr"])


@pytest.fixture(scope="module")
def sd():
    return calibrated_state_dict(0)


def _net(sd, max_batch, num_slots, graphs=False):
    return smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=max_batch, num_slots=num_slots,
                      graphs=graphs).load_state_dict(sd).eval().to("cuda")


def _step_outputs(net, x, bt, tsz, slot0=0, slots=None):
    out = net.step(x, bt.anchors, bt.window, tsz, 0.04, 0.4, slot0=slot0, refine=True, slots=slots)
    return {k: out[k].clone() for k in ("cls", "loc", "records", "refine", "pos")}


# ---------------------------------------------------------------------------------------------- 1. slot tables
@pytest.mark.parametrize("B", [3, 17])
def test_slot_tables_equal_contiguous_slots(sd, B):
    S = 24
    net = _net(sd, max_batch=17, num_slots=S)
    bt = BatchTracker(net, _params())                  # anchors / window only
    z, x = synthetic_inputs(5, B)
    z, x = z.cuda(), x.cuda()
    tsz = torch.rand(B, 2, dtype=torch.float64, device="cuda") * 60 + 20
    net.template(z, slot0=2)
    want = _step_outputs(net, x, bt, tsz, slot0=2)
    perm = np.random.RandomState(B).permutation(S)[:B]          # permuted, non-contiguous slot set
    slots = torch.tensor(perm, dtype=torch.int32, device="cuda")
    net.template(torch.zeros_like(z), slot0=S - B)             # other slots hold other templates
    net.template(z, slots=slots)
    got = _step_outputs(net, x, bt, tsz, slots=slots)
    torch.cuda.synchronize()
    for k in want:
        assert torch.equal(got[k], want[k]), k
    assert net.status() & 2 == 0


def test_slot_table_graph_replay_sees_new_contents(sd):
    B, S = 3, 8
    z, x = synthetic_inputs(6, S)
    z, x = z.cuda(), x.cuda()[:B]
    eager, graph = _net(sd, 8, S), _net(sd, 8, S, graphs=True)
    bt = BatchTracker(eager, _params())
    tsz = torch.full((B, 2), 40.0, dtype=torch.float64, device="cuda")
    for n in (eager, graph):
        n.template(z, slot0=0)
    for table in ([4, 1, 2], [4, 1, 2], [4, 1, 2], [0, 7, 3], [6, 5, 4]):   # eager, capture, replay, replays
        t = torch.tensor(table, dtype=torch.int32, device="cuda")
        want = _step_outputs(eager, x, bt, tsz, slots=t)
        got = _step_outputs(graph, x, bt, tsz, slots=t)
        torch.cuda.synchronize()
        for k in want:
            assert torch.equal(got[k], want[k]), (table, k)


def test_invalid_slot_tables_are_rejected(sd):
    net = _net(sd, 4, 6)
    bt = BatchTracker(net, _params())
    z, x = synthetic_inputs(7, 3)
    z, x = z.cuda(), x.cuda()
    tsz = torch.full((3, 2), 40.0, dtype=torch.float64, device="cuda")
    bad = [torch.tensor([0, 1, 6], dtype=torch.int32, device="cuda"),      # out of range
           torch.tensor([0, -1, 2], dtype=torch.int32, device="cuda"),
           torch.tensor([0, 1], dtype=torch.int32, device="cuda"),         # wrong length
           torch.tensor([0, 1, 2], dtype=torch.int64, device="cuda"),      # wrong dtype
           torch.tensor([0, 1, 2], dtype=torch.int32)]                     # host tensor
    for t in bad:
        with pytest.raises(ValueError):
            net.template(z, slots=t)
        with pytest.raises(ValueError):
            net.step(x, bt.anchors, bt.window, tsz, 0.04, 0.4, slots=t)
    with pytest.raises(ValueError):                                        # template slots must be distinct
        net.template(z, slots=torch.tensor([1, 1, 2], dtype=torch.int32, device="cuda"))
    assert net.status() == 0


# ---------------------------------------------------------------------------------------------- 2. indexed crop
def test_indexed_crop_equals_gathered_crop():
    rng = np.random.RandomState(0)
    F, H, W = 4, 97, 131
    frames = torch.from_numpy(rng.randint(0, 256, (F, H, W, 3)).astype(np.uint8)).cuda()
    idx = np.array([3, 0, 3, 1, 2, 2])
    boxes = np.array([[rng.randint(-40, 100), rng.randint(-40, 80), rng.randint(20, 150)] + list(rng.randint(0, 256, 3))
                      for _ in idx], np.int32)
    want = crop_resize(frames[torch.from_numpy(idx).cuda()], boxes, 127)
    full = torch.zeros(len(idx), 8, dtype=torch.int32)
    full[:, :6] = torch.from_numpy(boxes)
    full = full.cuda()
    got = torch.empty_like(want)
    fi = torch.tensor(idx, dtype=torch.int32, device="cuda")
    lib = _lib.load()
    _lib.check(lib.sm_crop_resize_indexed(frames.data_ptr(), H * W * 3, H, W, fi.data_ptr(), full.data_ptr(), len(idx),
                                          127, got.data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.equal(got, want)


# ---------------------------------------------------------------------------------------------- 3. paste + labels
def _crop_back_map(cx, cy, s, W, H, side=127):
    """The forward map of crop_back (tools/test.py:263-275) for a square sub-window of size s at (cx, cy)."""
    sub = [cx - s / 2, cy - s / 2, s, s]
    k = side / sub[2]
    back = [-sub[0] * k, -sub[1] * k, W * k, H * k]
    a, b = (W - 1) / back[2], (H - 1) / back[3]
    return np.array([a, 0, -a * back[0], 0, b, -b * back[1]], np.float64)


def test_paste_labels_equals_fusion_over_warp_affine():
    rng = np.random.RandomState(1)
    G, H, W, side, thr = 3, 120, 200, 127, 0.3
    yy, xx = np.mgrid[0:side, 0:side]
    blobs = []
    for r in range(5):                                   # smooth blob-shaped sigmoid masks, values across 0..1
        c = rng.rand(2) * 60 + 33
        d = np.sqrt((yy - c[0]) ** 2 + (xx - c[1]) ** 2)
        blobs.append((1 / (1 + np.exp((d - 30) / 6))).astype(np.float32))
    blobs[2][60, 60:64] = np.float32(thr)                # values equal to float32(seg_thr)
    masks = np.stack(blobs)
    maps = np.stack([_crop_back_map(60, 50, 90, W, H), _crop_back_map(90, 70, 120, W, H),
                     _crop_back_map(150, 60, 70, W, H), _crop_back_map(-500, -400, 60, W, H),   # entirely off frame
                     _crop_back_map(100, 100, 200, W, H)])
    anno = rng.randint(0, 4, (G, H, W)).astype(np.uint8)
    anno[0, :40] = 0
    # video 0: tracked, overlapping tracked, init id 2; video 1: none; video 2: tie (same row twice), off-frame, idle,
    # init id 3, tracked
    objects = [[(OBJ_TRACKED, 0), (OBJ_TRACKED, 1), (OBJ_INIT, 2)], [],
               [(OBJ_TRACKED, 2), (OBJ_TRACKED, 2), (OBJ_TRACKED, 3), (OBJ_IDLE, 0), (OBJ_INIT, 3), (OBJ_TRACKED, 4)]]
    off = np.concatenate([[0], np.cumsum([len(o) for o in objects])])
    flat = [e for o in objects for e in o]
    md, mp = torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda()
    ad = torch.from_numpy(anno).cuda()
    got = paste_labels(md, mp, ad, off, flat, (H, W), thr).cpu().numpy()
    dev_warp = warp_affine(md, mp, (W, H), -1.0).cpu().numpy()
    for use_dev in (False, True):
        for g in range(G):
            vals = []
            for kind, arg in objects[g]:
                if kind == OBJ_TRACKED:
                    v = dev_warp[arg] if use_dev else cv2.warpAffine(masks[arg], maps[arg].reshape(2, 3), (W, H),
                                                                      flags=cv2.INTER_LINEAR,
                                                                      borderMode=cv2.BORDER_CONSTANT, borderValue=-1)
                elif kind == OBJ_INIT:
                    v = (anno[g] == arg).astype(np.float64)
                else:
                    v = np.full((H, W), -1.0)
                vals.append(np.asarray(v, np.float64))
            if vals:
                p = np.stack(vals)
                want = (np.argmax(p, 0).astype(np.uint8) + 1) * (np.max(p, 0) > thr).astype(np.uint8)
            else:
                want = np.zeros((H, W), np.uint8)
            np.testing.assert_array_equal(got[g], want, err_msg=f"video {g} (device warp: {use_dev})")
    assert (got[2] == 1).any() and not (got[2] == 2).any()             # the tie goes to the lower index
    assert (got[0] == 2).any() and (got[0] == 3).any()


# ---------------------------------------------------------------------------------------------- 4. label boxes
def test_label_boxes_equal_cv2_bounding_rect():
    rng = np.random.RandomState(2)
    G, H, W = 3, 70, 90
    anno = np.zeros((G, H, W), np.uint8)
    for g in range(G):
        for oid in range(1, 5):
            x0, y0 = rng.randint(0, W - 5), rng.randint(0, H - 5)
            anno[g, y0:y0 + rng.randint(1, 30), x0:x0 + rng.randint(1, 40)] = oid
        anno[g][rng.rand(H, W) < 0.01] = 5                                    # scattered pixels
    anno[1, :, 0] = 6; anno[1, 0, :] = 6; anno[2, -1, :] = 7; anno[2, :, -1] = 7     # touching the borders
    queries = [(g, i) for g in range(G) for i in range(0, 9)]
    got = label_boxes(torch.from_numpy(anno).cuda(), queries).cpu().numpy()
    for (g, i), b in zip(queries, got):
        assert tuple(b) == cv2.boundingRect((anno[g] == i).astype(np.uint8)), (g, i)


# ---------------------------------------------------------------------------------------------- 5. lifecycle
def _single_run(sd, frames, box, start, stop):
    net = _net(sd, 1, 1)
    bt = BatchTracker(net, _params()).init(frames[start][None], [box])
    out = {}
    for t in range(start + 1, stop):
        r = bt.track(frames[t][None])
        out[t] = (r.cpu(), r.mask[0].cpu().numpy())
    return out


def test_streams_join_and_leave(sd):
    T = 6
    vids = [make_frames(n=T, seed=s) for s in range(3)]
    frames = [np.stack([v[0][t] for v in vids], 0) for t in range(T)]     # [3,H,W,3] per time step
    net = _net(sd, 4, 4)
    bt = BatchTracker(net, _params())
    ids = {0: None, 1: None, 2: None}
    ids[0], ids[1] = bt.add(frames[0], [vids[0][1][0], vids[1][1][0]], frame_index=[0, 1])
    assert bt.slots == [0, 1]
    got = {0: {}, 1: {}, 2: {}}
    for t in range(1, T):
        if t == 2:
            bt.remove([ids[0]])                          # stream 0 leaves after frame 1
        r = bt.track(frames[t])
        c = r.cpu()
        for v, sid in ids.items():
            if sid in r.extras["ids"]:
                row = r.extras["ids"].index(sid)
                got[v][t] = ({k: c[k][row] for k in c}, r.mask[row].cpu().numpy())
        if t == 2:
            ids[2], = bt.add(frames[t], [vids[2][1][t]], frame_index=[2])    # stream 2 joins at frame 2
            assert bt.slots == [1, 0]                    # the freed slot is reused
    spans = {0: (0, 2), 1: (0, T), 2: (2, T)}
    for v, (s, e) in spans.items():
        ref = _single_run(sd, list(vids[v][0]), vids[v][1][s], s, e)
        assert sorted(got[v]) == sorted(ref), v
        for t in got[v]:
            a, m = got[v][t]
            b, mr = ref[t]
            np.testing.assert_allclose(a["target_pos"], b["target_pos"][0], rtol=0, atol=1e-5)
            np.testing.assert_allclose(a["target_sz"], b["target_sz"][0], rtol=1e-6, atol=0)
            assert (m != mr).mean() < 1e-3, (v, t)


# ---------------------------------------------------------------------------------------------- 6. end to end
class _NoSelect:
    """The engine behind the reference's plain model API only (numpy selection in ref_loop)."""
    def __init__(self, net):
        self._n = net
        self.anchors, self.anchor_num = net.anchors, net.anchor_num

    def template(self, z):
        return self._n.template(z)

    def track_mask(self, x):
        return self._n.track_mask(x)

    def track(self, x):
        return self._n.track(x)

    def track_refine(self, pos):
        return self._n.track_refine(pos)


def test_video_segmenter_equals_track_vos(sd):
    T = 8
    v0 = make_multi_frames(n=T, seed=0)
    v1 = make_multi_frames(n=T, seed=1, objects=[(2, 0, 5, (40.0, 40.0), (5.0, 4.0), (8, 7)),
                                                 (1, 3, T - 1, (220.0, 130.0), (-6.0, -2.0), (6, 6))])
    videos = [v0, v1]
    objs = [(g, oid, s, e) for g, (_, _, ol) in enumerate(videos) for (oid, s, e) in ol]
    net = _net(sd, 6, 6)
    seg = smb.VideoSegmenter(net, _params()).open(objs, num_frames=T)
    labels, pos = [], []
    for f in range(T):
        fr = np.stack([v[0][f] for v in videos])
        an = np.stack([v[1][f] for v in videos])
        labels.append(seg.frame(fr, an).cpu().numpy())
        pos.append(seg.state()["target_pos"])
    single = _NoSelect(_net(sd, 1, 1))
    k0 = 0
    for g, (frames, annos, ol) in enumerate(videos):
        fdev = [torch.from_numpy(f).cuda() for f in frames]
        _, lab, rpos = track_vos(single, fdev, [annos[s] for (_, s, _) in ol], [o[0] for o in ol],
                                 [o[1] for o in ol], [o[2] for o in ol], HP, HP["seg_thr"], device="cuda")
        for f in range(T):
            diff = (labels[f][g] != lab[f]).mean()
            assert diff < 1e-3, f"video {g} frame {f}: labels differ on {diff:.2e} of the pixels"
            for k in range(len(ol)):
                want, have = rpos[k, f], pos[f][k0 + k]
                assert np.isnan(want).all() == np.isnan(have).all(), (g, f, k)
                if not np.isnan(want).any():
                    np.testing.assert_allclose(have, want, rtol=0, atol=1e-5)
        k0 += len(ol)
    assert any((l[0] == 3).any() for l in labels) and any((l[1] == 2).any() for l in labels)


def test_video_segmenter_rejects_missing_ids(sd):
    frames, annos, _ = make_multi_frames(n=2)
    seg = smb.VideoSegmenter(_net(sd, 2, 2), _params()).open([(0, 9, 0)], num_frames=2)
    with pytest.raises(ValueError):
        seg.frame(frames[0][None], annos[0][None])


def test_paste_labels_more_objects_than_one_chunk():
    """One video with 70 objects (more than the kernel's 64-object shared-memory chunk) plus a second video, against the
    numpy float64 fusion over cv2.warpAffine; and the kernel's guard for more than 255 objects in a video."""
    rng = np.random.RandomState(4)
    H, W, side, thr = 64, 96, 127, 0.35
    n = 70
    masks = rng.rand(n, side, side).astype(np.float32)
    maps = np.stack([_crop_back_map(rng.rand() * W, rng.rand() * H, rng.rand() * 40 + 10, W, H) for _ in range(n)])
    anno = rng.randint(0, 3, (2, H, W)).astype(np.uint8)
    objects = [[(OBJ_TRACKED, k) for k in range(n)], [(OBJ_TRACKED, 5), (OBJ_INIT, 1)]]
    objects[0][66] = (OBJ_INIT, 2)                          # an init object in the second chunk
    off = np.concatenate([[0], np.cumsum([len(o) for o in objects])])
    md, mp = torch.from_numpy(masks).cuda(), torch.from_numpy(maps).cuda()
    got = paste_labels(md, mp, torch.from_numpy(anno).cuda(), off, [e for o in objects for e in o], (H, W),
                       thr).cpu().numpy()
    for g in range(2):
        vals = []
        for kind, arg in objects[g]:
            if kind == OBJ_TRACKED:
                vals.append(cv2.warpAffine(masks[arg], maps[arg].reshape(2, 3), (W, H), flags=cv2.INTER_LINEAR,
                                           borderMode=cv2.BORDER_CONSTANT, borderValue=-1).astype(np.float64))
            else:
                vals.append((anno[g] == arg).astype(np.float64))
        p = np.stack(vals)
        want = (np.argmax(p, 0).astype(np.uint8) + 1) * (np.max(p, 0) > thr).astype(np.uint8)
        np.testing.assert_array_equal(got[g], want, err_msg=f"video {g}")
    assert (got[0] > 64).any()                               # labels from the second chunk won somewhere
    # 256 objects in one video: the device offsets bypass the host check, the kernel labels the video 0
    many = torch.tensor([(OBJ_INIT, 1)] * 256, dtype=torch.int32, device="cuda")
    ones = torch.ones(1, H, W, dtype=torch.uint8, device="cuda")
    off_dev = torch.tensor([0, 256], dtype=torch.int32, device="cuda")
    from siammask_b200.ops import _paste_labels
    assert int(_paste_labels(None, None, ones, off_dev, many, (H, W), thr).max()) == 0


def test_video_segmenter_rejects_end_before_start(sd):
    seg = smb.VideoSegmenter(_net(sd, 2, 2), _params())
    with pytest.raises(ValueError, match="before start_frame"):
        seg.open([(0, 1, 3, 2)])
    seg.open([(0, 1, 3, 3)])                                 # an object that lives for its start frame only
