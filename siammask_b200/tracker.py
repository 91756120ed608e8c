"""Batched, device-resident tracker loop around the hot path (SURVEY §8f rows 1-3): N concurrent tracker streams advance
frame to frame without the host touching per-stream state.

What the reference does per frame on the host in numpy, for ONE stream (tools/test.py:172-315) — search-window
arithmetic, crop + resize, score/box post-processing + argmax, learning-rate update and clamping of the target state,
mask paste-back — runs here as a fixed sequence of kernels over all streams (C ABI in include/siammask_b200.h):

    sm_tracker_prepare      state -> crop boxes, target size in the crop, scale          (tools/test.py:180-198, 71-76)
    sm_crop_resize_ragged   uint8 frames -> f32 [N,3,S,S] search crops (cv2-exact)        (:67-110)
    sm_step_slots_hp        track_mask -> select -> track_refine                          (:201-261)
    sm_tracker_update_hp    winner box + score -> new state (lr, clamps), paste-back map  (:239-249, 263-282, 305-315)
    sm_warp_affine_ragged   127x127 sigmoid mask -> frame, threshold                      (:263-284)

The state (target_pos, target_sz, float64) lives on the device; a frame costs one small D2H copy only if the caller
asks for the numbers (`TrackResult.cpu()`).  The rotated box of the pasted masks (contours + minAreaRect, :285-303) is
`ops.rotated_box`, which `VotRunner(mask=True)` runs on every frame's packed masks.

Streams join and leave a running tracker: `add` templates new streams into free engine slots, `remove` frees them.  The
active streams are kept as compact rows (state, slot, frame index, hyper-parameters), and every frame runs exactly those
rows as one batch through the slot table and the per-stream (penalty_k, window_influence, lr) table
(`sm_step_slots_hp`, `sm_tracker_update_hp`) and the frame-index table (`sm_crop_resize_ragged`); the tables are
uploaded only when the set changes.  A stream's hyper-parameters default to the tracker's `TrackerParams`.  Each stream
reads one frame of the frames passed to `track`: its frame index, set by `add` (for `init`, stream i reads frame i; a
single [H,W,3] frame is shared by all streams).  `add_state` starts streams from the centre form siamese_init receives
(target_pos, target_sz), and `reinit` runs siamese_init again for running streams in their own slots (the VOT
protocol's restart after a failure) without changing the active set; all three template through `_template`.

The frames of a call always reach the kernels as a `Packed`: one device buffer plus an `sm_image_desc` table (offset,
h, w per frame), from which the crop and the paste-back read each stream's own frame.  A list of frames (numpy arrays
or CUDA tensors, any mix of sizes) is packed by `FramePacker.pack`; a [F,H,W,3] array or tensor (and a shared [H,W,3]
frame) is wrapped by `FramePacker.wrap` without a copy, under a table that is uploaded only when the shape changes.
Frames of different sizes therefore run in one batch.  A stream is bound to the size of the frame it was added from;
the per-stream (W, H) table that the state update clamps against holds it.

The arithmetic is pinned by `tests/test_batch_tracker.py` to the reference loop's golden trajectory and to
single-stream runs of the host restatement in `oracle/ref_loop.py`.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib, ops
from .anchors import cosine_window, generate_anchor


@dataclass
class TrackerParams:
    """Hyper-parameters of the loop: defaults of utils/tracker_config.py:10-21 overlaid with the `hp` block of
    experiments/siammask_sharp/config_davis.json."""
    instance_size: int = 255
    exemplar_size: int = 127
    total_stride: int = 8
    base_size: int = 8
    out_size: int = 127              # 127 with the refine module, 63 for the plain mask head
    context_amount: float = 0.5
    penalty_k: float = 0.04
    window_influence: float = 0.4
    lr: float = 1.0
    seg_thr: float = 0.35
    windowing: str = "cosine"

    @property
    def score_size(self) -> int:     # utils/tracker_config.py:46
        return (self.instance_size - self.exemplar_size) // self.total_stride + 1 + self.base_size

    def c_struct(self) -> _lib.SmTrackerHp:
        return _lib.SmTrackerHp(self.context_amount, self.penalty_k, self.window_influence, self.lr, self.exemplar_size,
                                self.instance_size, self.total_stride, self.base_size, self.out_size, 0)


IMAGE_DESC = np.dtype([("offset", "<i8"), ("h", "<i4"), ("w", "<i4")])      # sm_image_desc of include/siammask_b200.h


def upload(values, dtype, dev) -> torch.Tensor:
    """A small host table (list or array) as a device tensor of `dtype`, copied asynchronously from pinned memory: the
    copy queues without waiting for the device (a pageable copy would wait for the stream)."""
    host = torch.as_tensor(np.asarray(values)).to(dtype)
    if torch.device(dev).type == "cuda" and host.numel():
        host = host.pin_memory()
    return host.to(dev, non_blocking=True)


def image_table(shapes, channels: int) -> np.ndarray:
    """sm_image_desc rows of images packed back to back: shapes (h, w) per image, None for an empty entry (h = w = 0,
    occupying nothing); channels elements per pixel."""
    t = np.zeros(len(shapes), IMAGE_DESC)
    off = 0
    for i, s in enumerate(shapes):
        if s is not None:
            t[i] = (off, s[0], s[1])
            off += s[0] * s[1] * channels
    return t


@dataclass
class Packed:
    """Images of different sizes in one contiguous device buffer: data (flat, uint8 for frames and label maps), desc
    the device sm_image_desc table (raw bytes, one row per entry), shapes the host (h, w) per entry (None for a skipped
    entry), channels the elements per pixel."""
    data: torch.Tensor
    desc: torch.Tensor
    shapes: list
    channels: int
    table: np.ndarray

    def view(self, i: int) -> torch.Tensor:
        """Entry i as a [h,w,channels] (or [h,w] for one channel) view of the buffer."""
        h, w = self.shapes[i]
        o = int(self.table[i]["offset"])
        v = self.data[o:o + h * w * self.channels]
        return v.view(h, w, self.channels) if self.channels > 1 else v.view(h, w)


class FramePacker:
    """Packs lists of images that differ in size (uint8 numpy arrays or CUDA tensors, [h,w,3] frames or [h,w] label
    maps) into one device buffer plus an sm_image_desc table, and wraps same-size batches in place.  The table depends
    only on the sequence of shapes and is uploaded only when that changes, asynchronously from pinned memory, so packing
    never waits for the device.  Host arrays are concatenated on the host and copied in one transfer; CUDA tensors are
    concatenated on the device."""

    def __init__(self, dev):
        self.dev = dev
        self._tables: dict = {}                     # channels -> ((shapes, shared) key, device table, host table)

    def table(self, shapes, channels: int, shared: bool = False):
        """(device sm_image_desc table, host table) of `shapes` at `channels` elements per pixel; shared: every entry
        at offset 0 (one image that all entries read)."""
        return self._table(tuple(None if s is None else (int(s[0]), int(s[1])) for s in shapes), channels, shared)

    def _table(self, shapes: tuple, channels: int, shared: bool):
        key = (shapes, shared)
        hit = self._tables.get(channels)
        if hit is not None and hit[0] == key:
            return hit[1], hit[2]
        t = image_table(shapes, channels)
        if shared:
            t["offset"] = 0
        dev = upload(t.view(np.uint8).reshape(-1), torch.uint8, self.dev)
        self._tables[channels] = (key, dev, t)
        return dev, t

    def pack(self, images, channels: int = 3) -> Packed:
        """images: a list of uint8 [h,w,3] (channels 3) or [h,w] (channels 1) arrays / tensors, or None (skipped)."""
        if not isinstance(images, (list, tuple)):
            raise ValueError("expected a list of images")
        want = "[h,w,3]" if channels == 3 else "[h,w]"
        shapes, present = [], []
        for i, im in enumerate(images):
            if im is None:
                shapes.append(None)
                continue
            t = im if torch.is_tensor(im) else np.asarray(im)
            if t.dtype not in (np.uint8, torch.uint8):
                raise ValueError(f"image {i}: uint8 expected (frames are HWC BGR as cv2.imread returns them)")
            shape = tuple(int(v) for v in t.shape)
            if len(shape) != (3 if channels == 3 else 2) or (channels == 3 and shape[2] != 3) or min(shape[:2]) < 1:
                raise ValueError(f"image {i} must be {want} with h, w >= 1, got {shape}")
            shapes.append(shape[:2])
            present.append(t)
        desc, table = self.table(shapes, channels)
        if present and all(torch.is_tensor(t) and t.is_cuda for t in present):
            data = torch.cat([t.to(self.dev).reshape(-1) for t in present])
        elif present:
            host = np.concatenate([np.ascontiguousarray(t.cpu().numpy() if torch.is_tensor(t) else t).reshape(-1)
                                   for t in present])
            data = torch.from_numpy(host).to(self.dev)
        else:
            data = torch.zeros(1, dtype=torch.uint8, device=self.dev)
        return Packed(data, desc, shapes, channels, table)

    def wrap(self, images, channels: int = 3, shared: int | None = None) -> Packed:
        """A batch of same-size images as a `Packed` without a copy: images uint8 [F,h,w,3] (channels 3) or [F,h,w]
        (channels 1), a tensor or a numpy array (moved to the device once), whose flat storage becomes `data` under the
        table of F images back to back.  With shared=n, images is one [h,w,3] (or [h,w]) image that all n entries read
        (every offset 0).  No checks: the callers validate dtype and rank."""
        t = torch.as_tensor(images).to(self.dev).contiguous()
        if shared is None:
            n, h, w = (int(v) for v in t.shape[:3])
        else:
            n, (h, w) = int(shared), (int(v) for v in t.shape[:2])
        desc, table = self._table(((h, w),) * n, channels, shared is not None)      # no per-entry key building
        return Packed(t.reshape(-1), desc, [(h, w)] * n, channels, table)


@dataclass
class TrackResult:
    """Per-frame outputs, all on the device, one row per active stream in the order of `BatchTracker.ids`.  state f64
    [N,8] = x, y, w, h (new target_pos / target_sz), score, penalty, lr (from the stream's own lr), best index; mask:
    bool [N,H,W] frame-sized masks (or None), or, when the streams' frames differ in size, a list of N bool [H_i,W_i]
    views of one packed buffer in row order.  With mask=True, extras also holds "mask_prob" f32 [N,side,side] (sigmoid
    masks), "maps" f64 [N,6] (their paste-back maps, overwritten by the next frame) and "unclamped" f64 [N,4]
    (target_pos, target_sz before the frame clamps: the mask-mode fallback of tools/test.py:299-303); with paste=True
    also "packed_mask" = (flat bool buffer, device sm_image_desc table, (max h, max w)) of the pasted masks, which
    `ops._rotated_box` reads in place."""
    state: torch.Tensor
    mask: torch.Tensor | list | None = None
    extras: dict = field(default_factory=dict)

    def cpu(self):
        s = self.state.cpu().numpy()
        return {"target_pos": s[:, 0:2].copy(), "target_sz": s[:, 2:4].copy(), "score": s[:, 4].copy(),
                "best_id": s[:, 7].astype(np.int64)}


class BatchTracker:
    """Tracker streams on one engine.  `net` is a `siammask_b200.Custom` on a CUDA device; at most max_batch streams are
    active at once, in engine slots slot0 .. num_slots-1."""

    def __init__(self, net, params: TrackerParams | None = None, slot0: int = 0):
        self.net = net
        self.p = params or TrackerParams(instance_size=net.search_size)
        if self.p.instance_size != net.search_size:
            raise ValueError("tracker instance_size must equal the engine's search_size")
        self.slot0 = int(slot0)
        self.dev = net._device
        self.lib = _lib.load()
        R, A = self.p.score_size, net.anchor_num
        self.anchors = torch.from_numpy(generate_anchor(net.anchors, R)).to(self.dev)
        self.window = torch.from_numpy(cosine_window(R, A, self.p.windowing)).to(self.dev)
        self.hp = self.p.c_struct()
        self.packer = FramePacker(self.dev)
        self._next_id = 0
        self._clear()

    def _clear(self):
        self.N = 0
        self._ids: list[int] = []
        self._slots: list[int] = []
        self._fidx: list[int] = []
        self._hp: list[tuple[float, float, float]] = []
        self._size: list[tuple[int, int]] = []         # (H, W) of the frames each stream reads
        dev = self.dev
        self.state = torch.zeros(0, 4, dtype=torch.float64, device=dev)
        self.avg = torch.zeros(0, 3, dtype=torch.int32, device=dev)
        self.imsize = torch.zeros(0, 2, dtype=torch.int32, device=dev)

    @property
    def ids(self) -> list[int]:
        """Ids of the active streams, in the row order of every per-frame output."""
        return list(self._ids)

    @property
    def slots(self) -> list[int]:
        return list(self._slots)

    # ------------------------------------------------------------------ helpers
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream)

    def _input(self, frames, shared: int = 1) -> Packed:
        """The frames of a call as a `Packed`: a list (or tuple) of frames, which may differ in size, is packed (None
        entries skipped); a uint8 [F,H,W,3] array or tensor is moved to the device once and wrapped without a copy; a
        single [H,W,3] frame is wrapped as `shared` entries that all read it."""
        if isinstance(frames, Packed):
            return frames
        if isinstance(frames, (list, tuple)):
            return self.packer.pack(frames, 3)
        t = torch.as_tensor(frames)
        if t.dtype != torch.uint8:
            raise ValueError("frames must be uint8 HWC (BGR as cv2.imread returns them)")
        if t.dim() not in (3, 4) or t.shape[-1] != 3:
            raise ValueError(f"frames must be [H,W,3] or [F,H,W,3], got {tuple(t.shape)}")
        return self.packer.wrap(t, 3, shared if t.dim() == 3 else None)

    def _sizes_read(self, fr: Packed, src: list[int]) -> list:
        """(H, W) of the frame each of the streams reading frames `src` of `fr` gets; ValueError for a missing one."""
        n = len(fr.shapes)
        got = [fr.shapes[i] if 0 <= i < n else None for i in src]
        if None in got:
            raise ValueError(f"a stream reads frame {src[got.index(None)]}, but {n} frames were given "
                             "(or that entry is None)")
        return got

    def _check_sizes(self, fr: Packed, rows, src: list[int]):
        """A stream is bound to the frame size it was added with: ValueError when rows read frames of another size."""
        got, want = self._sizes_read(fr, src), [self._size[r] for r in rows]
        if got != want:                             # one comparison on the hot path; the loop only finds the culprit
            r, hw = next((r, hw) for r, hw, s in zip(rows, got, want) if hw != s)
            raise ValueError(f"frames must be {self._size[r][0]}x{self._size[r][1]} for stream {self._ids[r]}, "
                             f"got {hw[0]}x{hw[1]}")

    def _upload_tables(self):
        """Device copies of the active set (slot table, frame-index table) and per-frame work buffers; runs only when the
        set changes."""
        N, dev = self.N, self.dev
        self._slots_dev = upload(np.asarray(self._slots, np.int64).reshape(N), torch.int32, dev)
        self._fidx_dev = upload(np.asarray(self._fidx, np.int64).reshape(N), torch.int32, dev)
        self._max_fidx = max(self._fidx) if self._fidx else -1
        self._hp_dev = upload(np.asarray(self._hp, np.float64).reshape(N, 3), torch.float64, dev)
        self.boxes = torch.zeros(N, 8, dtype=torch.int32, device=dev)
        self.tsz = torch.zeros(N, 2, dtype=torch.float64, device=dev)
        self.aux = torch.zeros(N, 4, dtype=torch.float64, device=dev)
        self.maps = torch.zeros(N, 6, dtype=torch.float64, device=dev)
        self.imsize = upload(np.asarray([[w, h] for h, w in self._size], np.int64).reshape(N, 2), torch.int32, dev)
        self._mask_table = None                         # paste-back table, buffer length, grid; built on first use

    def _template(self, fr: Packed, src: list[int], state: torch.Tensor, slots: list[int]) -> torch.Tensor:
        """The template half of siamese_init (tools/test.py:142-155) for n streams: fr the frames on the device, src
        [n] the frame of `fr` each stream reads, state f64 [n,4] (target_pos, target_sz) exactly as siamese_init
        receives them, slots [n] the engine slots to write.  Returns the streams' avg_chans, int32 [n,3]."""
        n = len(src)
        src_dev = torch.tensor(src, dtype=torch.int32, device=self.dev)
        # avg_chans = np.mean(im, axis=(0, 1)); written into a uint8 image it truncates (:146, :89-100).
        # Sums of < 2^53 integers are exact in float64, so sum / n equals numpy's mean bit for bit.  Each frame is
        # reduced once: the entries of a shared frame have one offset.
        offset = [int(fr.table["offset"][i]) for i in src]
        uniq = sorted(set(offset))
        entry = dict(zip(offset, src))
        mean = torch.stack([fr.view(entry[o]).to(torch.float64).sum(dim=(0, 1))
                            / float(fr.shapes[entry[o]][0] * fr.shapes[entry[o]][1]) for o in uniq])
        where = torch.tensor([uniq.index(o) for o in offset], device=self.dev)
        avg = mean[where].to(torch.uint8).to(torch.int32).contiguous()
        # template window (:149-155): s_z = round(sqrt(wc_z * hc_z)), crop around target_pos, resize to 127
        sw, sh = state[:, 2], state[:, 3]
        wc_z = sw + self.p.context_amount * (sw + sh)
        hc_z = sh + self.p.context_amount * (sw + sh)
        s_z = torch.round(torch.sqrt(wc_z * hc_z))                  # half-to-even, like Python's round()
        c = (s_z + 1) / 2
        zb = torch.zeros(n, 8, dtype=torch.int32, device=self.dev)
        zb[:, 0] = torch.round(state[:, 0] - c).to(torch.int32)
        zb[:, 1] = torch.round(state[:, 1] - c).to(torch.int32)
        zb[:, 2] = s_z.to(torch.int32)
        zb[:, 3:6] = avg
        z = ops._crop_resize_ragged(fr.data, fr.desc, src_dev, zb, self.p.exemplar_size)
        self.net.template(z, slots=torch.tensor(slots, dtype=torch.int32, device=self.dev))
        return avg

    def _state(self, target_pos, target_sz) -> torch.Tensor:
        """f64 [n,4] device rows (target_pos, target_sz) from host or device [n,2] arrays, values unchanged."""
        t = [(v if torch.is_tensor(v) else torch.as_tensor(np.asarray(v, dtype=np.float64))).to(self.dev, torch.float64)
             for v in (target_pos, target_sz)]
        if t[0].numel() % 2 or t[0].numel() != t[1].numel():
            raise ValueError("target_pos and target_sz must both be [n, 2]")
        return torch.cat([t[0].reshape(-1, 2), t[1].reshape(-1, 2)], 1).contiguous()

    # ------------------------------------------------------------------ stream lifecycle
    @torch.no_grad()
    def add(self, frames, boxes_xywh, frame_index=None, hp=None) -> list[int]:
        """siamese_init (tools/test.py:132-169) for new streams, which join the running batch in free engine slots.
        frames: uint8 [F,H,W,3] (or one shared [H,W,3]); boxes_xywh: [n,4] top-left x, y, w, h of the targets;
        frame_index: [n] frame of `frames` each new stream reads, now and in every later `track` (default: stream i reads
        frame i); hp: [n,3] per-stream (penalty_k, window_influence, lr) (default: the tracker's `TrackerParams`).
        Returns the new streams' ids."""
        with torch.cuda.device(self.dev):
            bx = torch.as_tensor(np.asarray(boxes_xywh, dtype=np.float64)).reshape(-1, 4).to(self.dev)
            # target_pos = box centre, target_sz = (w, h)  (tools/test.py:338-339 / demo.py)
            state = torch.stack([bx[:, 0] + bx[:, 2] / 2, bx[:, 1] + bx[:, 3] / 2, bx[:, 2], bx[:, 3]], 1).contiguous()
            return self._join(frames, state, frame_index, hp)

    @torch.no_grad()
    def add_state(self, frames, target_pos, target_sz, frame_index=None, hp=None) -> list[int]:
        """`add` from the centre form siamese_init receives: target_pos, target_sz float64 [n,2] (host or device).  A
        box round trip is not exact ((cx - w/2) + w/2 need not be cx in float64) and the tracker amplifies the ulp, so
        callers that hold centre-form state (the VOT protocol's get_axis_aligned_bbox) start streams here."""
        with torch.cuda.device(self.dev):
            return self._join(frames, self._state(target_pos, target_sz), frame_index, hp)

    def _join(self, frames, state: torch.Tensor, frame_index, hp) -> list[int]:
        n = state.shape[0]
        idx = list(range(n)) if frame_index is None else [int(i) for i in np.asarray(frame_index).reshape(-1)]
        if len(idx) != n:
            raise ValueError("one frame index per new stream expected")
        fr = self._input(frames, max(idx, default=0) + 1)
        if any(i < 0 for i in idx):
            raise ValueError("frame indices must be >= 0")
        if any(i >= len(fr.shapes) for i in idx):
            raise ValueError(f"frame index out of range [0, {len(fr.shapes)})")
        if hp is None:
            rows = [(float(self.p.penalty_k), float(self.p.window_influence), float(self.p.lr))] * n
        else:
            h = np.asarray(hp.cpu() if torch.is_tensor(hp) else hp, dtype=np.float64)
            if h.shape != (n, 3):
                raise ValueError(f"hp must have shape [{n}, 3] (penalty_k, window_influence, lr), got {h.shape}")
            if not np.isfinite(h).all():
                raise ValueError("hp entries must be finite")
            rows = [tuple(float(v) for v in r) for r in h]
        used = set(self._slots)
        free = [s for s in range(self.slot0, self.net.num_slots) if s not in used][:n]
        if n == 0:
            return []
        if self.N + n > self.net.max_batch or len(free) < n:
            raise ValueError("more streams than the engine was built for")
        sizes = self._sizes_read(fr, idx)                          # each new stream is bound to its frame's size
        avg = self._template(fr, idx, state, free)
        ids = list(range(self._next_id, self._next_id + n))
        self._next_id += n
        self.state = torch.cat([self.state, state], 0).contiguous()
        self.avg = torch.cat([self.avg, avg], 0).contiguous()
        self._size += sizes
        self._ids += ids
        self._slots += free
        self._fidx += idx
        self._hp += rows
        self.N += n
        self._upload_tables()
        return ids

    @torch.no_grad()
    def reinit(self, ids, frames, target_pos, target_sz) -> None:
        """siamese_init again for running streams, in their own engine slots: the streams `ids` are templated from
        `frames` (read like `track` reads them: each stream its own frame index) at target_pos, target_sz float64 [n,2]
        (host or device), and their state rows are overwritten.  The set of active streams, their rows, slots, frame
        indices and hyper-parameters stay as they are, so no table is uploaded."""
        ids = [int(i) for i in np.asarray(ids).reshape(-1)]
        unknown = set(ids) - set(self._ids)
        if unknown:
            raise ValueError(f"unknown stream ids {sorted(unknown)}")
        if len(set(ids)) != len(ids):
            raise ValueError("stream ids must be unique")
        if not ids:
            return
        with torch.cuda.device(self.dev):
            rows = [self._ids.index(i) for i in ids]
            src = [self._fidx[r] for r in rows]
            fr = self._input(frames, max(src) + 1)
            self._check_sizes(fr, rows, src)
            state = self._state(target_pos, target_sz)
            if state.shape[0] != len(ids):
                raise ValueError(f"target_pos and target_sz must be [{len(ids)}, 2]")
            avg = self._template(fr, src, state, [self._slots[r] for r in rows])
            r_dev = torch.tensor(rows, dtype=torch.long, device=self.dev)
            self.state.index_copy_(0, r_dev, state)
            self.avg.index_copy_(0, r_dev, avg)

    @torch.no_grad()
    def set_frame_index(self, ids, frame_index) -> None:
        """Point running streams at other entries of the frame lists of later calls: stream ids[i] reads frame
        frame_index[i] from now on (a queue whose frame list changes as sequences come and go).  The frame-index table
        is uploaded only when an index changes, asynchronously from pinned memory, so the call never waits for the
        device; the active set and every other table stay as they are.  The size check of `track` still binds each
        stream to the size it was added with."""
        ids = [int(i) for i in np.asarray(ids).reshape(-1)]
        idx = [int(i) for i in np.asarray(frame_index).reshape(-1)]
        if len(idx) != len(ids):
            raise ValueError("one frame index per stream id expected")
        unknown = set(ids) - set(self._ids)
        if unknown:
            raise ValueError(f"unknown stream ids {sorted(unknown)}")
        if len(set(ids)) != len(ids):
            raise ValueError("stream ids must be unique")
        if any(i < 0 for i in idx):
            raise ValueError("frame indices must be >= 0")
        row = {i: r for r, i in enumerate(self._ids)}
        fidx = list(self._fidx)
        for i, v in zip(ids, idx):
            fidx[row[i]] = v
        if fidx == self._fidx:
            return
        self._fidx = fidx
        self._max_fidx = max(fidx)
        self._fidx_dev = upload(fidx, torch.int32, self.dev)

    @torch.no_grad()
    def remove(self, ids) -> None:
        """Stop tracking the given streams and free their engine slots (a later `add` may reuse them)."""
        drop = {int(i) for i in np.asarray(ids).reshape(-1)}
        unknown = drop - set(self._ids)
        if unknown:
            raise ValueError(f"unknown stream ids {sorted(unknown)}")
        if not drop:
            return
        keep = [r for r, i in enumerate(self._ids) if i not in drop]
        with torch.cuda.device(self.dev):
            rows = upload(np.asarray(keep, np.int64), torch.long, self.dev)
            self.state = self.state.index_select(0, rows).contiguous()
            self.avg = self.avg.index_select(0, rows).contiguous()
            self._ids = [self._ids[r] for r in keep]
            self._size = [self._size[r] for r in keep]
            self._slots = [self._slots[r] for r in keep]
            self._fidx = [self._fidx[r] for r in keep]
            self._hp = [self._hp[r] for r in keep]
            self.N = len(keep)
            self._upload_tables()

    # ------------------------------------------------------------------ siamese_init (tools/test.py:132-169)
    @torch.no_grad()
    def init(self, frames, boxes_xywh):
        """Start over with N streams in slots slot0 .. slot0+N-1.  frames: uint8 [N,H,W,3] (or one shared [H,W,3], or a
        list of N frames that may differ in size); boxes_xywh: [N,4] top-left x, y, w, h of the targets.  Stream i reads frame i of later per-stream frame tensors."""
        n = np.asarray(boxes_xywh).reshape(-1, 4).shape[0]
        if n > self.net.max_batch or self.slot0 + n > self.net.num_slots:
            raise ValueError("more streams than the engine was built for")
        self._clear()
        self.add(frames, boxes_xywh, frame_index=range(n))
        return self

    # ------------------------------------------------------------------ siamese_track (tools/test.py:172-315)
    @torch.no_grad()
    def track(self, frames, mask: bool = True, refine: bool = True, paste: bool = True) -> TrackResult:
        """Advance all active streams by one frame.  mask=True computes the (refined) mask; with paste=True it is pasted
        back into the frame and thresholded at seg_thr.  refine=False uses the 63x63 mask head column instead of the
        refine module (tools/test.py:256-260)."""
        if self.N == 0:
            raise RuntimeError("no active streams: call init() or add() first")
        p, N = self.p, self.N
        with torch.cuda.device(self.dev):
            fr = self._input(frames, self._max_fidx + 1)
            self._check_sizes(fr, range(N), self._fidx)
            st = self._stream()
            _lib.check(self.lib.sm_tracker_prepare(N, self.state.data_ptr(), self.avg.data_ptr(), C.byref(self.hp),
                                                   self.boxes.data_ptr(), self.tsz.data_ptr(), self.aux.data_ptr(), st))
            x = ops._crop_resize_ragged(fr.data, fr.desc, self._fidx_dev, self.boxes, p.instance_size)
            use_refine = mask and refine
            use_head = mask and not refine
            out = self.net._step(x, self.anchors, self.window, self.tsz, p.penalty_k, p.window_influence,
                                 refine=use_refine, mask_head=use_head, mask_col=use_head, slots=self._slots_dev,
                                 hp=self._hp_dev)
            res = torch.empty(N, 8, dtype=torch.float64, device=self.dev)
            unclamped = torch.empty(N, 4, dtype=torch.float64, device=self.dev) if mask else None
            _lib.check(self.lib.sm_tracker_update_hp_ex(N, self.state.data_ptr(), out["records"].data_ptr(),
                                                        self.aux.data_ptr(), self.imsize.data_ptr(), C.byref(self.hp),
                                                        self._hp_dev.data_ptr(), self.net.anchor_num, p.score_size,
                                                        self.maps.data_ptr() if mask else None, res.data_ptr(),
                                                        unclamped.data_ptr() if mask else None, st))
            extras = {"records": out["records"], "pos": out["pos"], "x_crop": x, "ids": list(self._ids)}
            mask_out = None
            if mask:
                logits = out["refine"] if use_refine else out["mask_col"]
                side = 127 if use_refine else 63
                if side != p.out_size:
                    raise ValueError(f"out_size {p.out_size} does not match the mask source ({side})")
                m = logits.sigmoid().view(N, side, side).contiguous()
                extras["mask_prob"], extras["maps"], extras["unclamped"] = m, self.maps, unclamped
                if paste:                                   # every row's mask in one packed buffer
                    if self._mask_table is None:
                        desc, table = self.packer.table(self._size, 1)
                        hs, ws = zip(*self._size)
                        self._mask_table = desc, table, int(table["offset"][-1]) + hs[-1] * ws[-1], (max(hs), max(ws))
                    desc, table, total, max_hw = self._mask_table
                    flat = ops._warp_affine_ragged(m, self.maps, desc, max_hw, total) > p.seg_thr
                    extras["packed_mask"] = (flat, desc, max_hw)
                    if len(set(self._size)) == 1:                  # one frame size: rows back to back, [N,H,W]
                        mask_out = flat.view(N, *max_hw)
                    else:
                        mask_out = [flat[int(o):int(o) + h * w].view(h, w)
                                    for o, (h, w) in zip(table["offset"], self._size)]
            return TrackResult(state=res, mask=mask_out, extras=extras)
