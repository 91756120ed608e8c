"""Drop-in replacement for the reference's `Custom` model object (experiments/siammask_sharp/custom.py:162-190,
experiments/siamrpn_resnet/custom.py:81-93) as used by the tracker loop in tools/test.py:

    siamese_init  :155       net.template(z)
    siamese_track :201,203   net.track_mask(x) / net.track(x)
    siamese_track :257       net.track_refine((delta_y, delta_x))
    siamese_init  :137,142-145   net.anchors, net.anchor_num
    main          :560-569   Custom(anchors=cfg['anchors']); load_pretrain(model, path); model.eval().to(device)

Python here is plumbing only: tensors in, tensors out, every FLOP happens in libsiammask_b200.so
(hand-written sm_90a kernels) reached through the C ABI in include/siammask_b200.h.

Batched extension (not in the reference, SURVEY §8b): every method accepts B>1 *paired* templates/searches
bound to engine slots slot0..slot0+B-1, and `track_refine` additionally accepts an int tensor/array [B,2]
of per-stream positions (the reference applies one (dy,dx) to the whole batch, custom.py:131-135).
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .checkpoint import expected_keys, normalize_keys

DEFAULT_ANCHORS = {"stride": 8, "ratios": [0.33, 0.5, 1, 2, 3], "scales": [8], "round_dight": 0}


class Custom:
    def __init__(self, pretrain: bool = False, anchors: dict | None = None, *, search_size: int = 255,
                 max_batch: int = 1, num_slots: int | None = None, precision: str = "exact",
                 backend: str = "tensor", mask: bool = True, graphs: bool = False, **_unused):
        self.anchors = anchors if anchors is not None else dict(DEFAULT_ANCHORS)      # siammask_sharp.py:16
        self.anchor_num = len(self.anchors["ratios"]) * len(self.anchors["scales"])   # siammask_sharp.py:17
        self.search_size = int(search_size)
        self.max_batch = int(max_batch)
        self.num_slots = int(num_slots) if num_slots is not None else self.max_batch
        self.precision = {"exact": _lib.SM_PRECISION_EXACT, "fast": _lib.SM_PRECISION_FAST}[precision]
        self.backend = {"tensor": _lib.SM_BACKEND_TENSOR, "simt": _lib.SM_BACKEND_SIMT}[backend]
        self.with_mask = bool(mask)
        self.graphs = bool(graphs)          # CUDA-graph replay: persistent I/O buffers, outputs overwritten per call
        self._io: dict = {}
        self.score_size = (self.search_size - 127) // 8 + 1 + 8            # utils/tracker_config.py:23
        self.training = False
        self._sd: dict[str, torch.Tensor] | None = None
        self._engine = C.c_void_p(None)
        self._device: torch.device | None = None
        self._lib = _lib.load()

    # ------------------------------------------------------------------ nn.Module protocol subset
    def state_dict(self):
        if self._sd is not None:
            return OrderedDict(self._sd)
        return OrderedDict((k, torch.empty(s, device="meta")) for k, s in
                           expected_keys(self.with_mask, self.with_mask).items())

    def load_state_dict(self, state_dict, strict: bool = False):
        """strict=False mirrors the reference (utils/load_helper.py:53 -> nn.Module.load_state_dict(strict=False)):
        tensors the checkpoint lacks keep the values of a freshly constructed module (here: the seeded random init
        of `checkpoint.synthetic_state_dict`) and are reported with a warning; unexpected keys are ignored.  At least
        one key must match (load_helper.py:19 asserts the same).  strict=True raises KeyError on any missing key."""
        sd = normalize_keys(state_dict)
        want = expected_keys(self.with_mask, self.with_mask)
        missing = [k for k in want if k not in sd]
        if len(missing) == len(want):
            raise AssertionError("load NONE from pretrained checkpoint")             # load_helper.py:19
        if missing:
            if strict:
                raise KeyError(f"checkpoint lacks {len(missing)} tensors needed on the hot path, e.g. {missing[:3]}")
            import warnings
            from .checkpoint import synthetic_state_dict
            warnings.warn(f"checkpoint lacks {len(missing)} hot-path tensors (e.g. {missing[:3]}): they keep their "
                          "initial values, as with the reference's strict=False load", RuntimeWarning)
            init = synthetic_state_dict(0, self.with_mask, self.with_mask)
            sd = dict(sd)
            for k in missing:
                sd[k] = init[k]
        for k, shp in want.items():
            if tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != expected {tuple(shp)}")
        self._sd = {k: sd[k].detach().to("cpu", torch.float32).contiguous() for k in want}
        if self._engine.value:
            self._upload()
        return self

    def eval(self):
        self.training = False
        return self

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("siammask_b200 implements the inference path only")
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", torch.cuda.current_device() if device is None else device))

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("siammask_b200 runs on CUDA (sm_90a) devices only; there is no CPU path")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if self._engine.value and self._device == device:
            return self
        self._destroy()
        self._device = device
        with torch.cuda.device(device):
            cfg = _lib.SmConfig(self.search_size, self.max_batch, self.num_slots, self.precision, self.backend,
                                self.anchor_num, int(self.with_mask))
            _lib.check(self._lib.sm_engine_create(C.byref(cfg), C.byref(self._engine)))
            _lib.check(self._lib.sm_engine_set_graphs(self._engine, int(self.graphs)))
            self._io = {}
            self._gstream = torch.cuda.Stream(device) if self.graphs else None
            if self._sd is not None:
                self._upload()
        return self

    # ------------------------------------------------------------------ weights
    def _upload(self):
        descs = (_lib.SmTensorDesc * len(self._sd))()
        keep = []
        for i, (k, t) in enumerate(self._sd.items()):
            name = k.encode()
            keep.append(name)
            descs[i].name = name
            descs[i].data = t.data_ptr()
            descs[i].ndim = t.dim()
            for j, s in enumerate(t.shape):
                descs[i].shape[j] = s
        with torch.cuda.device(self._device):
            _lib.check(self._lib.sm_engine_load_weights(self._engine, descs, len(self._sd)))

    def weight_blob(self) -> torch.Tensor:
        """uint8 CUDA view of the engine's packed weight arena (for the one-off NCCL broadcast)."""
        ptr, n = C.c_void_p(), C.c_size_t()
        _lib.check(self._lib.sm_engine_weight_blob(self._engine, C.byref(ptr), C.byref(n)))

        class _Arena:
            __cuda_array_interface__ = {"shape": (n.value,), "typestr": "|u1", "data": (ptr.value, False),
                                        "version": 2}
        t = torch.as_tensor(_Arena(), device=self._device)
        t._sm_owner = self           # keep the engine alive while the view exists
        return t

    def adopt_weights(self):
        _lib.check(self._lib.sm_engine_adopt_weights(self._engine))

    @torch.no_grad()
    def calibrate(self, z, x):
        """Pick static power-of-two activation scales from a representative sample (z [B,3,127,127], x [B,3,S,S], raw
        0..255 crops; engine slots 0..B-1 are overwritten).  Results are unchanged for well-scaled checkpoints; it
        is what keeps checkpoints whose activations sit far from O(1) inside the fp16 split format's range."""
        z, x = self._prep(z, 127), self._prep(x, self.search_size)
        if z.shape[0] != x.shape[0]:
            raise ValueError("paired sample batch expected")
        with torch.cuda.device(self._device):
            self._fence_in()
            _lib.check(self._lib.sm_engine_calibrate(self._engine, z.shape[0], z.data_ptr(), x.data_ptr(), self._stream()))
            self._fence_out()
        return self

    def status(self) -> int:
        """Synchronises; bit 0 set = an activation left fp16's range (call `calibrate`)."""
        v = C.c_int32()
        _lib.check(self._lib.sm_engine_status(self._engine, C.byref(v)))
        return int(v.value)

    # packed-weight file (SURVEY §8f row 4): BN-folded, repacked, fp16-split arena exactly as it sits in HBM, so a
    # fleet of ranks loads (or receives by broadcast) the blob instead of re-folding the 21 M-parameter checkpoint
    # the version digit moves with the arena layout, so a file of another layout is rejected by name, not by size
    _PACK_MAGIC = b"SMB200PK2"

    def _pack_tag(self) -> bytes:
        return ("%d,%d,%d,%d" % (self.search_size, self.precision, self.anchor_num, int(self.with_mask))).encode()

    def save_packed(self, path: str):
        blob = self.weight_blob()
        torch.cuda.synchronize(self._device)
        with open(path, "wb") as f:
            tag = self._pack_tag()
            f.write(self._PACK_MAGIC + len(tag).to_bytes(4, "little") + tag + blob.numel().to_bytes(8, "little"))
            f.write(blob.cpu().numpy().tobytes())

    def load_packed(self, path: str):
        if not self._engine.value:
            raise RuntimeError("call .to(cuda device) first")
        with open(path, "rb") as f:
            magic = f.read(len(self._PACK_MAGIC))
            if magic != self._PACK_MAGIC:
                if magic.startswith(self._PACK_MAGIC[:-1]):
                    raise ValueError(f"packed-weight file of another arena layout ({magic!r}; this engine reads "
                                     f"{self._PACK_MAGIC!r}): pack the weights again")
                raise ValueError("not a siammask_b200 packed-weight file")
            tag = f.read(int.from_bytes(f.read(4), "little"))
            n = int.from_bytes(f.read(8), "little")
            blob = self.weight_blob()
            # the arena layout depends on anchor_num / with_mask only; precision and search size are recorded for
            # information (both precisions read the same hi/lo planes)
            if tag.split(b",")[2:] != self._pack_tag().split(b",")[2:] or n != blob.numel():
                raise ValueError(f"packed weights were written for a different engine configuration ({tag!r})")
            data = np.frombuffer(f.read(n), dtype=np.uint8)
        blob.copy_(torch.from_numpy(data.copy()))
        torch.cuda.synchronize(self._device)
        self.adopt_weights()
        return self

    # ------------------------------------------------------------------ the tracker-facing API
    def _prep(self, t: torch.Tensor, size: int) -> torch.Tensor:
        if not self._engine.value:
            raise RuntimeError("call .to(cuda device) (and load weights) before inference")
        if t.dim() != 4 or t.shape[1] != 3 or t.shape[2] != size or t.shape[3] != size:
            raise ValueError(f"expected [B,3,{size},{size}], got {tuple(t.shape)}")
        if t.shape[0] > self.max_batch:
            raise ValueError(f"batch {t.shape[0]} > max_batch {self.max_batch}")
        t = t.to(self._device, torch.float32).contiguous()
        if self.graphs:                      # graph replay needs stable addresses: stage into a persistent buffer
            buf = self._buf(("in", size, t.shape[0]), t.shape, torch.float32)
            buf.copy_(t)
            return buf
        return t

    def _buf(self, key, shape, dtype):
        if not self.graphs:
            return torch.empty(*shape, device=self._device, dtype=dtype)
        b = self._io.get(key)
        if b is None:
            b = self._io[key] = torch.empty(*shape, device=self._device, dtype=dtype)
        return b

    def _stream(self):
        """Stream the engine call is enqueued on.  Graph capture is impossible on the legacy default stream, so in
        graph mode the work runs on a private stream fenced against the caller's current stream on both sides
        (`_fence_in` before the call, `_fence_out` after)."""
        if self.graphs:
            return C.c_void_p(self._gstream.cuda_stream)
        return C.c_void_p(torch.cuda.current_stream(self._device).cuda_stream)

    def _fence_in(self):
        if self.graphs:
            self._gstream.wait_stream(torch.cuda.current_stream(self._device))

    def _fence_out(self):
        if self.graphs:
            torch.cuda.current_stream(self._device).wait_stream(self._gstream)

    def _check_slots(self, slots, B: int, distinct: bool) -> torch.Tensor:
        """A slot table: int32 CUDA tensor [B] with entries in [0, num_slots) (distinct for template).  The check reads
        the table back to the host, so it runs before anything is enqueued."""
        if not (isinstance(slots, torch.Tensor) and slots.is_cuda and slots.dtype == torch.int32):
            raise ValueError("slots must be an int32 CUDA tensor")
        if slots.device != self._device:
            raise ValueError(f"slots live on {slots.device}, the engine on {self._device}")
        if slots.dim() != 1 or slots.numel() != B:
            raise ValueError(f"slots must have shape [{B}], got {tuple(slots.shape)}")
        host = slots.cpu().numpy()
        if ((host < 0) | (host >= self.num_slots)).any():
            raise ValueError(f"slot table entries must lie in [0, {self.num_slots})")
        if distinct and np.unique(host).size != B:
            raise ValueError("slot table entries must be distinct")
        return slots.contiguous()

    def _stage_slots(self, slots: torch.Tensor) -> torch.Tensor:
        """Graph replay reads the table at a stable address: copy it there on the caller's stream.  Call before
        `_fence_in`, so that the engine's stream is ordered after the copy."""
        if self.graphs:
            buf = self._buf(("slots", slots.numel()), (slots.numel(),), torch.int32)
            buf.copy_(slots)
            return buf
        return slots

    def _check_hp(self, hp, B: int) -> torch.Tensor:
        """A per-stream hyper-parameter table: float64 CUDA tensor [B,3] of finite (penalty_k, window_influence, lr)
        rows.  The finiteness check reads the table back to the host, so it runs before anything is enqueued."""
        if not (isinstance(hp, torch.Tensor) and hp.is_cuda and hp.dtype == torch.float64):
            raise ValueError("hp must be a float64 CUDA tensor")
        if hp.device != self._device:
            raise ValueError(f"hp lives on {hp.device}, the engine on {self._device}")
        if tuple(hp.shape) != (B, 3):
            raise ValueError(f"hp must have shape [{B}, 3], got {tuple(hp.shape)}")
        if not bool(torch.isfinite(hp).all()):
            raise ValueError("hp entries must be finite")
        return hp.contiguous()

    def _stage_hp(self, hp: torch.Tensor) -> torch.Tensor:
        """`_stage_slots` for the hyper-parameter table."""
        if self.graphs:
            buf = self._buf(("hp", hp.shape[0]), tuple(hp.shape), torch.float64)
            buf.copy_(hp)
            return buf
        return hp

    @torch.no_grad()
    def template(self, z, slot0: int = 0, slots=None):
        """slots (optional): int32 CUDA tensor [B] of distinct engine slots; stream b's template is cached in slots[b]
        instead of slot0 + b."""
        if slots is not None:
            slots = self._check_slots(slots, z.shape[0], distinct=True)
        z = self._prep(z, 127)
        with torch.cuda.device(self._device):
            if slots is not None:
                slots = self._stage_slots(slots)
            self._fence_in()
            if slots is None:
                _lib.check(self._lib.sm_template(self._engine, slot0, z.shape[0], z.data_ptr(), self._stream()))
            else:
                _lib.check(self._lib.sm_template_slots(self._engine, z.shape[0], slots.data_ptr(), z.data_ptr(),
                                                       self._stream()))
            self._fence_out()
        self._keep_slots = slots

    def _track(self, x, slot0, flags):
        x = self._prep(x, self.search_size)
        B, A, R = x.shape[0], self.anchor_num, self.score_size
        cls = self._buf(("cls", B), (B, 2 * A, R, R), torch.float32)
        loc = self._buf(("loc", B), (B, 4 * A, R, R), torch.float32)
        mask = None
        if flags & _lib.SM_TRACK_MASK_HEAD:
            mask = self._buf(("mask", B), (B, 63 * 63, R, R), torch.float32)
        with torch.cuda.device(self._device):
            self._fence_in()
            _lib.check(self._lib.sm_track(self._engine, slot0, B, x.data_ptr(), cls.data_ptr(), loc.data_ptr(),
                                          mask.data_ptr() if mask is not None else None, flags, self._stream()))
            self._fence_out()
        self._last_B = B
        return cls, loc, mask

    @torch.no_grad()
    def track(self, x, slot0: int = 0):
        cls, loc, _ = self._track(x, slot0, 0)
        return cls, loc

    @torch.no_grad()
    def track_mask(self, x, slot0: int = 0, mask_head: bool = True):
        """mask_head=False skips the 256->3969 head, which tools/test.py:256-258 discards under --refine."""
        flags = _lib.SM_TRACK_MASK_FEATURES | (_lib.SM_TRACK_MASK_HEAD if mask_head else 0)
        return self._track(x, slot0, flags)

    @torch.no_grad()
    def track_refine(self, pos):
        B = self._last_B
        R = self.score_size
        if isinstance(pos, torch.Tensor) and pos.is_cuda:
            p = pos.to(self._device, torch.int32).reshape(-1, 2)     # device tensor: no host sync, caller's contract
        else:
            host = np.asarray(pos.cpu() if isinstance(pos, torch.Tensor) else pos, dtype=np.int64).reshape(-1, 2)
            if ((host < 0) | (host >= R)).any():
                raise IndexError(f"refine position out of range [0,{R})")
            p = torch.as_tensor(host.astype(np.int32), device=self._device)
        if p.shape[0] == 1 and B > 1:
            p = p.expand(B, 2)
        p = p.contiguous()
        if p.shape[0] != B:
            raise ValueError(f"pos has {p.shape[0]} rows, last track had batch {B}")
        if self.graphs:
            pb = self._buf(("pos", B), (B, 2), torch.int32)
            pb.copy_(p)
            p = pb
        out = self._buf(("refine", B), (B, 127 * 127), torch.float32)
        with torch.cuda.device(self._device):
            self._fence_in()
            _lib.check(self._lib.sm_refine(self._engine, B, p.data_ptr(), out.data_ptr(), self._stream()))
            self._fence_out()
        return out

    @torch.no_grad()
    def select(self, cls, loc, anchors, window, target_sz_in_crop, penalty_k: float, window_influence: float):
        """On-device restatement of tools/test.py:205-254.  cls/loc: outputs of track/track_mask; anchors f32
        [A*R*R,4] (cx,cy,w,h) and window [A*R*R] as built by siamese_init (used in float64, as the reference's
        np.hanning window is); target_sz_in_crop [B,2] (used in float64).
        Returns (best_idx int32 [B], pos int32 [B,2] = (delta_y, delta_x), records f32 [B,8])."""
        B = cls.shape[0]
        dev = self._device
        anchors = anchors.to(dev, torch.float32).contiguous()
        window = window.to(dev, torch.float64).contiguous()
        tsz = torch.as_tensor(target_sz_in_crop).to(dev, torch.float64).reshape(B, 2).contiguous()
        n = self.anchor_num * self.score_size ** 2
        if anchors.shape != (n, 4) or window.numel() != n:
            raise ValueError(f"anchors/window must have {n} entries")
        best = torch.empty(B, dtype=torch.int32, device=dev)
        pos = torch.empty(B, 2, dtype=torch.int32, device=dev)
        rec = torch.empty(B, 8, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            self._fence_in()
            _lib.check(self._lib.sm_select(self._engine, B, cls.data_ptr(), loc.data_ptr(), anchors.data_ptr(),
                                           window.data_ptr(), tsz.data_ptr(), float(penalty_k),
                                           float(window_influence), best.data_ptr(), pos.data_ptr(), rec.data_ptr(),
                                           self._stream()))
            self._fence_out()
        return best, pos, rec

    @torch.no_grad()
    def step(self, x, anchors, window, target_sz_in_crop, penalty_k: float, window_influence: float, slot0: int = 0,
             refine: bool = True, mask_head: bool = False, mask_col: bool = False, slots=None, hp=None):
        """One whole frame of siamese_track (tools/test.py:201-261) in ONE engine call (C ABI `sm_step`):
        track(_mask) -> on-device selection -> track_refine at the selected position.  Returns a dict with cls, loc,
        mask (raw head or None), best, pos, records, refine (or None), mask_col (or None).  slots (optional): int32
        CUDA tensor [B]; stream b then uses the template cached in slots[b] (`sm_step_slots`) instead of slot0 + b.
        hp (optional): float64 CUDA tensor [B,3] of per-stream (penalty_k, window_influence, lr); stream b's selection
        then uses row b instead of the two scalars (`sm_step_slots_hp`; without `slots` the table is slot0 + b)."""
        B = x.shape[0]
        if slots is not None:
            slots = self._check_slots(slots, B, distinct=False)
        if hp is not None:
            hp = self._check_hp(hp, B)
            if slots is None:
                if slot0 < 0 or slot0 + B > self.num_slots:
                    raise ValueError(f"slots {slot0}..{slot0 + B - 1} outside [0, {self.num_slots})")
                slots = torch.arange(slot0, slot0 + B, dtype=torch.int32, device=self._device)
        return self._step(x, anchors, window, target_sz_in_crop, penalty_k, window_influence, slot0, refine, mask_head,
                          mask_col, slots, hp)

    def _step(self, x, anchors, window, target_sz_in_crop, penalty_k, window_influence, slot0=0, refine=True,
              mask_head=False, mask_col=False, slots=None, hp=None):
        """`step` without the host-side checks of `slots` and `hp` (callers that own tables they have validated;
        `hp` needs `slots`)."""
        x = self._prep(x, self.search_size)
        dev = self._device
        B, A, R = x.shape[0], self.anchor_num, self.score_size
        n = A * R * R
        anchors = anchors.to(dev, torch.float32).contiguous()
        window = window.to(dev, torch.float64).contiguous()
        if anchors.shape != (n, 4) or window.numel() != n:
            raise ValueError(f"anchors/window must have {n} entries")
        tsz = torch.as_tensor(target_sz_in_crop).to(dev, torch.float64).reshape(B, 2).contiguous()
        flags = (_lib.SM_TRACK_MASK_FEATURES if (refine or mask_head) else 0) | (_lib.SM_TRACK_MASK_HEAD if mask_head else 0)
        out = {"cls": self._buf(("cls", B), (B, 2 * A, R, R), torch.float32),
               "loc": self._buf(("loc", B), (B, 4 * A, R, R), torch.float32),
               "mask": self._buf(("mask", B), (B, 63 * 63, R, R), torch.float32) if mask_head else None,
               "best": self._buf(("best", B), (B,), torch.int32), "pos": self._buf(("spos", B), (B, 2), torch.int32),
               "records": self._buf(("rec", B), (B, 8), torch.float32),
               "refine": self._buf(("refine", B), (B, 127 * 127), torch.float32) if refine else None,
               "mask_col": self._buf(("mcol", B), (B, 63 * 63), torch.float32) if (mask_col and mask_head) else None}
        if self.graphs:
            tb = self._buf(("tsz", B), (B, 2), torch.float64)
            tb.copy_(tsz)
            tsz = tb

        def ptr(t):
            return t.data_ptr() if t is not None else None
        outs = (ptr(out["cls"]), ptr(out["loc"]), ptr(out["mask"]), ptr(out["best"]), ptr(out["pos"]),
                ptr(out["records"]), ptr(out["refine"]), ptr(out["mask_col"]), self._stream())
        with torch.cuda.device(dev):
            if slots is not None:
                slots = self._stage_slots(slots)
            if hp is not None:
                hp = self._stage_hp(hp)
            self._fence_in()
            if hp is not None:
                _lib.check(self._lib.sm_step_slots_hp(self._engine, B, slots.data_ptr(), hp.data_ptr(), x.data_ptr(),
                                                      tsz.data_ptr(), anchors.data_ptr(), window.data_ptr(), flags,
                                                      *outs))
            elif slots is None:
                _lib.check(self._lib.sm_step(self._engine, slot0, B, x.data_ptr(), tsz.data_ptr(), anchors.data_ptr(),
                                             window.data_ptr(), float(penalty_k), float(window_influence), flags, *outs))
            else:
                _lib.check(self._lib.sm_step_slots(self._engine, B, slots.data_ptr(), x.data_ptr(), tsz.data_ptr(),
                                                   anchors.data_ptr(), window.data_ptr(), float(penalty_k),
                                                   float(window_influence), flags, *outs))
            self._fence_out()
        self._last_B = B
        self._keep = (anchors, window, tsz, slots, hp)   # alive until the next call (the work is asynchronous)
        return out

    # ------------------------------------------------------------------ introspection used by tests / bench
    def export(self, what: str) -> torch.Tensor:
        shape = (C.c_int64 * 4)()
        with torch.cuda.device(self._device):
            _lib.check(self._lib.sm_export(self._engine, what.encode(), None, shape, self._stream()))
            out = torch.empty(*[int(s) for s in shape], device=self._device, dtype=torch.float32)
            self._fence_in()
            _lib.check(self._lib.sm_export(self._engine, what.encode(), out.data_ptr(), shape, self._stream()))
            self._fence_out()
        return out

    def profile(self, on: bool):
        _lib.check(self._lib.sm_profile_enable(self._engine, int(on)))

    def profile_dump(self):
        """-> list of (name, category, ms, flops, bytes) for every launch since profiling was enabled."""
        n = int(self._lib.sm_profile_dump(self._engine, None, 0))
        if n < 0:
            _lib.check(-1)
        buf = C.create_string_buffer(n + 16)
        if int(self._lib.sm_profile_dump(self._engine, buf, n + 16)) < 0:
            _lib.check(-1)
        rows = []
        for line in buf.value.decode().splitlines():
            name, cat, ms, fl, by = line.split("\t")
            rows.append((name, cat, float(ms), float(fl), float(by)))
        return rows

    @property
    def launch_count(self) -> int:
        return int(self._lib.sm_launch_count(self._engine))

    @property
    def device_bytes(self) -> int:
        return int(self._lib.sm_engine_bytes(self._engine))

    @property
    def handle(self):
        return self._engine

    def _destroy(self):
        if self._engine.value:
            self._lib.sm_engine_destroy(self._engine)
            self._engine = C.c_void_p(None)

    def __del__(self):
        try:
            self._destroy()
        except Exception:
            pass
