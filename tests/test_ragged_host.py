"""Frames of different sizes in one batch, host side: the packing helper (offsets, shapes, None entries, the descriptor
table reused while the shapes repeat), argument checks that fire before any device work, and the exported C ABI."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.synthetic_video import make_frames
from siammask_b200 import _lib
from siammask_b200.tracker import IMAGE_DESC, FramePacker, image_table

SIZES = [(240, 320), (480, 854), (720, 1280), (97, 131)]


def _frames():
    """make_frames' drifting rectangle needs at least 128 x 184 pixels: the small odd size is noise."""
    rng = np.random.RandomState(5)
    return [make_frames(n=1, h=h, w=w, seed=i)[0][0] if h >= 128 else rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
            for i, (h, w) in enumerate(SIZES)]


def test_descriptor_layout_matches_the_c_struct():
    assert IMAGE_DESC.itemsize == 16
    assert [IMAGE_DESC.fields[k][1] for k in ("offset", "h", "w")] == [0, 8, 12]


def test_pack_offsets_shapes_and_none_entries():
    fr = _frames()
    items = [fr[0], None, fr[1], fr[2], None, fr[3]]
    p = FramePacker("cpu").pack(items, 3)
    want = [None if f is None else f.shape[:2] for f in items]
    assert p.shapes == want
    off = 0
    for i, f in enumerate(items):
        row = p.table[i]
        if f is None:
            assert (row["h"], row["w"]) == (0, 0)
            continue
        assert (int(row["offset"]), int(row["h"]), int(row["w"])) == (off, f.shape[0], f.shape[1])
        np.testing.assert_array_equal(p.view(i).numpy(), f)
        off += f.size
    assert p.data.numel() == off
    assert bytes(p.desc.numpy()) == p.table.tobytes()


def test_pack_label_maps_one_byte_per_pixel():
    maps = [np.full((h, w), i + 1, np.uint8) for i, (h, w) in enumerate(SIZES)]
    p = FramePacker("cpu").pack(maps, 1)
    assert list(p.table["offset"]) == list(np.cumsum([0] + [h * w for h, w in SIZES[:-1]]))
    for i, m in enumerate(maps):
        np.testing.assert_array_equal(p.view(i).numpy(), m)


def test_pack_tensors_and_arrays_give_the_same_buffer():
    fr = _frames()
    a = FramePacker("cpu").pack(fr, 3)
    b = FramePacker("cpu").pack([torch.from_numpy(f) for f in fr], 3)
    assert torch.equal(a.data, b.data) and a.shapes == b.shapes


def test_descriptor_table_is_reused_while_shapes_repeat():
    fr = _frames()
    pk = FramePacker("cpu")
    first = pk.pack(fr, 3).desc
    assert pk.pack([f.copy() for f in fr], 3).desc is first            # same shapes: no new table
    changed = pk.pack(fr[::-1], 3).desc
    assert changed is not first
    assert pk.pack(fr[::-1], 3).desc is changed
    assert pk.table([f.shape[:2] for f in fr[::-1]], 3)[0] is changed


def test_wrap_a_batch_in_place_under_the_uniform_table():
    pk = FramePacker("cpu")
    t = torch.from_numpy(np.random.RandomState(1).randint(0, 256, (4, 6, 5, 3)).astype(np.uint8))
    p = pk.wrap(t, 3)
    assert p.data.data_ptr() == t.data_ptr() and p.data.numel() == t.numel()       # no copy
    assert p.table.tobytes() == image_table([(6, 5)] * 4, 3).tobytes()
    assert bytes(p.desc.numpy()) == p.table.tobytes()
    assert p.shapes == [(6, 5)] * 4 and p.channels == 3
    for i in range(4):
        assert torch.equal(p.view(i), t[i])
    assert pk.wrap(t.clone(), 3).desc is p.desc                                      # same shape: no new table
    assert pk.table([(6, 5)] * 4, 3)[0] is p.desc


def test_wrap_a_shared_frame_and_label_maps():
    pk = FramePacker("cpu")
    frame = torch.from_numpy(np.random.RandomState(2).randint(0, 256, (6, 5, 3)).astype(np.uint8))
    p = pk.wrap(frame, 3, shared=3)                                                  # 3 entries read one frame
    assert p.data.data_ptr() == frame.data_ptr() and p.data.numel() == frame.numel()
    assert list(p.table["offset"]) == [0, 0, 0] and list(p.table["h"]) == [6] * 3 and list(p.table["w"]) == [5] * 3
    assert bytes(p.desc.numpy()) == p.table.tobytes()
    assert all(torch.equal(p.view(i), frame) for i in range(3))
    assert pk.wrap(frame, 3).desc is not p.desc                                      # [3 back to back] is another table
    maps = np.random.RandomState(3).randint(0, 4, (3, 6, 5)).astype(np.uint8)         # [G,H,W] label maps, from numpy
    m = pk.wrap(maps, 1)
    assert m.table.tobytes() == image_table([(6, 5)] * 3, 1).tobytes() and m.channels == 1
    for g in range(3):
        np.testing.assert_array_equal(m.view(g).numpy(), maps[g])
    assert pk.wrap(maps, 1).desc is m.desc


def test_image_table_of_empty_and_single_entries():
    assert image_table([], 3).size == 0
    t = image_table([None, (2, 3)], 1)
    assert list(t["offset"]) == [0, 0] and list(t["h"]) == [0, 2] and list(t["w"]) == [0, 3]


@pytest.mark.parametrize("bad", [np.zeros((4, 5, 3), np.float32), np.zeros((4, 5), np.uint8),
                                 np.zeros((0, 5, 3), np.uint8), np.zeros((4, 5, 4), np.uint8)])
def test_pack_rejects_bad_frames(bad):
    with pytest.raises(ValueError):
        FramePacker("cpu").pack([np.zeros((4, 5, 3), np.uint8), bad], 3)


def test_pack_rejects_a_non_list():
    with pytest.raises(ValueError):
        FramePacker("cpu").pack(np.zeros((2, 4, 5, 3), np.uint8), 3)


def test_new_c_abi_symbols_are_exported():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in ("sm_crop_resize_ragged", "sm_warp_affine_ragged", "sm_vot_overlap_sized", "sm_paste_labels_ragged",
                 "sm_paste_labels_iou_ragged", "sm_label_boxes_ragged"):
        assert hasattr(lib, name), name
        assert name in _lib.SIGNATURES
