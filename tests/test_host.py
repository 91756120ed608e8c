"""Host-side logic that needs no GPU: the C-ABI library loads and exports every symbol the header declares,
the checkpoint contract, and loud failure (never a CPU fallback) when no CUDA device is present."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import ROOT
import siammask_b200
from siammask_b200 import _lib
from siammask_b200.checkpoint import expected_keys, normalize_keys, synthetic_state_dict


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "siammask_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sm_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = C.CDLL(_lib.LIB_PATH)
    syms = _header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/siammask_b200.h but not exported"
    assert set(syms) == set(_lib.SIGNATURES), "ctypes prototypes out of sync with the header"
    assert b"sm_90a" in _lib.load().sm_version()


def test_ctypes_struct_layouts_match_the_header(tmp_path):
    """The ctypes mirrors of the C-ABI structs (sm_config, sm_tensor_desc, sm_step_io, sm_tracker_hp) against what a C
    compiler makes of include/siammask_b200.h: sizes and field offsets."""
    import shutil
    import subprocess
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    structs = {"sm_config": _lib.SmConfig, "sm_tensor_desc": _lib.SmTensorDesc, "sm_step_io": _lib.SmStepIO,
               "sm_tracker_hp": _lib.SmTrackerHp}
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "siammask_b200.h"', "int main(void) {"]
    for cname, ct in structs.items():
        prog.append(f'  printf("{cname} %zu", sizeof({cname}));')
        for fname, _ in ct._fields_:
            prog.append(f'  printf(" %zu", offsetof({cname}, {fname}));')
        prog.append('  printf("\\n");')
    prog += ["  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "abi"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    for line in filter(None, out):
        name, size, *offs = line.split()
        ct = structs[name]
        assert int(size) == C.sizeof(ct), name
        assert [int(o) for o in offs] == [getattr(ct, f).offset for f, _ in ct._fields_], name


def test_checkpoint_contract():
    keys = expected_keys()
    assert len(keys) == 303                         # 356 state tensors minus 53 num_batches_tracked
    assert sum(int(torch.Size(s).numel()) for k, s in keys.items()
               if not k.endswith(("running_mean", "running_var"))) == 21482052   # SURVEY §8a parameter count
    assert keys["features.features.layer2.0.downsample.0.weight"] == (512, 256, 3, 3)
    assert keys["features.features.layer3.0.downsample.0.weight"] == (1024, 512, 3, 3)
    assert keys["mask_model.mask.head.3.weight"] == (3969, 256, 1, 1)
    assert keys["refine_model.deconv.weight"] == (256, 32, 15, 15)
    assert len(expected_keys(mask=False, refine=False)) < len(keys)
    sd = synthetic_state_dict(3)
    assert set(sd) == set(keys) and all(tuple(sd[k].shape) == keys[k] for k in keys)
    sd2 = synthetic_state_dict(3)
    assert all(torch.equal(sd[k], sd2[k]) for k in keys)          # deterministic
    wrapped = {"state_dict": {"module." + k: v for k, v in sd.items()}}
    assert set(normalize_keys(wrapped)) == set(keys)               # utils/load_helper.py:38-41


def test_custom_surface_and_validation():
    m = siammask_b200.Custom(anchors=siammask_b200.DEFAULT_ANCHORS)
    assert m.anchor_num == 5 and m.score_size == 25
    assert siammask_b200.Custom(search_size=383).score_size == 41
    assert set(m.state_dict()) == set(expected_keys())
    for name in ("template", "track", "track_mask", "track_refine", "eval", "to", "load_state_dict"):
        assert callable(getattr(m, name))
    sd = synthetic_state_dict(0)
    bad = dict(sd)
    bad.pop("rpn_model.cls.head.3.bias")
    with pytest.raises(KeyError):
        m.load_state_dict(bad, strict=True)
    # strict=False (the reference's mode, utils/load_helper.py:53): the missing tensor keeps its initial value
    with pytest.warns(RuntimeWarning, match="lacks 1 hot-path"):
        m.load_state_dict(bad)
    assert "rpn_model.cls.head.3.bias" in m.state_dict()
    with pytest.raises(AssertionError):                # nothing matches at all: load_helper.py:19
        m.load_state_dict({"unrelated.weight": torch.zeros(1)})
    bad = dict(sd)
    bad["features.features.conv1.weight"] = torch.zeros(64, 3, 3, 3)
    with pytest.raises(ValueError):
        m.load_state_dict(bad)
    assert m.load_state_dict(sd) is m and m.eval() is m
    with pytest.raises(RuntimeError):
        m.to("cpu")
    with pytest.raises(NotImplementedError):
        m.train(True)


def test_load_checkpoint_from_disk(tmp_path):
    """`load_checkpoint` restates utils/load_helper.py:30-54: bare or {'state_dict':...} files, 'module.' prefix,
    and the 'features.' retry for a backbone-only checkpoint."""
    from siammask_b200.checkpoint import load_checkpoint
    sd = synthetic_state_dict(5)
    p1 = str(tmp_path / "full.pth")
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "epoch": 3}, p1)
    got = load_checkpoint(p1)
    assert set(got) >= set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    p2 = str(tmp_path / "backbone.pth")                # torchvision-style backbone file: keys lack 'features.'
    bb = {k[len("features."):]: v for k, v in sd.items() if k.startswith("features.features.")}
    torch.save(bb, p2)
    got = load_checkpoint(p2)
    assert set(got) == {"features." + k for k in bb}
    m = siammask_b200.Custom(anchors=siammask_b200.DEFAULT_ANCHORS)
    with pytest.warns(RuntimeWarning):
        m.load_state_dict(got)                         # heads keep their init, as with the reference's strict=False
    p3 = str(tmp_path / "junk.pth")
    torch.save({"a": torch.zeros(1)}, p3)
    with pytest.raises(AssertionError):
        load_checkpoint(p3)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks behaviour on a box WITHOUT a GPU")
def test_no_silent_cpu_fallback():
    lib = _lib.load()
    cfg = _lib.SmConfig(255, 1, 1, 0, 0, 5, 1)
    h = C.c_void_p()
    assert lib.sm_engine_create(C.byref(cfg), C.byref(h)) != 0
    assert b"no CUDA device" in lib.sm_last_error()
    buf = (C.c_float * 16)()
    assert lib.sm_xcorr_depthwise(buf, buf, buf, 1, 1, 2, 2, 1, 1, None) != 0
    with pytest.raises(RuntimeError):
        siammask_b200.conv2d_dw_group(torch.zeros(1, 1, 8, 8), torch.zeros(1, 1, 3, 3))
