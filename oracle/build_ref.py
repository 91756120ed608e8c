"""Compiles the reference's VOT region library into oracle/_ref/libvot_region.so.  TEST INFRASTRUCTURE ONLY: the
library is the live oracle of `sm_vot_overlap` (`compute_polygon_overlap`, called through ctypes by the tests and
tools/make_vot_golden.py).  It needs the reference source tree (SIAMMASK_REFERENCE); without it nothing is built and
the tests that want the library skip, while the golden file still pins the kernel.

    python -m oracle.build_ref

Plain x86-64 flags, no -march: like the reference's distutils build of utils/pyvotkit, the compiler may not contract
a * b + c into an FMA, so the library's double arithmetic is the one the reference runs."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

REF = os.environ.get("SIAMMASK_REFERENCE", "/root/reference")
OUT_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")
LIB = os.path.join(OUT_DIR, "libvot_region.so")


def build(verbose: bool = True) -> str | None:
    """Returns the library's path, or None when the reference tree (or a C compiler) is absent."""
    src = os.path.join(REF, "utils", "pyvotkit", "src", "region.c")
    cc = os.environ.get("CC") or shutil.which("cc") or shutil.which("gcc")
    if not os.path.exists(src) or cc is None:
        if verbose:
            print(f"oracle/_ref: skipped ({'no reference tree at ' + REF if cc else 'no C compiler'})")
        return None
    if os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(src):
        return LIB
    tmp = f"{LIB}.tmp{os.getpid()}"
    try:
        os.makedirs(OUT_DIR, exist_ok=True)
        res = subprocess.run([cc, "-O2", "-fPIC", "-shared", "-o", tmp, src, "-lm"], capture_output=True, text=True)
        if res.returncode != 0:
            raise OSError(res.stdout + res.stderr)
        os.replace(tmp, LIB)
    except OSError as e:            # the oracle is optional: the tests that want it skip
        if os.path.exists(tmp):
            os.remove(tmp)
        print(f"oracle/_ref: skipped (building the VOT region library failed: {e})")
        return None
    if verbose:
        print("built", LIB)
    return LIB


def load():
    """ctypes handle of the library with `overlap(poly_a, poly_b, W, H)` bound, or None when it was not built."""
    import ctypes as C
    if not os.path.exists(LIB):
        return None
    lib = C.CDLL(LIB)

    class Polygon(C.Structure):
        _fields_ = [("count", C.c_int), ("x", C.POINTER(C.c_float)), ("y", C.POINTER(C.c_float))]

    class Bounds(C.Structure):
        _fields_ = [("top", C.c_float), ("bottom", C.c_float), ("left", C.c_float), ("right", C.c_float)]

    fn = lib.compute_polygon_overlap
    fn.restype = C.c_float
    fn.argtypes = [C.POINTER(Polygon), C.POINTER(Polygon), C.POINTER(C.c_float), C.POINTER(C.c_float), Bounds]

    def overlap(poly_a, poly_b, W, H):
        """pyvotkit's vot_overlap(poly_a, poly_b, (W, H)) for one pair of 8-value polygons: the float32 bits."""
        import numpy as np
        polys = []
        for p in (poly_a, poly_b):
            p = np.asarray(p, dtype=np.float32).reshape(4, 2)
            xs, ys = (C.c_float * 4)(*p[:, 0].tolist()), (C.c_float * 4)(*p[:, 1].tolist())
            polys.append((Polygon(4, xs, ys), xs, ys))
        only1, only2 = C.c_float(0), C.c_float(0)
        v = fn(C.byref(polys[0][0]), C.byref(polys[1][0]), C.byref(only1), C.byref(only2),
               Bounds(0.0, float(H), 0.0, float(W)))
        return np.float32(v)

    lib.overlap = overlap
    return lib


if __name__ == "__main__":
    sys.exit(0 if build() else 1)
