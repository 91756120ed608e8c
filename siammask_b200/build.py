"""In-tree build of the CUDA extension: nvcc -> siammask_b200/libsiammask_b200.so (sm_90a only)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsiammask_b200.so")
SOURCES = ["conv_gemm_sm90.cu", "conv3x3_patch_sm90.cu", "stem_sm90.cu", "simt_kernels.cu", "xcorr_bulk.cu", "rbox_sm90.cu",
           "engine.cu"]
HEADERS = ["common.cuh", "ptx.cuh", os.path.join("..", "..", "include", "siammask_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libsiammask_b200.so")


HASH = LIB + ".srchash"


def source_hash() -> str:
    """sha256 over the sources, headers and compiler flags the library is built from (content, not mtimes: a snapshot
    copy to another box shuffles the time stamps but not the bytes)."""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for d in SOURCES + HEADERS:
        path = os.path.join(CSRC, d)
        h.update(d.encode())
        if os.path.exists(path):
            with open(path, "rb") as f:
                h.update(f.read())
    return h.hexdigest()


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    try:
        with open(HASH) as f:
            return f.read().strip() != source_hash()
    except OSError:
        return True


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    tmp = f"{LIB}.tmp{os.getpid()}"          # several ranks may build at once: private temp file, atomic replace
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", tmp, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    digest = source_hash()
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB)
    with open(f"{HASH}.tmp{os.getpid()}", "w") as f:
        f.write(digest + "\n")
    os.replace(f"{HASH}.tmp{os.getpid()}", HASH)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
