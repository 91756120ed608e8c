"""Generates tests/golden/vot_eval.npz with the reference's own pysot evaluation code.  TEST INFRASTRUCTURE ONLY; it
needs the reference source tree (SIAMMASK_REFERENCE), Cython, numba and a C compiler:

    python tools/make_vot_eval_golden.py

It compiles the reference's utils/pysot/utils/region.pyx (with src/region.c) in a temporary directory, stubs colorama,
writes K trackers' trajectories over G synthetic sequences with `siammask_b200.vot.write_result` into a pysot results
tree, and runs pysot's AccuracyRobustnessBenchmark and EAOBenchmark over a dataset of pysot VOTVideo objects, which
read the files back with load_tracker.  The per-frame overlaps the benchmarks compute (calculate_accuracy) and the
expected-overlap curve (calculate_expected_overlap) are captured on their way through.  Cases: no failure; a failure at
frame 1; failures in the last 5 frames (point dropped); a failure at exactly T-5 (empty last fragment); back-to-back
failures; NaN overlaps from a degenerate gt in a sequence without and with failures; T below low, between low and high,
above high; a 2x2 frame; locations on exact .xxxx5 ties and ones printed as -0.0000; three trackers; EAO with the
VOT2018 and the VOT2019 bounds.
"""
from __future__ import annotations

import glob
import importlib.util
import os
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "vot_eval.npz")
REF = os.environ.get("SIAMMASK_REFERENCE", "/root/reference")

# (T, W, H, failure plan per tracker, degenerate gt frames)
SEQUENCES = [
    (60, 320, 240, ([], [1, 7], [55]), []),                 # below low; back-to-back; failure at T-5
    (150, 640, 360, ([], [40, 146], [20, 26, 32, 148]), []),  # between; failures in the last 5 frames
    (420, 1280, 720, ([300], [1], []), []),                 # above high; failure at frame 1
    (30, 2, 2, ([], [3], [10, 25]), []),                    # a 2x2 frame
    (120, 320, 240, ([], [50], [31]), [30, 31, 32, 33, 90]),  # degenerate gt: NaN with and without failures
    (80, 400, 300, ([78], [75], []), []),                   # dropped point; failure at T-5
]
K = 3


def _rect(x, y, w, h):
    return [x, y, x + w, y, x + w, y + h, x, y + h]


def make_inputs(rng):
    """gts (G float64 [T, 8]), sizes (G (W, H)), regions[g][k] in the form VotRunner.result() returns."""
    gts, sizes, regions = [], [], []
    for T, W, H, plans, degenerate in SEQUENCES:
        small = W <= 2
        gt, boxes = [], []
        for f in range(T):
            if small:
                x, y, w, h = rng.uniform(0, 0.6), rng.uniform(0, 0.6), rng.uniform(0.8, 1.4), rng.uniform(0.8, 1.4)
            else:
                w, h = W * rng.uniform(0.1, 0.3), H * rng.uniform(0.1, 0.3)
                x, y = rng.uniform(-0.05 * W, W - 0.9 * w), rng.uniform(-0.05 * H, H - 0.9 * h)
            a = rng.uniform(-0.3, 0.3)
            c, s = np.cos(a), np.sin(a)
            cx, cy = x + w / 2, y + h / 2
            pts = [(-w / 2, -h / 2), (w / 2, -h / 2), (w / 2, h / 2), (-w / 2, h / 2)]
            gt.append([v for dx, dy in pts for v in (cx + c * dx - s * dy, cy + s * dx + c * dy)])
            boxes.append((x, y, w, h))
        for f in degenerate:
            gt[f] = [1.2, 1.2] * 4                                         # a single point
        gts.append(np.asarray(gt, np.float64))
        sizes.append((W, H))
        per_k = []
        for k in range(K):
            traj, start, plan = [], 0, set(plans[k])
            for f in range(T):
                if f == start:
                    traj.append(1)
                elif f > start and f in plan:
                    traj.append(2)
                    start = f + 5
                elif f > start:
                    x, y, w, h = boxes[f]
                    j = (1.0 if small else 0.1 * w) * rng.uniform(-1, 1, 4)
                    loc = np.array([x + j[0], y + j[1], w * (1 + 0.1 * j[2]), h * (1 + 0.1 * j[3])])
                    u = rng.rand()
                    if f in degenerate:
                        loc = np.array([1.2, 1.2, 0.05, 0.05])                 # inside the gt's pixel: NaN
                    elif u < 0.15:                                             # exact ties at the 5th decimal
                        loc = np.floor(loc) + rng.choice([1, 3, 5, 7, 9, 11, 13, 29], 4) / 32.0
                    elif u < 0.2:
                        loc[0] = -rng.uniform(0, 4.9e-5)                       # printed as -0.0000
                    traj.append(loc)
                else:
                    traj.append(0)
            per_k.append(traj)
        regions.append(per_k)
    return gts, sizes, regions


def build_region(tmp):
    """The reference's Cython region module, compiled in tmp; returns the extension's path."""
    src = os.path.join(REF, "utils", "pysot", "utils")
    for name in ("region.pyx", "c_region.pxd"):
        shutil.copy(os.path.join(src, name), tmp)
    shutil.copytree(os.path.join(src, "src"), os.path.join(tmp, "src"))
    code = ("from setuptools import setup, Extension; from Cython.Build import cythonize; "
            "setup(ext_modules=cythonize([Extension('region', ['region.pyx', 'src/region.c'])], quiet=True))")
    subprocess.run([sys.executable, "-c", code, "build_ext", "--inplace"], cwd=tmp, check=True, capture_output=True)
    return glob.glob(os.path.join(tmp, "region*.so"))[0]


def import_pysot(region_so):
    colorama = types.ModuleType("colorama")
    colorama.Style = types.SimpleNamespace(RESET_ALL="")
    colorama.Fore = types.SimpleNamespace(RED="")
    sys.modules["colorama"] = colorama
    sys.path.insert(0, os.path.join(REF, "utils"))
    spec = importlib.util.spec_from_file_location("pysot.utils.region", region_so)
    region = importlib.util.module_from_spec(spec)
    sys.modules["pysot.utils.region"] = region
    spec.loader.exec_module(region)
    from pysot.datasets.vot import VOTVideo
    from pysot.evaluation import ar_benchmark, eao_benchmark
    return VOTVideo, ar_benchmark, eao_benchmark


class Dataset:
    """What the two benchmarks use of a pysot VOTDataset."""

    def __init__(self, name, videos, tracker_path):
        self.name, self.videos, self.tracker_path = name, {v.name: v for v in videos}, tracker_path

    def __len__(self):
        return len(self.videos)

    def __getitem__(self, i):
        return list(self.videos.values())[i] if isinstance(i, int) else self.videos[i]

    def __iter__(self):
        return iter(self.videos.values())


def main():
    from siammask_b200 import vot
    rng = np.random.RandomState(7)
    gts, sizes, regions = make_inputs(rng)
    G = len(gts)
    names = [f"seq{g}" for g in range(G)]
    trackers = [f"combo{k}" for k in range(K)]
    with tempfile.TemporaryDirectory() as tmp:
        VOTVideo, ar_benchmark, eao_benchmark = import_pysot(build_region(tmp))
        results = os.path.join(tmp, "results")
        for g in range(G):
            for k in range(K):
                d = os.path.join(results, trackers[k], "baseline", names[g])
                os.makedirs(d)
                vot.write_result(os.path.join(d, f"{names[g]}_001.txt"), regions[g][k])
        T = [len(a) for a in gts]

        def videos():
            return [VOTVideo(names[g], tmp, names[g], gts[g][0].tolist(), [], gts[g].tolist(), *([[0] * T[g]] * 5),
                             sizes[g][0], sizes[g][1]) for g in range(G)]

        captured = {"acc": [], "eao": [], "curve": []}

        def capture(module, key):
            fn = module.calculate_accuracy

            def wrapped(*a, **kw):
                out = fn(*a, **kw)
                captured[key].append(out[1])
                return out
            module.calculate_accuracy = wrapped
        capture(ar_benchmark, "acc")
        capture(eao_benchmark, "eao")
        curve_fn = eao_benchmark.calculate_expected_overlap

        def curve(fragments, fweights):
            out = curve_fn(fragments, fweights)
            captured["curve"].append(out)
            return out
        eao_benchmark.calculate_expected_overlap = curve

        ds = Dataset("VOT2018", videos(), results)
        ar = ar_benchmark.AccuracyRobustnessBenchmark(ds).eval(trackers)
        eao18 = eao_benchmark.EAOBenchmark(ds).eval(trackers)
        curves = list(captured["curve"])
        eao19 = eao_benchmark.EAOBenchmark(Dataset("VOT2019", videos(), results)).eval(trackers)

    Tmax = max(T)
    acc_bits = np.full((K, G, Tmax), 0x7FC00000, np.uint32)
    eao_bits = np.full((K, G, Tmax), 0x7FC00000, np.uint32)
    for k in range(K):                      # both benchmarks visit tracker by tracker, sequence by sequence
        for g in range(G):
            acc_bits[k, g, :T[g]] = np.asarray(captured["acc"][k * G + g], np.float32).view(np.uint32)
            eao_bits[k, g, :T[g]] = np.asarray(captured["eao"][k * G + g], np.float32).view(np.uint32)
    accuracy, robustness, lost = [], [], []
    for t in trackers:                       # AccuracyRobustnessBenchmark.show_result's figures
        ov = np.concatenate([np.asarray(v, np.float64) for v in ar[t]["overlaps"].values()])
        with np.errstate(invalid="ignore"):
            accuracy.append(np.nanmean(ov))
        n = int(np.sum([f for f in ar[t]["failures"].values()]))
        lost.append(n)
        robustness.append(n / len(ov) * 100)
    rec = np.zeros((K, G, Tmax, 5))
    for g in range(G):
        for k in range(K):
            for f, x in enumerate(regions[g][k]):
                rec[k, g, f] = (x, 0, 0, 0, 0) if isinstance(x, int) else (3, *x)
    gt = np.zeros((G, Tmax, 8))
    for g in range(G):
        gt[g, :T[g]] = gts[g]
    np.savez_compressed(OUT, rec=rec, gt=gt, length=np.asarray(T, np.int32), size=np.asarray(sizes, np.int32),
                        acc_overlap_bits=acc_bits, eao_overlap_bits=eao_bits, accuracy=np.asarray(accuracy),
                        robustness=np.asarray(robustness), lost_number=np.asarray(lost, np.int64),
                        curve=np.asarray(curves, np.float32), eao_vot2018=np.asarray([eao18[t]["all"] for t in trackers]),
                        eao_vot2019=np.asarray([eao19[t]["all"] for t in trackers]))
    print(f"wrote {OUT}: {K} trackers x {G} sequences, lengths {T}; accuracy {np.round(accuracy, 4).tolist()}, "
          f"lost {lost}, EAO 2018 {[round(eao18[t]['all'], 4) for t in trackers]}, "
          f"2019 {[round(eao19[t]['all'], 4) for t in trackers]}")


if __name__ == "__main__":
    main()
