"""Time of `VotScore.add` + `result` (tools/eval.py's VOT accuracy, robustness and EAO on the device) on a
tune_vot-sized record, against the numpy restatement of tests/vot_eval_reference.py on the same data.

    python tools/bench_vot_eval.py [--combos 378 --sequences 60 --reps 3 --out profiles/bench_vot_eval_h100_700w.json]

The record is seeded: 60 sequences with lengths spread over 41..1500 frames and frame sizes from 320x240 to 1280x720,
each run under 378 combinations (tune_vot's default 9 x 14 x 3 grid), the protocol's entry codes with about one failure
per 100 frames, and locations jittered around a moving gt box.  One add() takes the whole record, as a duck-typed
finished `VotRunner`.  The host baseline is the restatement's scoring (accuracy / robustness, fragments, curve, EAO) of
the device's per-frame overlap planes copied to the host; the per-frame polygon rasterisation, which pysot runs in C,
is not part of it.  The two outputs are checked against each other.  Writes one JSON with the card name and power
limit (read-only nvidia-smi query) to --out and prints it.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import siammask_b200 as smb                                     # noqa: E402
import vot_eval_reference as R                                  # noqa: E402
from siammask_b200 import ops, vot                              # noqa: E402
from bench_vos import gpu_info                                  # noqa: E402

SIZES = [(240, 320), (360, 640), (480, 640), (720, 1280)]       # (H, W)


class FinishedRun:
    """What VotScore.add reads of a VotRunner whose sequences have all ended."""

    def __init__(self, rec, gt, T, hw, K):
        self._rec, self._gt, self.T, self._hw, self.K = rec, gt, T, hw, K
        self.G, self.f = len(T), int(T.max())


def make_run(G, K, seed=0):
    rng = np.random.RandomState(seed)
    T = np.round(np.linspace(41, 1500, G)).astype(np.int64)
    rng.shuffle(T)
    Tmax, S = int(T.max()), G * K
    hw = [SIZES[g % len(SIZES)] for g in range(G)]
    boxes = np.zeros((G, Tmax, 4))
    for g, (H, W) in enumerate(hw):
        w, h = W * rng.uniform(0.1, 0.3), H * rng.uniform(0.1, 0.3)
        t = np.arange(Tmax)
        boxes[g] = np.stack([(W - w) * (0.5 + 0.4 * np.sin(t / 50 + g)), (H - h) * (0.5 + 0.4 * np.cos(t / 70 + g)),
                             np.full(Tmax, w), np.full(Tmax, h)], 1)
    x, y, w, h = np.moveaxis(boxes, 2, 0)
    gt = np.stack([x, y, x + w, y, x + w, y + h, x, y + h], 2).astype(np.float32)
    codes = np.zeros((Tmax, S), np.int8)
    for s in range(S):
        Ts, start = int(T[s // K]), 0
        fails = np.cumsum(rng.geometric(1 / 100, Ts // 20 + 2))
        for f in fails:
            if f >= Ts:
                break
            if f <= start:
                continue
            codes[start, s] = vot.CODE_INIT
            codes[start + 1:f, s] = vot.CODE_LOCATION
            codes[f, s] = vot.CODE_LOST
            start = f + vot.SKIP_FRAMES
        if start < Ts:
            codes[start, s] = vot.CODE_INIT
            codes[start + 1:Ts, s] = vot.CODE_LOCATION
    dev = "cuda"
    rec = torch.zeros(Tmax + 1, S, 5, dtype=torch.float64, device=dev)
    rec[:Tmax, :, 0] = torch.from_numpy(codes).to(dev).double()
    b = torch.from_numpy(boxes).to(dev).repeat_interleave(K, 0).transpose(0, 1)          # [Tmax, S, 4]
    jit = torch.randn(Tmax, S, 4, dtype=torch.float64, device=dev, generator=torch.Generator(dev).manual_seed(seed))
    rec[:Tmax, :, 1:] = b + jit * b[..., 2:].repeat(1, 1, 2) * 0.1
    return FinishedRun(rec, torch.from_numpy(gt).to(dev), T, hw, K)


def host_scores(run, low, high):
    """The restatement's scores of every combination from the device's per-frame overlap planes."""
    G, K, T = run.G, run.K, run.T
    Tmax, S = int(T.max()), G * K
    seq = np.repeat(np.arange(G), K)
    i32 = lambda a: torch.as_tensor(np.asarray(a, np.int32), device="cuda")       # noqa: E731
    wh = np.array([(w, h) for h, w in run._hw])[seq]
    acc, eao = ops._vot_trajectory_overlap(run._rec, Tmax, S, run._gt, i32(seq), i32(wh), i32(T[seq]))
    acc, eao, codes = acc.cpu().numpy(), eao.cpu().numpy(), run._rec[:Tmax, :, 0].cpu().numpy()
    t0 = time.perf_counter()
    out = {"accuracy": [], "robustness": [], "lost_number": [], "eao": [], "expected_overlaps": []}
    for k in range(K):
        accs, eaos, fails = [], [], []
        for g in range(G):
            s = g * K + k
            accs.append(acc[:T[g], s])
            eaos.append(eao[:T[g], s])
            fails.append(np.nonzero(codes[:T[g], s] == vot.CODE_LOST)[0].tolist())
        a, r, n = R.accuracy_robustness(accs, [len(f) for f in fails])
        curve = R.expected_overlaps(eaos, fails, Tmax)
        for key, v in zip(out, (a, r, n, R.eao(curve, low, high), curve)):
            out[key].append(v)
    return {k: np.asarray(v) for k, v in out.items()}, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--combos", type=int, default=378)
    ap.add_argument("--sequences", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "bench_vot_eval_h100_700w.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vot_eval needs a CUDA device")
    info = gpu_info()
    run = make_run(a.sequences, a.combos)
    frames = int(run.T.sum()) * run.K
    smb.VotScore(run.K).add(run).result()                                 # warm-up: module load, allocator
    times, dev_res = [], None
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dev_res = smb.VotScore(run.K).add(run).result()
        times.append(time.perf_counter() - t0)
    host_res, host_t = host_scores(run, 100, 356)
    ulps = np.abs(dev_res["expected_overlaps"].view(np.int32).astype(np.int64) -
                  host_res["expected_overlaps"].view(np.int32))
    ok = ~np.isnan(host_res["expected_overlaps"])
    agree = {
        "lost_number_equal": bool((dev_res["lost_number"] == host_res["lost_number"]).all()),
        "accuracy_max_rel": float(np.max(np.abs(dev_res["accuracy"] / host_res["accuracy"] - 1))),
        "robustness_max_rel": float(np.max(np.abs(dev_res["robustness"] / host_res["robustness"] - 1))),
        "curve_nan_pattern_equal": bool((np.isnan(dev_res["expected_overlaps"]) == ~ok).all()),
        "curve_max_ulp": int(ulps[ok].max()),
        "eao_max_abs": float(np.max(np.abs(dev_res["eao"] - host_res["eao"]))),
    }
    res = {"bench": "vot_eval", **info, "combos": run.K, "sequences": run.G, "streams": run.G * run.K,
           "max_T": int(run.T.max()), "stream_frames": frames,
           "lost_entries": int(dev_res["lost_number"].sum()),
           "device_add_result_s": {"median": float(np.median(times)), "min": float(min(times)),
                                   "max": float(max(times)), "reps": a.reps},
           "host_restatement_scoring_s": host_t,
           "host_baseline": "tests/vot_eval_reference.py scoring of the device's per-frame overlaps (rasterisation "
                            "excluded)",
           "speedup_vs_host_scoring": host_t / float(np.median(times)), "agree": agree}
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    assert agree["lost_number_equal"] and agree["curve_nan_pattern_equal"] and agree["curve_max_ulp"] <= 1, agree


if __name__ == "__main__":
    main()
