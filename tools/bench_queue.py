"""Whole benchmarks through one engine: the queue of `VotRunner.open_queue` / `ParamSweep.open_queue` against today's
fixed chunks, on the same workload in the same process.

    python tools/bench_queue.py [--reps 3 --max-batch 256] [--baseline-tracker FILE]
    python tools/bench_queue.py --count-only          # host only: the scheduler's step counts, no GPU

VOT workload: 60 sequences whose lengths are np.random.default_rng(0).lognormal(5.6, 0.7, 60), rounded and clipped to
[41, 1500] (53 .. 1067 frames, 20 768 in all), frame sizes 1280x720, 854x480 and 640x360 in turn, x K = 16
hyper-parameter combinations = 960 streams through an engine of max_batch 256.  Each sequence cycles a pool of 5
synthetic frames kept on the device (a textured rectangle swinging over a textured background), so decoding and host
memory stay out of the timing; its gt quad jumps to a far corner every 50th frame, so streams fail, skip and
re-initialise.  The chunked baseline is today's way: one `VotRunner.open` per 16 sequences in index order (256
streams), run to its longest sequence.

Sweep workload: 20 videos of 40-104 frames at 854x480 and 640x360 x 100 combinations (2 000 streams), the queue
against one `ParamSweep.open` per (length, size) group, split so that each fits the engine.

Prints one JSON line: the card name and power limit (read-only nvidia-smi query in the same call), the step counts, and
per leg the wall times of --reps alternated runs (host clock around work that ends in a device synchronise; medians and
ranges) and stream-frames/s; whether the queue's outputs equal the chunked runs'; with --baseline-tracker (a
siammask_b200/tracker.py from another revision) bench.py's `loop` leg with that tracker and with this one, alternated.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from siammask_b200 import schedule                              # noqa: E402

K_VOT, CAPACITY = 16, 256
SIZES = [(720, 1280), (480, 854), (360, 640)]
SWEEP_SIZES = [(480, 854), (360, 640)]
POOL = [0, 1, 2, 3, 4, 3, 2, 1]          # frame t of a sequence is pool frame POOL[t % 8]: the target swings, no jump


def vot_lengths() -> np.ndarray:
    return np.clip(np.round(np.random.default_rng(0).lognormal(5.6, 0.7, 60)), 41, 1500).astype(np.int64)


def sweep_lengths() -> np.ndarray:
    return np.random.default_rng(1).integers(40, 105, 20).astype(np.int64)


def counts(lengths, K, capacity) -> dict:
    steps = schedule.plan(lengths, K, capacity)
    chunked = schedule.chunked_steps(lengths, K, capacity)
    per = capacity // K
    T = np.asarray(lengths)
    busy = sum(int(T[i:i + per].sum()) * K for i in range(0, T.size, per))      # stream-steps of the chunked runs
    return {"queue_steps": len(steps), "chunked_steps": chunked,
            "queue_mean_batch": float(np.mean([len(s.track) + len(s.admit) for s in steps])),
            "chunked_mean_batch": busy / chunked}


# ---------------------------------------------------------------------------------------------- GPU legs
def make_pools(lengths, sizes, seed=0, fail_every=50):
    """Per sequence: a pool of 5 uint8 CUDA frames [H,W,3], its gt float64 [T,8] and the target's box of each pool
    frame (x, y, w, h)."""
    import torch
    rng = np.random.RandomState(seed)
    pools, gts, boxes = [], [], []
    for g, T in enumerate(lengths):
        H, W = sizes[g % len(sizes)]
        bg = np.kron((rng.rand(H // 8 + 1, W // 8 + 1, 3) * 255).astype(np.uint8), np.ones((8, 8, 1), np.uint8))[:H, :W]
        w, h = rng.randint(60, 120, 2)
        tex = np.kron((rng.rand(h // 8 + 1, w // 8 + 1, 3) * 255).astype(np.uint8), np.ones((8, 8, 1), np.uint8))[:h, :w]
        x0, y0 = rng.rand(2) * [W - w - 40, H - h - 40] + 20
        frames, bx = [], []
        for p in range(5):
            x, y = int(min(x0 + 4 * p, W - w)), int(min(y0 + 3 * p, H - h))
            f = bg.copy()
            f[y:y + h, x:x + w] = tex
            frames.append(torch.from_numpy(f).cuda())
            bx.append((x, y, int(w), int(h)))
        gt = np.zeros((T, 8))
        for t in range(T):
            x, y, bw, bh = bx[POOL[t % 8]]
            gt[t] = [x, y, x + bw, y, x + bw, y + bh, x, y + bh]
            if t and t % fail_every == 0:
                gt[t] = [0, 0, 10, 0, 10, 10, 0, 10]
        pools.append(frames)
        gts.append(gt)
        boxes.append(bx)
    return pools, gts, boxes


def frame_of(pools, g, t):
    return pools[g][POOL[t % 8]]


def run_vot_queue(net, params, combos, pools, gts):
    import siammask_b200 as smb
    runner = smb.VotRunner(net, params, combos)
    runner.open_queue(gts)
    while runner.pending:
        runner.step([frame_of(pools, g, t) for g, t in runner.needed()])
    return runner


def run_vot_chunked(net, params, combos, pools, gts):
    import siammask_b200 as smb
    per = net.max_batch // combos.shape[0]
    out = []
    for c in range(0, len(gts), per):
        seqs = range(c, min(c + per, len(gts)))
        runner = smb.VotRunner(net, params, combos)
        T = [len(gts[g]) for g in seqs]
        runner.open([frame_of(pools, g, 0) for g in seqs], [gts[g] for g in seqs])
        for f in range(1, max(T)):
            runner.frame([frame_of(pools, g, f) if f < T[i] else None for i, g in enumerate(seqs)])
        out.append(runner)
    return out


def annos_of(pools, boxes):
    import torch
    out = []
    for g, frames in enumerate(pools):
        H, W = frames[0].shape[:2]
        a = []
        for (x, y, w, h) in boxes[g]:
            m = torch.zeros(H, W, dtype=torch.uint8, device="cuda")
            m[y:y + h, x:x + w] = 1
            a.append(m)
        out.append(a)
    return out


def run_sweep_queue(net, params, combos, pools, boxes, annos, T):
    import siammask_b200 as smb
    sweep = smb.ParamSweep(net, params, combos)
    sweep.open_queue([boxes[g][0] for g in range(len(T))], T)
    while sweep.pending:
        need = sweep.needed()
        sweep.step([frame_of(pools, g, t) for g, t in need],
                   [annos[g][POOL[t % 8]] if 0 < t < T[g] - 1 else None for g, t in need])
    return sweep


def sweep_groups(T, sizes, per):
    """Videos grouped by (length, size), each group split into runs of at most `per` videos."""
    groups = {}
    for g in range(len(T)):
        groups.setdefault((int(T[g]), sizes[g % len(sizes)]), []).append(g)
    return [v[i:i + per] for v in groups.values() for i in range(0, len(v), per)]


def run_sweep_grouped(net, params, combos, pools, boxes, annos, T, runs):
    import torch
    import siammask_b200 as smb
    out = []
    for vids in runs:
        sweep = smb.ParamSweep(net, params, combos)
        sweep.open(torch.stack([frame_of(pools, g, 0) for g in vids]), [boxes[g][0] for g in vids], int(T[vids[0]]))
        for f in range(1, int(T[vids[0]])):
            a = torch.stack([annos[g][POOL[f % 8]] for g in vids]) if f < T[vids[0]] - 1 else None
            sweep.frame(torch.stack([frame_of(pools, g, f) for g in vids]), a)
        out.append((vids, sweep))
    return out


def alternate(legs, reps):
    """Wall seconds of each leg over `reps` alternated runs, and the last run's output of each."""
    import torch
    times = {k: [] for k in legs}
    last = {}
    for _ in range(reps):
        for name, fn in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            last[name] = fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - t0)
            print(f"{name}: {times[name][-1]:.2f} s", file=sys.stderr, flush=True)
    return times, last


def summary(times, stream_frames):
    out = {}
    for name, ts in times.items():
        out[name] = {"seconds": ts, "median_s": float(np.median(ts)), "range_s": [min(ts), max(ts)],
                     "stream_frames_per_s": stream_frames / float(np.median(ts)),
                     "range_stream_frames_per_s": [stream_frames / max(ts), stream_frames / min(ts)]}
    return out


def build_net(max_batch):
    """The sharp engine (mask and refine branches) at the largest of max_batch, 3/4, 1/2 ... that fits."""
    import torch
    import siammask_b200 as smb
    from oracle.calibrate import calibrated_state_dict
    sd = calibrated_state_dict(0)
    B = max_batch
    while True:
        try:
            net = smb.Custom(anchors=smb.DEFAULT_ANCHORS, max_batch=B, num_slots=B)
            return net.load_state_dict(sd).eval().to("cuda"), B
        except (RuntimeError, torch.cuda.OutOfMemoryError):
            if B <= 16:
                raise
            B = B * 3 // 4
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--count-only", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-batch", type=int, default=CAPACITY)
    ap.add_argument("--sequences", type=int, default=60, help="use the first N sequences of the VOT workload")
    ap.add_argument("--videos", type=int, default=20, help="use the first N videos of the sweep workload")
    ap.add_argument("--sweep-combos", type=int, default=100)
    ap.add_argument("--legs", default="vot,sweep", help="comma-separated subset of vot, sweep")
    ap.add_argument("--baseline-tracker", default=None)
    ap.add_argument("--loop-reps", type=int, default=3)
    args = ap.parse_args()
    L = vot_lengths()[:args.sequences]
    TS = sweep_lengths()[:args.videos]
    res = {"metric": "queue_vs_chunked", "vot_lengths": {"min": int(L.min()), "max": int(L.max()),
                                                           "mean": float(L.mean()), "frames": int(L.sum())}}
    if args.count_only:
        res["vot"] = counts(L, K_VOT, args.max_batch)
        print(json.dumps(res))
        return
    import torch
    from bench_vos import gpu_info, loop_legs
    torch.cuda.set_device(0)
    res.update(gpu_info())
    net, B = build_net(args.max_batch)
    res["max_batch"], res["reps"] = B, args.reps
    legs = args.legs.split(",")
    if "vot" in legs:
        vot_leg(res, net, B, L, args.reps)
    if "sweep" in legs:
        sweep_leg(res, net, B, TS, args.reps, args.sweep_combos)
    if args.baseline_tracker:
        res["loop"] = loop_legs(args.baseline_tracker, args.loop_reps)
    print(json.dumps(res))


def vot_leg(res, net, B, L, reps):
    import torch
    from siammask_b200.tracker import TrackerParams
    from siammask_b200.tune import grid
    params = TrackerParams(instance_size=255)
    combos = grid([0.04, 0.1, 0.2, 0.3], [0.3, 0.4], [0.35, 0.45])[:K_VOT]
    res["vot"] = counts(L, K_VOT, B)
    pools, gts, _ = make_pools(L, SIZES)
    stream_frames = int(L.sum()) * K_VOT
    run_vot_queue(net, params, combos, [p for p in pools[:2]], [g[:60] for g in gts[:2]])          # warm-up
    times, last = alternate({"queue": lambda: run_vot_queue(net, params, combos, pools, gts),
                             "chunked": lambda: run_vot_chunked(net, params, combos, pools, gts)}, reps)
    res["vot"].update(summary(times, stream_frames))
    res["vot"]["stream_frames"] = stream_frames
    q_reg, q_lost = last["queue"].result()
    same, per = True, B // K_VOT
    for c, runner in enumerate(last["chunked"]):
        reg, lost = runner.result()
        for i in range(len(reg)):
            g = c * per + i
            same = same and (lost[i] == q_lost[g]).all() and all(
                [x if isinstance(x, int) else tuple(x) for x in reg[i][k]] ==
                [x if isinstance(x, int) else tuple(x) for x in q_reg[g][k]] for k in range(K_VOT))
    res["vot"]["identical"] = bool(same)
    res["vot"]["lost_times_total"] = int(q_lost.sum())
    del pools, last
    torch.cuda.empty_cache()


def sweep_leg(res, net, B, TS, reps, n_combos):
    from siammask_b200.tracker import TrackerParams
    from siammask_b200.tune import grid
    sc = grid(np.linspace(0.0, 0.09, 4), np.linspace(0.3, 0.46, 5), np.linspace(0.8, 1.0, 5))[:n_combos]
    Ks = sc.shape[0]
    sp = TrackerParams(instance_size=255, out_size=127)
    pools, _, boxes = make_pools(TS, SWEEP_SIZES, seed=1)
    annos = annos_of(pools, boxes)
    runs = sweep_groups(TS, SWEEP_SIZES, max(1, B // Ks))
    res["sweep"] = {"videos": len(TS), "combinations": Ks, "lengths": [int(t) for t in TS],
                    "queue_steps": len(schedule.plan(TS, Ks, B)),
                    "grouped_runs": len(runs), "grouped_steps": int(sum(int(TS[v[0]]) for v in runs))}
    times, last = alternate({"queue": lambda: run_sweep_queue(net, sp, sc, pools, boxes, annos, TS),
                             "grouped": lambda: run_sweep_grouped(net, sp, sc, pools, boxes, annos, TS, runs)},
                            reps)
    res["sweep"].update(summary(times, int(TS.sum()) * Ks))
    q_mean, q_rows = last["queue"].result()
    same = True
    for vids, sweep in last["grouped"]:
        mean, rows = sweep.result()
        for i, g in enumerate(vids):
            same = same and np.array_equal(mean[i], q_mean[g]) and np.array_equal(rows[:, i], q_rows[g])
    res["sweep"]["identical"] = bool(same)


if __name__ == "__main__":
    main()
