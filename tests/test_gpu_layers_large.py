"""Every engine layer against float64 at the batch sizes the benchmarks and queues run (up to 256 streams at search
255, 128 at 383), and on an engine built for more streams than the batch it runs.

Tile classes (layer_reference.tile_classes): a launch ends its last 128-row M tile in the first consumer warpgroup's
rows (a) or in the second's (b), has more work items than SMs (c) or more than two per CTA of its persistent grid (d).
At these batch sizes launches reach pairs no batch up to 64 does: the search side's layer1 convs end in (b) only from a
lane of 65 streams, template layer3 and the corr / cls / loc launches reach (d) from B = 67..109.  The batch plan is a
greedy set cover over (a)-(d) up to the largest batch; each planned batch runs on a fresh engine built as bench.py
builds it (max_batch = B, num_slots = 2B) in both precision modes, through the gate and mutations of
test_gpu_layers.py.  The benchmark's own points (255: B = 256, sharp and SiamRPN-only; 383: B = 128) add no pair to
the plan.  Sharp 255 / 256 and 383 / 128 are checked as the first call of the batch sequences below; SiamRPN-only
255 / 256 is listed on the host only.

Streams: each tap is checked on the first and last stream of every lane, the streams holding rows of its launch's last
M tile, and the streams holding the first rows of the work items a persistent CTA takes on its second and third pass,
in both M orders for the GEMM (layer_reference.pass_streams says why both).  A defect confined to a mid-lane tile is
seen there, and the float64 work stays proportional to a few streams per tap.  The mutations, which show that a
layer's gate sees a defect of that layer at all, are evaluated at one stream, the last, which holds the last tile of
every launch.

A queue runs every batch from 1 to max_batch through one engine, so each batch follows a larger or smaller one and the
rows past this call's M hold an earlier call's data.  One engine per precision mode and search size, built for
max_batch = num_slots streams, runs a shrinking and growing sequence the way the queues do (tracker.py): every call is
template(z, slots=) into a permuted slot table, then step(..., slots=) with its on-device selection and the refine at
the position it picked.  The template kernels then go through the slot scatter buffer, which is strided by max_batch
(engine.cu do_template), at B < max_batch.  Every call is checked per layer; from the second on, the call before ran on
other inputs (another seed, the image inverted), and mutation (d) shows that the gate rejects input rows of the
previous call read in the last tile.  Run with -s for the plans, the tables and the per-config worst measured gammas.
"""
import collections
import gc
import time

import numpy as np
import pytest
import torch

import layer_reference as lr
from oracle.calibrate import synthetic_inputs
from siammask_b200.schedule import lane_split
from test_gpu_layers import TABLE, Run, _assert, _consts, _engine, _frame, _tap_list, check, print_table

gpu = pytest.mark.gpu

NUM_SMS = 132                            # H100 SXM
CLASSES = "abcd"
# (search size, mask + refine) -> the largest batch planned: bench.py runs SiamRPN-only at B = 256 (config 3), search
# 383 at B = 128 (config 5); tools/bench_queue.py builds max_batch = 256 at 255.
BOUND = {(255, True): 256, (255, False): 256, (383, True): 128}
ENGINES = list(BOUND)


def _name(key):
    return ("template:" if key[0] == "template" else "") + key[1]


@pytest.fixture(scope="module", autouse=True)
def _table():
    TABLE.clear()
    yield
    print_table()


# ---------------------------------------------------------------------------------------------------- batch plans
_PER_B = {}


def pairs(S, B, with_mask=True):
    """{((side, name), class)} that one call at batch B exercises (engine built with max_batch = B)."""
    if (S, B, with_mask) not in _PER_B:
        _PER_B[(S, B, with_mask)] = {((d["side"], d["name"]), c)
                                     for d in lr.launches(S, B, with_mask=with_mask, refine=with_mask)
                                     for c in lr.tile_classes(d, NUM_SMS)}
    return _PER_B[(S, B, with_mask)]


def batch_plan(S, with_mask=True):
    """Greedy set cover of every (launch, class) pair reachable up to the bound: the batch covering the most missing
    pairs first, the smaller on ties."""
    per_b = {B: pairs(S, B, with_mask) for B in range(1, BOUND[(S, with_mask)] + 1)}
    left, plan = set().union(*per_b.values()), []
    while left:
        B = max(per_b, key=lambda b: (len(per_b[b] & left), -b))
        plan.append(B)
        left -= per_b[B]
    return sorted(plan)


PLAN = {k: batch_plan(*k) for k in ENGINES}
WITH_BENCH = {k: sorted(set(PLAN[k]) | {BOUND[k]}) for k in ENGINES}       # and the benchmark's own batch

# (side, name, class) no batch up to the bound reaches -> (reason, the first batch that does; None: never)
_KERNEL = {("template", b + "conv_kernel.0", c): ("5 x 5 outputs: 25 rows per stream, two N tiles", n)
           for b in lr.BRANCHES for c, n in (("c", 338), ("d", 676))}
_CORR = {("search", lr.CORR[b], "d"): ("the xcorr is not persistent: one block per work item", None)
         for b in lr.BRANCHES}
_V2 = {("refine", "refine_model." + v, c): ("15 x 15 outputs of a lane's streams, one N tile", n)
       for v in ("v2.0", "v2.2") for c, n in (("c", 151), ("d", 301))}
_T2 = {("template", "features.features.layer2.0.conv2", "d"): ("15 x 15 template outputs, GEMM, one N tile", 151)} | {
    ("template", f"features.features.layer2.{i}.conv1", "d"): ("15 x 15 template outputs, GEMM, one N tile", 151)
    for i in (1, 2, 3)} | {
    ("template", f"features.features.layer2.{i}.conv2", "d"): ("15 x 15 template outputs, patch conv, 2 blocks per image",
                                                               133) for i in (1, 2, 3)}


UNREACHABLE = {
    (255, True): _KERNEL | _CORR | {k: v for k, v in _V2.items() if k[2] == "d"},
    (255, False): {k: v for k, v in (_KERNEL | _CORR).items() if "mask" not in k[1]},
    (383, True): _KERNEL | _CORR | _V2 | _T2,
}


def test_batch_plans_cover_every_tile_class():
    """Host only.  Every (launch, class) pair reachable up to the bound is exercised by a planned batch, and the pairs
    that are not reachable are exactly the listed ones; a layer change or a lane-split change that leaves a class
    unchecked fails here.  Prints the (launch, class) -> first batch table."""
    for key in ENGINES:
        S, mask = key
        bound = BOUND[key]
        first = {}
        for B in range(1, bound + 1):
            for p in pairs(S, B, mask):
                first.setdefault(p, B)
        launch_keys = {(d["side"], d["name"]) for d in lr.launches(S, 1, with_mask=mask, refine=mask)}
        print(f"\n[plan] search {S} {'sharp' if mask else 'rpn-only'} up to B={bound}: batches {PLAN[key]} "
              f"(lanes {[lane_split(B, B) for B in PLAN[key]]})")
        for k in sorted(launch_keys):
            print(f"[plan]   {k[0]:8s} {k[1]:42s} " + "  ".join(
                f"{c}: B={first[(k, c)]:3d}" if (k, c) in first else f"{c}:  -   " for c in CLASSES))
        covered = set().union(*(pairs(S, B, mask) for B in PLAN[key]))
        assert covered == set(first), f"search {S}: reachable pairs the plan misses: {set(first) - covered}"
        unreachable = {(*k, c) for k in launch_keys for c in CLASSES if (k, c) not in first}
        print(f"[plan]   not reachable up to B={bound}:")
        for k in sorted(unreachable):
            print(f"[plan]     {k[0]:8s} {k[1]:42s} {k[2]}: {UNREACHABLE[key].get(k, ('NOT LISTED',))[0]}"
                  f"{'' if UNREACHABLE[key].get(k, (0, None))[1] is None else ', needs B >= %d' % UNREACHABLE[key][k][1]}")
        assert unreachable == set(UNREACHABLE[key])
        above = sorted({p for p, b in first.items() if b > 64})
        print(f"[plan]   pairs first reached above B=64: {len(above)}")
    # the listed thresholds: the first batch (one lane's worth of streams for the lane-split sides) that reaches them
    for key in ENGINES:
        S, mask = key
        for (side, name, c), (_, n) in UNREACHABLE[key].items():
            if n is not None:
                assert ((side, name), c) in pairs(S, n, mask) and ((side, name), c) not in pairs(S, n - 1, mask)


# ---------------------------------------------------------------------------------------------------- stream selection
def checked_streams(S, B, max_batch=None, with_mask=True):
    """tap name -> the streams checked at that tap: the first and last stream of every lane of its side (the template
    side is one launch over all B streams), the streams holding rows of its launch's last M tile and the first rows of
    the work items a persistent CTA takes on its second and third pass.  Taps without a tensor-core / xcorr launch
    (copies, SIMT refine convs, the deconv) get the lane boundaries."""
    lanes = lane_split(B, max_batch or B)
    off = np.cumsum([0] + lanes)
    search_edges = {int(s) for a, b in zip(off[:-1], off[1:]) for s in (a, b - 1)}
    edges = {"template:": {0, B - 1}, "": search_edges}
    taps = {p + t.name: set(edges[p]) for t, p in _tap_list("tensor", with_mask, with_mask, with_mask)}
    for d in lr.launches(S, B, max_batch, with_mask=with_mask, refine=with_mask):
        taps[_name((d["side"], d["name"]))] |= lr.last_tile_streams(d) | lr.pass_streams(d, NUM_SMS)
    return taps


def test_checked_streams():
    """Host only.  Every launch's last-tile streams are checked at its tap, the per-tap and total counts stay bounded."""
    for key in ENGINES:
        S, mask = key
        for B in WITH_BENCH[key]:
            taps = checked_streams(S, B, with_mask=mask)
            union = set().union(*taps.values())
            per_tap = sum(len(v) for v in taps.values())
            print(f"[streams] search {S} {'sharp' if mask else 'rpn-only'} B={B:3d}: {len(union):3d} streams, "
                  f"{per_tap} tap-streams ({per_tap / len(taps):.1f} per tap, at most "
                  f"{max(len(v) for v in taps.values())}): {sorted(union)}")
            for d in lr.launches(S, B, with_mask=mask, refine=mask):
                assert lr.last_tile_streams(d) <= taps[_name((d["side"], d["name"]))]
                assert d["s0"] + d["M"] // d["hw"] - 1 in taps[_name((d["side"], d["name"]))]
            assert max(len(v) for v in taps.values()) <= 16 and len(union) <= 72


def test_pass_streams_follow_the_tile_walk():
    """The pass streams of a GEMM launch in both M orders and of a patch launch, on a hand-checked case: search 255,
    B = 153 (lanes 77 + 76), layer3.0.conv3 (31 x 31 = 961 rows per stream, 1024 channels: 8 N tiles)."""
    d = next(d for d in lr.launches(255, 153) if d["side"] == "search" and d["lane"] == 1
             and d["name"] == "features.features.layer3.0.conv3")
    assert (d["s0"], d["hw"], d["ntile"], d["tiles"]) == (77, 961, 8, 571 * 8)
    # work item 132 -> M block 16 (rows 2048..): stream 77 + 2; reversed: block 554 (rows 70912..): stream 77 + 73;
    # work item 264 -> block 33 (rows 4224..): stream 77 + 4; reversed: block 537 (rows 68736..): stream 77 + 71
    assert lr.pass_streams(d) == {79, 150, 81, 148}
    p = next(d for d in lr.launches(255, 153) if d["side"] == "search" and d["lane"] == 0
             and d["name"] == "features.features.layer1.0.conv2")
    # 63 x 63 at RO = 2 rows per block: 32 blocks per image; items 132 and 264 start images 4 and 8
    assert (p["kernel"], p["ntile"]) == ("patch", 32) and lr.pass_streams(p) == {4, 8}


# ---------------------------------------------------------------------------------------------------- GPU
def _release(m=None):
    """Free engine m's device memory now, even if something still references the object (a traceback pytest keeps
    after a failure holds the test's frames), and return the cached blocks, so the next engine is not built beside it
    on a shared GPU."""
    if m is not None:
        torch.cuda.synchronize()
        m._destroy()
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()


def _fresh_engine(sd, label, **kw):
    """A new engine after the previous one is gone; prints the device memory it took."""
    _release()
    free0 = torch.cuda.mem_get_info()[0]
    m = _engine(sd, **kw)
    torch.cuda.synchronize()
    print(f"\n[memory] {label}: {(free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30:.2f} GiB (mem_get_info drop, "
          f"engine built)")
    return m, free0


def _frame_memory(label, free0):
    print(f"[memory] {label}: {(free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30:.2f} GiB (after the first call, "
          f"its outputs included)")


def _worst(cfg, t0):
    worst = collections.defaultdict(float)
    for c, _, fam, mode, raw, _ in TABLE:
        if c == cfg:
            worst[(fam, mode)] = max(worst[(fam, mode)], raw)
    print(f"[worst] {cfg:30s} " + "  ".join(f"{f}/{m} {v:.2e}" for (f, m), v in sorted(worst.items()))
          + f"  ({time.time() - t0:.0f} s)")


def _pos(B, S):
    R = (S - 127) // 8 + 1 + 8
    return np.array([[(5 * b) % R, (11 * b + 3) % R] for b in range(B)])


def _sd(calib_sd, with_mask):
    if with_mask:
        return calib_sd
    return {k: v for k, v in calib_sd.items() if not k.startswith(("mask_model.", "refine_model."))}


PLANNED = [(S, B, mask) for (S, mask) in ENGINES for B in PLAN[(S, mask)]]
# the smallest planned batch of each search size runs through step() with a permuted slot table
SLOTS = {(S, min(PLAN[(S, True)])) for S in (255, 383)}


def _slot_step(m, z, x, S, num_slots, seed):
    """template(z, slots=) into a permuted table of `num_slots` slots, then step(x, slots=) with the template slots in
    another order.  Returns (outputs, selected positions, kernel row of every step stream): step stream b reads the
    template of template stream kernel_rows[b]."""
    B = z.shape[0]
    rs = np.random.RandomState(seed)
    t_slots = rs.permutation(num_slots)[:B]                        # template stream j -> slot t_slots[j]
    s_slots = t_slots[rs.permutation(B)]                           # step stream b reads slot s_slots[b]
    m.template(z.cuda(), slots=torch.from_numpy(t_slots.astype(np.int32)).cuda())
    a, w, tsz = _consts(B, (S - 127) // 8 + 1 + 8)
    out = m.step(x.cuda(), a, w, tsz, 0.04, 0.4, refine=True, mask_head=True,
                 slots=torch.from_numpy(s_slots.astype(np.int32)).cuda())
    torch.cuda.synchronize()
    row_of_slot = {int(s): j for j, s in enumerate(t_slots)}
    return ({k: out[k] for k in ("cls", "loc", "mask", "refine")}, out["pos"].cpu().numpy(),
            [row_of_slot[int(s)] for s in s_slots])


PLANNED = [(S, B, mask) for (S, mask) in ENGINES for B in PLAN[(S, mask)]]
# the smallest planned batch of each search size runs through step() with a permuted slot table
SLOTS = {(S, min(PLAN[(S, True)])) for S in (255, 383)}


@gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("S,B,mask", PLANNED,
                         ids=[f"{S}-B{B}-{'sharp' if mask else 'rpn'}" for S, B, mask in PLANNED])
def test_planned_batches(calib_sd, S, B, mask, precision):
    t0 = time.time()
    sd = _sd(calib_sd, mask)
    kind = "sharp" if mask else "rpn"
    label = f"{S} {kind} max_batch={B} num_slots={2 * B} {precision}"
    m, free0 = _fresh_engine(sd, label, search_size=S, max_batch=B, num_slots=2 * B, mask=mask, precision=precision)
    try:
        z, x = synthetic_inputs(50 + B, B, S)
        taps = checked_streams(S, B, with_mask=mask)
        streams = sorted(set().union(*taps.values()))
        cfg = f"{precision} {S} {kind} B={B}"
        if not mask:
            m.template(z.cuda())
            cls, loc = m.track(x.cuda())
            torch.cuda.synchronize()
            run = Run(m, z, x, streams, np.zeros((B, 2), int), {"cls": cls, "loc": loc}, tap_streams=taps,
                      mutation_streams=[B - 1])
        elif (S, B) in SLOTS:
            cfg += " slots"
            outputs, pos, kernel_rows = _slot_step(m, z, x, S, 2 * B, B)
            # the template-side taps are checked at the same rows as the search side; the xcorr reads its template
            # kernels at the kernel rows of the checked step streams
            run = Run(m, z, x, streams, pos, outputs, kernel_rows=[kernel_rows[b] for b in streams], tap_streams=taps,
                      mutation_streams=[B - 1])
        else:
            pos = _pos(B, S)
            run = Run(m, z, x, streams, pos, _frame(m, z, x, pos), tap_streams=taps, mutation_streams=[B - 1])
        _frame_memory(label, free0)
        res = check(cfg, run, sd, precision, with_mask=mask, refine=mask)
        _worst(cfg, t0)
    finally:
        run = None
        _release(m)
    _assert(*res)


# one engine per (search size, precision), built for max_batch = num_slots streams, runs these batches in order
SEQUENCES = {255: (256, [256, 153, 16, 1, 153]), 383: (128, [128, 113, 19, 1])}


class StaleRows:
    """Mutation (d): the previous call's tensors at one stream read in place of this call's.  For each tap, the first
    pixel of the checked stream `stream` (the last one, which holds the last tile of every launch) that lies in its
    launch's last 128-row tile gives an output image row; that row is mapped to the tap's first input in proportion to
    the image heights, and the input rows from there to the bottom of the image are taken from the previous call.  That
    is a superset of the rows feeding the last tile (for the upsampling refine convs and the heads, an approximate one),
    which is enough for what the mutation shows: the previous call's inputs differ in every pixel."""

    def __init__(self, prev, run, stream, B, max_batch):
        self.prev, self.run, self.stream = prev, run, stream
        self.lane = {"template:": B, "": lane_split(B, max_batch)[-1]}

    def __call__(self, name, tap, fetch, streams):
        n0 = tap.inputs[0]
        if n0 == "pos" or lr.family(tap) == "exact":
            return None
        if self.stream not in streams:
            return None
        j = streams.index(self.stream)
        prefix = "template:" if name.startswith("template:") else ""
        src = n0 if n0 in ("x", "z") or not prefix else prefix + n0
        ho, wo = self.run.get(name).shape[-2:]
        b = self.lane[prefix]
        first = max(0, (-(-b * ho * wo // 128) - 1) * 128 - (b - 1) * ho * wo)   # first last-tile pixel of the stream
        x = fetch(n0).clone()
        y0 = (first // wo) * x.shape[-2] // ho
        x[j, :, y0:] = self.prev.get(src)[0, :, y0:].to(x.dtype)

        def stale_fetch(n):
            return x if n == n0 else fetch(n)
        return stale_fetch


def _inputs(i, B, S):
    """Call i's inputs: a seed per call, and every other call's images inverted, so that no stream of a call sees the
    previous call's pixels."""
    z, x = synthetic_inputs(60 + 7 * i, B, S)
    return (255.0 - z, 255.0 - x) if i % 2 else (z, x)


@gpu
@pytest.mark.parametrize("precision", ["exact", "fast"])
@pytest.mark.parametrize("S", sorted(SEQUENCES))
def test_shrinking_and_growing_batches(calib_sd, S, precision):
    """One engine built for max_batch = num_slots streams runs a shrinking and growing batch sequence as a queue does:
    template into a permuted slot table, then step() with the slots in another order, at every batch."""
    max_batch, seq = SEQUENCES[S]
    label = f"{S} sharp max_batch={max_batch} num_slots={max_batch} {precision}"
    m, free0 = _fresh_engine(calib_sd, label, search_size=S, max_batch=max_batch, num_slots=max_batch,
                             precision=precision)
    prev, run, outputs, fails = None, None, None, []
    try:
        for i, B in enumerate(seq):
            t0 = time.time()
            z, x = _inputs(i, B, S)
            outputs, pos, kernel_rows = _slot_step(m, z, x, S, max_batch, 100 + i)
            if i == 0:
                _frame_memory(label, free0)
            taps = checked_streams(S, B, max_batch)
            streams = sorted(set().union(*taps.values()))
            run = Run(m, z, x, streams, pos, outputs, kernel_rows=[kernel_rows[b] for b in streams],
                      tap_streams=taps, mutation_streams=[B - 1])
            cfg = f"{precision} {S} seq{i} B={B}" + (f" after {seq[i - 1]}" if i else "")
            res = check(cfg, run, calib_sd, precision,
                        stale=None if prev is None else StaleRows(prev, run, B - 1, B, max_batch))
            fails += [f"{cfg}: {f}" for f in res[0]] + [f"{cfg}: gate does not reject {f}" for f in res[1]]
            _worst(cfg, t0)
            if i + 1 < len(seq):
                # this call's tensors at the stream mutation (d) of the next call replaces (clamped into this call)
                s = min(seq[i + 1] - 1, B - 1)
                prev = Run(m, z, x, [s], pos, outputs)
                for tap, p in _tap_list("tensor", True, True, True):
                    n0 = tap.inputs[0]
                    if n0 != "pos":
                        prev.get(n0 if n0 in ("x", "z") or not p else p + n0)
                prev.m = prev.outputs = None
            run = outputs = None
    finally:
        prev = run = outputs = None
        _release(m)
    assert not fails, "\n".join(fails)
