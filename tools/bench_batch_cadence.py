"""The reference's whole main loop (swirld.py:319-328) for many node-views at its own cadence, a handful of events per
call.  Per turn every view appends and divides its next call, then one sw_batch_decide_fame and one sw_batch_find_order
run over all views.  Three loops over the same seeded views, alternated within one run after a warm-up:
    (a) per-view sw_append and sw_divide_rounds;
    (b) per-view sw_append, then one sw_batch_divide_rounds;
    (c) one sw_batch_append, then one sw_batch_divide_rounds.
Shapes: 64 members x 600 events, 3 per call, with B = 1, 8, 64 and 256 views; 256 members x 1536 events, 3 per call,
with B = 64.  Per shape and loop: ms per turn (device-synchronised wall time of a whole schedule over its turns; median
and min over the repetitions), events/s over all views, kernel launches per turn, and whether every loop left every view
with identical rounds, fame, consensus, order and idx.  Prints one JSON line per shape and writes them to
OUT_DIR/bench_batch_cadence.json.
    python tools/bench_batch_cadence.py [--reps R] [--shapes m64_b1,...] [--out OUT_DIR]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from bench_batch_consensus import card, launches  # noqa: E402
from swirld_b200 import engine, traces  # noqa: E402
from swirld_b200.traces import chunks  # noqa: E402

# name: (members, events per view, events per call, views)
SHAPES = {
    "m64_b1": (64, 600, 3, 1),
    "m64_b8": (64, 600, 3, 8),
    "m64_b64": (64, 600, 3, 64),
    "m64_b256": (64, 600, 3, 256),
    "m256_b64": (256, 1536, 3, 64),
}


def outputs(engs):
    return [(e.rounds(), e.famous(), e.consensus(), e.transactions(), e.idx()) for e in engs]


def run_shape(name, reps):
    M, N, K, B = SHAPES[name]
    trs = [traces.gossip(M, N, 1000 + v) for v in range(B)]
    engs = [engine.Engine(M, N) for _ in range(B)]
    sched = list(chunks(N, K))

    def cols(tr, first, cnt):
        s = slice(first, first + cnt)
        return (tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s])

    def consensus():
        engine.batch_find_order(engs, engine.batch_decide_fame(engs))

    def loop_a():
        for first, cnt in sched:
            for e, tr in zip(engs, trs):
                e.append_trace(tr, first, cnt)
                e.divide_rounds(first, cnt)
            consensus()

    def loop_b():
        for first, cnt in sched:
            for e, tr in zip(engs, trs):
                e.append_trace(tr, first, cnt)
            engine.batch_divide_rounds(engs, [first] * B, [cnt] * B)
            consensus()

    def loop_c():
        for first, cnt in sched:
            engine.batch_append(engs, [cols(tr, first, cnt) for tr in trs])
            engine.batch_divide_rounds(engs, [first] * B, [cnt] * B)
            consensus()

    loops = {"a": loop_a, "b": loop_b, "c": loop_c}
    times, nlaunch, outs = {k: [] for k in loops}, {}, {}
    for rep in range(reps + 1):                        # (rep 0 is the warm-up of every loop)
        order = list(loops)[rep % 3:] + list(loops)[:rep % 3]
        for arm in order:
            for e in engs:
                e.reset()
            l0 = launches(engs)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loops[arm]()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            nlaunch[arm] = launches(engs) - l0        # (sw_reset zeroes the counters: l0 is 0)
            if rep:
                times[arm].append(dt / len(sched))
            if rep == reps:
                outs[arm] = outputs(engs)
    same = all(all(all(np.array_equal(x, y) for x, y in zip(va, vb)) for va, vb in zip(outs["a"], outs[k]))
               for k in ("b", "c"))
    res = {"shape": name, "M": M, "events_per_view": N, "events_per_call": K, "views": B, "turns": len(sched),
           "identical_outputs": same}
    for arm in loops:
        t = times[arm]
        res[arm] = {"ms_per_turn_median": statistics.median(t) * 1e3, "ms_per_turn_min": min(t) * 1e3,
                    "events_per_s_median": B * K / statistics.median(t),
                    "kernel_launches_per_turn": nlaunch[arm] / len(sched)}
    res["speedup_median_a_to_c"] = res["a"]["ms_per_turn_median"] / res["c"]["ms_per_turn_median"]
    for e in engs:
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=4)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch_cadence: no CUDA device (the engine has no CPU path)")
    torch.cuda.set_device(0)
    name, limits = card()
    lines = []
    for s in args.shapes.split(","):
        r = run_shape(s, args.reps)
        r.update(card=name, power_limit_and_max_sm_clock=limits)
        print(json.dumps(r), flush=True)
        lines.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_batch_cadence.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
