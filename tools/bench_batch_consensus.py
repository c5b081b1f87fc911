"""What batching decide_fame and find_order over node-views saves: two loops over the same seeded views, alternated
within one run.
    (a) per chunk: sw_batch_divide_rounds (per-view sw_divide_rounds above 64 members), then decide_fame and find_order
        one view after the other -- what a simulation of the reference's main loop (swirld.py:325-328) did so far;
    (b) per chunk: the same divide, then one sw_batch_decide_fame and one sw_batch_find_order over all views.
Shapes: C3 views (64 members, 262 144 events per view, chunks of 65 536) with B = 1, 8 and 32; the reference's cadence
(64 members, 3 events per call) with B = 64; 256-member views (per-view divide_rounds) with B = 8.
Per shape and loop: device-synchronised wall time per step (min and median over the repetitions), events/s over all
views, kernel launches per step, and whether (a) and (b) left every view with identical rounds, fame, consensus and
order.  Prints one JSON line per shape and writes them to OUT_DIR/bench_batch_consensus.json.
    python tools/bench_batch_consensus.py [--reps R] [--shapes c3_b1,...] [--out OUT_DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from swirld_b200 import engine, traces  # noqa: E402
from swirld_b200.traces import chunks  # noqa: E402

# name: (members, events per view, events per call, views, one sw_batch_divide_rounds for all views)
SHAPES = {
    "c3_b1": (64, 262144, 65536, 1, True),
    "c3_b8": (64, 262144, 65536, 8, True),
    "c3_b32": (64, 262144, 65536, 32, True),
    "cadence_b64": (64, 600, 3, 64, True),
    "m256_b8": (256, 131072, 32768, 8, False),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:            # (the power limit is part of the number: say that it could not be read)
        q = "unknown (%s)" % ex
    return name, q


def launches(engs):
    return sum(e.stats()["kernel_launches"] for e in engs)


def outputs(engs):
    return [(e.rounds(), e.famous(), e.consensus(), e.transactions(), e.idx()) for e in engs]


def run_shape(name, reps):
    M, N, K, B, batch_div = SHAPES[name]
    gen = traces.gossip_np if N >= 4096 else traces.gossip
    trs = [gen(M, N, 1000 + v) for v in range(B)]
    engs = [engine.Engine(M, N) for _ in range(B)]
    for e, tr in zip(engs, trs):
        e.append_trace(tr)
    sched = list(chunks(N, K))

    def divide(first, cnt):
        if batch_div:
            engine.batch_divide_rounds(engs, [first] * B, [cnt] * B)
        else:
            for e in engs:
                e.divide_rounds(first, cnt)

    def step_a():
        for first, cnt in sched:
            divide(first, cnt)
            for e in engs:
                e.find_order(e.decide_fame())

    def step_b():
        for first, cnt in sched:
            divide(first, cnt)
            engine.batch_find_order(engs, engine.batch_decide_fame(engs))

    times, nlaunch, outs = {"a": [], "b": []}, {}, {}
    for rep in range(reps + 1):                        # (rep 0 is the warm-up of both loops)
        for arm, step in (("a", step_a), ("b", step_b)) if rep % 2 == 0 else (("b", step_b), ("a", step_a)):
            for e in engs:
                e.rewind()
            l0 = launches(engs)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            nlaunch[arm] = launches(engs) - l0
            if rep:
                times[arm].append(dt)
            if rep == reps:
                outs[arm] = outputs(engs)
    same = all(all(np.array_equal(x, y) for x, y in zip(va, vb)) for va, vb in zip(outs["a"], outs["b"]))
    res = {"shape": name, "M": M, "events_per_view": N, "events_per_call": K, "views": B,
           "divide": "sw_batch_divide_rounds" if batch_div else "sw_divide_rounds per view",
           "calls_per_step": len(sched), "identical_outputs": same}
    for arm in ("a", "b"):
        t = times[arm]
        res[arm] = {"ms_min": min(t) * 1e3, "ms_median": statistics.median(t) * 1e3,
                    "events_per_s_median": B * N / statistics.median(t), "kernel_launches_per_step": nlaunch[arm]}
    res["speedup_median"] = res["a"]["ms_median"] / res["b"]["ms_median"]
    for e in engs:
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch_consensus: no CUDA device (the engine has no CPU path)")
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
        with open(os.path.join(args.out, "bench_batch_consensus.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
