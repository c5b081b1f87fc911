"""What reading the order costs a driver that keeps every node-view's `transactions`, in the reference's main loop
(swirld.py:319-328) for many views at its own cadence, on the shapes of tools/bench_batch_cadence.py.  Two loops over
the same seeded views, alternated within one run after a warm-up:
    (c) bench_batch_cadence's loop (c) -- one sw_batch_append, sw_batch_divide_rounds, sw_batch_decide_fame and
        sw_batch_find_order per turn -- plus, for every view that ordered something, one sw_get_transactions of its new
        events (a copy and a synchronisation each);
    (d) the same loop with sw_batch_find_order_out, which brings every view's new events (with their consensus times
        and rounds received) back in the copy sw_batch_find_order makes anyway.
Per shape and loop: ms per turn (device-synchronised wall time of a whole schedule over its turns; median and min over
the repetitions), kernel launches per turn, device-to-host copies per turn (each one synchronises the host) and bytes
copied back per turn; and whether both loops left every view with identical transactions, consensus times and rounds
received (and loop (d)'s outputs equal to them).  Prints the card and its power limit, one JSON line per shape, and
writes them to OUT_DIR/bench_order_output.json.
    python tools/bench_order_output.py [--reps R] [--shapes m64_b1,...] [--out OUT_DIR]"""
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
from bench_batch_cadence import SHAPES as CADENCE_SHAPES  # noqa: E402
from bench_batch_consensus import card, launches  # noqa: E402
from swirld_b200 import engine, traces  # noqa: E402
from swirld_b200.traces import chunks  # noqa: E402

# bench_batch_cadence's shapes reach no consensus within their 600 / 1536 events per view; the 16-member views of 2400
# events order most of them, which is what a driver that keeps `transactions` pays for
SHAPES = dict({k: CADENCE_SHAPES[k] for k in ("m64_b1", "m64_b64", "m64_b256", "m256_b64")},
              m16_b1=(16, 2400, 3, 1), m16_b64=(16, 2400, 3, 64), m16_b256=(16, 2400, 3, 256))


def run_shape(name, reps):
    M, N, K, B = SHAPES[name]
    trs = [traces.gossip(M, N, 1000 + v) for v in range(B)]
    engs = [engine.Engine(M, N) for _ in range(B)]
    sched = list(chunks(N, K))
    kept = [[] for _ in range(B)]                      # each view's transactions, as a driver keeps them
    copies = [0]

    def cols(tr, first, cnt):
        s = slice(first, first + cnt)
        return (tr.p0[s], tr.p1[s], tr.creator[s], tr.t[s], tr.sig[s])

    def step(first, cnt):
        engine.batch_append(engs, [cols(tr, first, cnt) for tr in trs])
        engine.batch_divide_rounds(engs, [first] * B, [cnt] * B)
        ncs = engine.batch_decide_fame(engs)
        copies[0] += 1
        return ncs

    def loop_c():
        for first, cnt in sched:
            ncs = step(first, cnt)
            added = engine.batch_find_order(engs, ncs)
            copies[0] += 1
            for v, n in enumerate(added):
                if n:
                    kept[v].extend(engs[v].transactions(len(kept[v]), n).tolist())
                    copies[0] += 1

    def loop_d():
        for first, cnt in sched:
            ncs = step(first, cnt)
            got = engine.batch_find_order_out(engs, ncs)
            copies[0] += 1
            for v, (ev, ts, rr) in enumerate(got):
                kept[v].extend(ev.tolist())
                copies[0] += len(ev) > 1024          # (a view past the window adds one round trip per call)

    loops = {"c": loop_c, "d": loop_d}
    times, res_arm, outs = {k: [] for k in loops}, {}, {}
    for rep in range(reps + 1):                        # (rep 0 is the warm-up of both loops)
        order = list(loops)[rep % 2:] + list(loops)[:rep % 2]
        for arm in order:
            for e in engs:
                e.reset()
            for k in kept:
                k.clear()
            copies[0] = 0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loops[arm]()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            st = [e.stats() for e in engs]
            res_arm[arm] = {"kernel_launches_per_turn": launches(engs) / len(sched),
                            "d2h_copies_per_turn": copies[0] / len(sched),
                            "d2h_bytes_per_turn": sum(s["d2h_bytes"] for s in st) / len(sched)}
            if rep:
                times[arm].append(dt / len(sched))
            if rep == reps:
                outs[arm] = [(e.transactions(), e.consensus_times(), e.rounds_received(), list(k))
                             for e, k in zip(engs, kept)]
    same = all(np.array_equal(a[0], b[0]) and a[1].tobytes() == b[1].tobytes() and np.array_equal(a[2], b[2])
               and a[3] == a[0].tolist() and b[3] == b[0].tolist() for a, b in zip(outs["c"], outs["d"]))
    res = {"shape": name, "M": M, "events_per_view": N, "events_per_call": K, "views": B, "turns": len(sched),
           "ordered_per_view": float(np.mean([len(o[0]) for o in outs["d"]])),
           "identical_outputs": same}
    for arm in loops:
        t = times[arm]
        res[arm] = dict(res_arm[arm], ms_per_turn_median=statistics.median(t) * 1e3, ms_per_turn_min=min(t) * 1e3)
    res["speedup_median_c_to_d"] = res["c"]["ms_per_turn_median"] / res["d"]["ms_per_turn_median"]
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
        sys.exit("bench_order_output: no CUDA device (the engine has no CPU path)")
    torch.cuda.set_device(0)
    name, limits = card()
    print("card: %s, power limit and max SM clock: %s" % (name, limits), flush=True)
    lines = []
    for s in args.shapes.split(","):
        r = run_shape(s, args.reps)
        r.update(card=name, power_limit_and_max_sm_clock=limits)
        print(json.dumps(r), flush=True)
        lines.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_order_output.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
