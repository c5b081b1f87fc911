"""What the ingest stage of a turn costs for many node-views: B sw_ingest_verified calls against one
sw_batch_ingest_verified, which verifies each distinct event once however many views receive it.

A seeded signed gossip of M members (the reference's event shapes, swirld.py:88-95: msg = dumps((d, p, t, pk)),
preimage = dumps(Event(d, p, t, pk, sig)), id = BLAKE2b-256(preimage)), signed with PyNaCl before anything is timed.
Its source reveals `step` new events per turn; every turn each view ingests one reply, from a random peer view or from
the source: what that peer holds beyond the view's own events, shuffled.  The replies of every turn are built before
the timed window.  Two engine sets run the same turns, alternated turn by turn (which goes first alternates too):
    (a) B sw_ingest_verified calls, one per view;
    (b) one sw_batch_ingest_verified over the B views.
Shapes: B = 1, 16 and 64 views at M = 64, and B = 256 at M = 16.  Per shape and loop: ms per turn (device-synchronised
wall time: the calls, then every engine of the set synchronised; median and min over the timed turns), events received
and events verified on the GPU per turn, kernel launches per turn, and whether both sets ended with identical events,
heights and id maps.  The card's name, power limit and max SM clock come from a read-only nvidia-smi query in the same
run.  Prints one JSON line per shape and writes them to OUT_DIR/bench_batch_ingest.json.
    python tools/bench_batch_ingest.py [--turns T] [--warmup W] [--shapes m64_b1,...] [--out OUT_DIR]"""
import argparse
import hashlib
import json
import os
import pickle
import random
import statistics
import sys
import time
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
import numpy as np  # noqa: E402
from nacl import bindings as nb  # noqa: E402

Event = namedtuple("Event", "d p t c s")

SHAPES = {                     # members, views, events the source reveals per turn
    "m64_b1": (64, 1, 64),
    "m64_b16": (64, 16, 64),
    "m64_b64": (64, 64, 64),
    "m16_b256": (16, 256, 32),
}


def gossip(M, n, seed):
    """n signed events of M members in creation order: (id, Event, msg, preimage, member)."""
    rng = random.Random(seed)
    keys = [nb.crypto_sign_seed_keypair(rng.randbytes(32)) for _ in range(M)]
    heads, evs, t = [None] * M, [], 1.7e9

    def make(c, p):
        nonlocal t
        t += rng.random()
        d = None if rng.random() < 0.7 else [rng.randbytes(8)]
        pk, sk = keys[c]
        msg = pickle.dumps((d, p, t, pk))
        ev = Event(d, p, t, pk, nb.crypto_sign(msg, sk)[:64])
        pre = pickle.dumps(ev)
        h = hashlib.blake2b(pre, digest_size=32).digest()
        heads[c] = h
        evs.append((h, ev, msg, pre, c))

    for c in range(M):
        make(c, ())
    while len(evs) < n:
        c = rng.randrange(M)
        make(c, (heads[c], heads[rng.choice([x for x in range(M) if x != c])]))
    return [k[0] for k in keys], evs


def replies(evs, B, step, turns, seed):
    """Per turn, per view, the rows it receives (every event is valid, so a view then knows all it received)."""
    rng = random.Random(seed)
    known = [set() for _ in range(B)]
    out, F = [], 0
    for _ in range(turns):
        F = min(len(evs), F + step)
        src = {x[0] for x in evs[:F]}
        rows = []
        for v in range(B):
            u = rng.randrange(B + 1)
            have = src if u == B or u == v else known[u]
            r = [x for x in evs if x[0] in have and x[0] not in known[v]]
            rng.shuffle(r)
            rows.append(r)
        for v in range(B):
            known[v].update(x[0] for x in rows[v])
        out.append(rows)
    return out


def columns(items):
    zero = bytes(32)
    cat = lambda parts: np.frombuffer(b"".join(parts), np.uint8) if parts else np.zeros(0, np.uint8)
    return (cat([x[0] for x in items]), cat([x[1].p[0] if x[1].p else zero for x in items]),
            cat([x[1].p[1] if x[1].p else zero for x in items]), np.array([x[4] for x in items], np.int32),
            np.array([x[1].t for x in items], np.float64), cat([x[1].s for x in items]),
            [x[2] for x in items], [x[3] for x in items])


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:            # (the power limit is part of the number: say that it could not be read)
        return "unknown (%s)" % ex


def run_shape(name, turns, warmup, seed):
    from swirld_b200 import engine as E
    M, B, step = SHAPES[name]
    total = warmup + turns
    pks, evs = gossip(M, step * total + M, seed)
    plan = replies(evs, B, step, total, seed)
    cols = [[columns(r) for r in rows] for rows in plan]
    sets = []
    for _ in range(2):
        engs = [E.Engine(M, len(evs) + 16) for _ in range(B)]
        for e in engs:
            e.set_member_keys(pks)
        sets.append(engs)
    single, batched = sets

    def loop_a(i):
        n = 0
        for e, c in zip(single, cols[i]):
            e.ingest(*c[:6], msgs=c[6], preimages=c[7])
            n += len(c[6])
        for e in single:
            e.sync()
        return n

    def loop_b(i):
        _, nv = E.batch_ingest(batched, cols[i])
        for e in batched:
            e.sync()
        return nv

    def launches(engs):
        return sum(e.stats()["kernel_launches"] for e in engs)

    ms = {"a": [], "b": []}
    ver = {"a": 0, "b": 0}
    la = {"a": 0, "b": 0}
    received = 0
    for i in range(total):
        order = ("a", "b") if i % 2 == 0 else ("b", "a")
        for k in order:
            engs = single if k == "a" else batched
            l0 = launches(engs)
            t0 = time.perf_counter()
            nv = (loop_a if k == "a" else loop_b)(i)
            dt = (time.perf_counter() - t0) * 1e3
            if i >= warmup:
                ms[k].append(dt)
                ver[k] += nv
                la[k] += launches(engs) - l0
        if i >= warmup:
            received += sum(len(r) for r in plan[i])
    ids = np.frombuffer(b"".join(x[0] for x in evs), np.uint8)
    same = all(a.n_events == b.n_events and np.array_equal(a.heights(), b.heights()) and
               np.array_equal(a.lookup(ids), b.lookup(ids)) for a, b in zip(single, batched))
    out = {"shape": name, "members": M, "views": B, "turns": turns, "warmup": warmup,
           "events_received_per_turn": received / turns, "identical_state": bool(same)}
    for k, what in (("a", "single"), ("b", "batched")):
        out[what] = {"ms_per_turn_median": round(statistics.median(ms[k]), 3), "ms_per_turn_min": round(min(ms[k]), 3),
                     "verified_per_turn": ver[k] / turns, "launches_per_turn": la[k] / turns}
    out["speedup_median"] = round(statistics.median(ms["a"]) / statistics.median(ms["b"]), 2)
    for engs in sets:
        for e in engs:
            e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--turns", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default="", help="directory for bench_batch_ingest.json (the lines are printed either way)")
    args = ap.parse_args()
    gpu = card()
    lines = []
    for name in args.shapes.split(","):
        r = run_shape(name, args.turns, args.warmup, args.seed)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
        lines.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_batch_ingest.json"), "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
