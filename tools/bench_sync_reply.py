"""What the sending end of a sync costs for many node-views: B sync replies built in Python per turn against one
sw_batch_sync_reply, which selects every view's reply on the GPU from its can_see rows.

Each view is an engine that ingested one member's view of a seeded gossip (traces.node_view) under ids made from
(creator, chain position).  Every turn each view answers one requester: in the steady shapes the summary of another
member's view a few events behind its head (a peer that synced recently), in the catch-up shape the empty summary of a
fresh requester, so the reply is the whole view.  Two loops answer the same requests, alternated turn by turn (which
goes first alternates too):
    (a) Python: ask_sync restated over host dicts of each view (parents, creator, height, id, t, sig), as the batched
        drivers build replies today: a BFS from the head over the parents the requester lacks, then the rows;
    (b) one batch_sync_reply over the B views, rows included (ids, parent ids, creator, t, sig).
Shapes: tools/bench_batch_ingest.py's (B = 1, 16 and 64 views at M = 64; B = 256 at M = 16) with views of 40 M
events, and the catch-up: 8 views of 262 144 events at M = 64.  Per shape and loop: ms per turn (wall time around the
calls, which end in a device synchronisation; median and min over the timed turns), events sent per turn, kernel
launches per turn, and whether both loops sent the same rows.  The card's name, power limit and max SM clock come from
a read-only nvidia-smi query in the same run.  Prints one JSON line per shape and writes them to
OUT_DIR/bench_sync_reply.json.
    python tools/bench_sync_reply.py [--turns T] [--warmup W] [--shapes m64_b1,...] [--out OUT_DIR]"""
import argparse
import hashlib
import json
import os
import random
import statistics
import sys
import time
from collections import deque

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
import numpy as np  # noqa: E402

SHAPES = {                     # members, views, events per view (None: the catch-up's 262 144-event gossip)
    "m64_b1": (64, 1, 40 * 64),
    "m64_b16": (64, 16, 40 * 64),
    "m64_b64": (64, 64, 40 * 64),
    "m16_b256": (16, 256, 40 * 16),
    "catchup_m64_b8": (64, 8, None),
}
CATCHUP_TURNS = 3              # the Python loop takes seconds per turn there


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:            # (the power limit is part of the number: say that it could not be read)
        return "unknown (%s)" % ex


def chain_ids(tr):
    seq, cnt = [], {}
    for c in tr.creator.tolist():
        seq.append(cnt.get(c, 0))
        cnt[c] = seq[-1] + 1
    return np.frombuffer(b"".join(hashlib.blake2b(b"%d:%d" % (c, s), digest_size=32).digest()
                                  for c, s in zip(tr.creator.tolist(), seq)), np.uint8).reshape(-1, 32)


class HostView:
    """One view as the host drivers keep it: per event its parents, creator, height, id, t and signature."""

    def __init__(self, tr):
        from swirld_b200 import traces
        self.tr, self.M = tr, tr.M
        self.ids = chain_ids(tr)
        self.p0, self.p1, self.creator = tr.p0.tolist(), tr.p1.tolist(), tr.creator.tolist()
        self.height = traces.heights(tr).tolist()
        z = np.zeros((1, 32), np.uint8)
        pick = lambda p: np.where((p >= 0)[:, None], self.ids[np.maximum(p, 0)], z)
        self.p0_ids, self.p1_ids = pick(tr.p0), pick(tr.p1)
        self.row = traces.can_see_rows(tr) if tr.N <= 1 << 14 else None

    def summary(self, head):
        if head < 0:
            return np.full(self.M, -1, np.int32)
        r = self.row[head]
        h = np.asarray(self.height, np.int32)
        return np.where(r >= 0, h[np.maximum(r, 0)], -1).astype(np.int32)

    def reply(self, head, S):
        """ask_sync (swirld.py:154-161): bfs from head over the parents p with S[creator p] = -1 or height[p] > it."""
        seen, q = {head}, deque([head])
        p0, p1, cr, hg = self.p0, self.p1, self.creator, self.height
        while q:
            u = q.popleft()
            if p0[u] < 0:
                continue
            for p in (p0[u], p1[u]):
                if p not in seen and (S[cr[p]] < 0 or hg[p] > S[cr[p]]):
                    seen.add(p)
                    q.append(p)
        idx = np.array(sorted(seen), np.int64)
        tr = self.tr
        return idx, (self.ids[idx], self.p0_ids[idx], self.p1_ids[idx], tr.creator[idx], tr.t[idx], tr.sig[idx])


def build(name, seed):
    from swirld_b200 import engine as E, traces
    M, B, n = SHAPES[name]
    if n is None:
        base = traces.gossip_np(M, 1 << 18, seed=seed)
        hosts = [HostView(base)] * B
    else:
        base = traces.gossip(M, n * 2, seed=seed)
        hosts = []
        for X in range(min(B, M)):
            tr, _ = traces.node_view(base, X)
            hosts.append(HostView(tr.slice(0, min(tr.N, n))))
        hosts = [hosts[v % len(hosts)] for v in range(B)]
    engs = []
    for h in hosts:
        e = E.Engine(M, h.tr.N)
        e.ingest(h.ids, h.p0_ids, h.p1_ids, h.tr.creator, h.tr.t, h.tr.sig)
        e.divide_rounds(0, h.tr.N)
        e.sync()
        engs.append(e)
    return hosts, engs


def run_shape(name, turns, warmup, seed):
    from swirld_b200 import engine as E
    M, B, n = SHAPES[name]
    if n is None:
        turns, warmup = min(turns, CATCHUP_TURNS), min(warmup, 1)
    hosts, engs = build(name, seed)
    rng = random.Random(seed)
    total = warmup + turns
    plan = []                  # per turn: heads, summaries
    for _ in range(total):
        heads = [h.tr.N - 1 for h in hosts]
        if n is None:
            sums = [np.full(M, -1, np.int32)] * B
        else:
            sums = []
            for v in range(B):
                w = hosts[rng.randrange(len(hosts))]
                sums.append(w.summary(w.tr.N - 1 - rng.randrange(2 * M)))
        plan.append((heads, sums))

    def loop_a(i):
        heads, sums = plan[i]
        return [h.reply(x, s) for h, x, s in zip(hosts, heads, sums)]

    def loop_b(i):
        heads, sums = plan[i]
        idx, cols = E.batch_sync_reply(engs, heads, sums)
        return list(zip(idx, cols))

    ms = {"a": [], "b": []}
    sent, same, launches = 0, True, 0
    for i in range(total):
        res = {}
        for k in (("a", "b") if i % 2 == 0 else ("b", "a")):
            l0 = engs[0].stats()["kernel_launches"]
            t0 = time.perf_counter()
            res[k] = (loop_a if k == "a" else loop_b)(i)
            dt = (time.perf_counter() - t0) * 1e3
            if i >= warmup:
                ms[k].append(dt)
                if k == "b":
                    launches += engs[0].stats()["kernel_launches"] - l0
        if i >= warmup:
            sent += sum(len(r[0]) for r in res["a"])
        for (ia, ca), (ib, cb) in zip(res["a"], res["b"]):
            same = same and np.array_equal(ia, ib) and all(np.array_equal(x, y) for x, y in zip(ca, cb))
    out = {"shape": name, "members": M, "views": B, "events_per_view": hosts[0].tr.N, "turns": turns,
           "warmup": warmup, "events_sent_per_turn": sent / turns, "identical_rows": bool(same)}
    for k, what in (("a", "python"), ("b", "batched")):
        out[what] = {"ms_per_turn_median": round(statistics.median(ms[k]), 3), "ms_per_turn_min": round(min(ms[k]), 3)}
    out["batched"]["launches_per_turn"] = launches / turns
    out["speedup_median"] = round(statistics.median(ms["a"]) / statistics.median(ms["b"]), 2)
    for e in engs:
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--turns", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default="", help="directory for bench_sync_reply.json (the lines are printed either way)")
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
        with open(os.path.join(args.out, "bench_sync_reply.json"), "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
