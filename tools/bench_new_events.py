"""What a turn's own new events cost: one sw_batch_new_events (Ed25519 signatures and BLAKE2b ids on the GPU, the events
entered into each view) against a host loop (libsodium's crypto_sign through PyNaCl, hashlib BLAKE2b, one sw_ingest
per view).

Shapes: one event per view at B = 1, 16, 64 (M = 64) and 256 (M = 16); and 2^16 events by 64 members in one call
(sign and hash only, against libsodium and hashlib on one host core) for throughput.  Each turn every view makes its
member's root event and the views are reset after the turn, so every turn signs, hashes and appends B events.  The two
loops alternate, turn by turn, on twin sets of views, and must give the same ids; prints one JSON line with median (min) ms per turn and the card's name and power limit
(read-only nvidia-smi query, same run).
    python tools/bench_new_events.py [--turns T] [--out OUT_DIR]"""
import argparse
import hashlib
import json
import os
import random
import statistics
import subprocess
import sys
import time
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
import numpy as np  # noqa: E402
from nacl import bindings as nb  # noqa: E402

from swirld_b200 import engine as E  # noqa: E402
from swirld_b200.events import event_template  # noqa: E402

Event = namedtuple("Event", "d p t c s")


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        return "unknown (%s)" % ex


def views(M, B, kp):
    V = []
    for v in range(B):
        e = E.Engine(M, 1 << 14)
        e.set_member_keys([pk for pk, _ in kp])
        e.set_signing_key(v % M, kp[v % M][1])
        V.append(e)
    return V


def turn_rows(kp, M, B, turn):
    """View v's root event of this turn."""
    z = np.zeros((1, 32), np.uint8)
    ts = [[1.0 + turn + v * 1e-3] for v in range(B)]
    tms = [[event_template(Event, None, (), ts[v][0], kp[v % M][0])] for v in range(B)]
    return tms, [z] * B, [z] * B, ts


def gpu_turn(V, rows):
    tms, p0, p1, ts = rows
    res = E.batch_new_events(V, tms, p0, p1, ts)
    return [bytes(r[1][0]) for r in res]


def host_turn(V, kp, M, rows):
    tms, p0, p1, ts = rows
    out = []
    for v, e in enumerate(V):
        msg, pre, at = tms[v][0]
        sig = nb.crypto_sign(msg, kp[v % M][1])[:64]
        full = pre[:at] + sig + pre[at + 64:]
        h = hashlib.blake2b(full, digest_size=32).digest()
        e.ingest(np.frombuffer(h, np.uint8), p0[v], p1[v], [v % M], ts[v], np.frombuffer(sig, np.uint8))
        out.append(h)
    return out


def per_turn(M, B, turns, kp):
    """One event per view and turn, median (min) ms per turn of each loop after two warm-up turns."""
    Vg, Vh = views(M, B, kp), views(M, B, kp)
    tg, th = [], []
    for turn in range(turns + 2):
        rows = turn_rows(kp, M, B, turn)
        for who in ((0, 1) if turn % 2 else (1, 0)):
            t0 = time.perf_counter()
            if who == 0:
                ids_g = gpu_turn(Vg, rows)
            else:
                ids_h = host_turn(Vh, kp, M, rows)
            (tg if who == 0 else th).append(1e3 * (time.perf_counter() - t0))
        assert ids_g == ids_h
        for e in Vg + Vh:
            e.reset()
    tg, th = tg[2:], th[2:]
    return {"M": M, "B": B, "gpu_ms": [statistics.median(tg), min(tg)], "host_ms": [statistics.median(th), min(th)],
            "speedup_median": statistics.median(th) / statistics.median(tg)}


def throughput(n, M, kp):
    e = views(M, 1, kp)[0]
    tms = [event_template(Event, None, (), float(i), kp[0][0]) for i in range(n)]
    e.new_events(tms[:1024], ingest=False)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        sig, ids = e.new_events(tms, ingest=False)
        ts.append(1e3 * (time.perf_counter() - t0))
    k = 2048
    t0 = time.perf_counter()
    for msg, pre, at in tms[:k]:
        s = nb.crypto_sign(msg, kp[0][1])[:64]
        hashlib.blake2b(pre[:at] + s + pre[at + 64:], digest_size=32).digest()
    host_ms = 1e3 * (time.perf_counter() - t0) * n / k
    assert bytes(sig[7]) == nb.crypto_sign(tms[7][0], kp[0][1])[:64]
    return {"n": n, "gpu_ms": [statistics.median(ts), min(ts)], "host_one_core_ms_est": host_ms,
            "gpu_events_per_s": n / (min(ts) / 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--turns", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rng = random.Random(1)
    kp = [nb.crypto_sign_seed_keypair(bytes(rng.randrange(256) for _ in range(32))) for _ in range(64)]
    res = {"card": card(), "turns": a.turns, "shapes": []}
    for M, B in ((64, 1), (64, 16), (64, 64), (16, 256)):
        res["shapes"].append(per_turn(M, B, a.turns, kp[:M]))
    res["throughput"] = throughput(1 << 16, 64, kp)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_new_events.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
