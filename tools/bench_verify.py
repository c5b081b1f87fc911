"""What checking incoming events costs: sw_verify_events (Ed25519 signature with libsodium's verdicts + BLAKE2b-256 id,
swirld.py:97-103) against libsodium on the host.

N events (default 2^20) by M members (default 64), shaped like the reference's: msg = dumps((None, (h0, h1), t, pk)),
preimage = dumps(Event(None, (h0, h1), t, pk, sig)), id = BLAKE2b-256(preimage); signed in this run from a seed, over
all host cores.  1 % of them are tampered with (one bit of the signature).  Prints one JSON line (also written to
OUT_DIR/bench_verify.json with --out) with:
  - the card's name, power limit and max SM clock (read-only nvidia-smi query, same run);
  - sw_verify_events per call, after one warm-up call, over five timed calls (median, min, max): end to end on the
    host clock (the call synchronises) and device time between sw_event_record slots around it;
  - libsodium's crypto_sign_open (PyNaCl) on one host core over a subset, and on all host cores over every event (the
    verdicts every GPU flag is checked against);
  - hashlib BLAKE2b-256 of every preimage on one core;
  - with --profile, one more call under torch.profiler: each kernel's and copy's device time.
    python tools/bench_verify.py [--n N] [--members M] [--subset K] [--out OUT_DIR] [--profile]"""
import argparse
import json
import multiprocessing as mp
import os
import pickle
import random
import statistics
import sys
import time
from collections import namedtuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import hashlib  # noqa: E402

import numpy as np  # noqa: E402
from nacl import bindings as nb  # noqa: E402
from nacl import exceptions as nexc  # noqa: E402

Event = namedtuple("Event", "d p t c s")


def _keys(seed, M):
    rng = random.Random(seed)
    return [nb.crypto_sign_seed_keypair(rng.randbytes(32)) for _ in range(M)]


def _make(args):
    """Events [lo, hi): (creator, sig, msg, preimage, id), the signature of 1 in 100 flipped in one bit."""
    seed, M, lo, hi = args
    keys = _keys(seed, M)
    rng = random.Random(seed * 1000003 + lo)
    out = []
    for i in range(lo, hi):
        c = i % M
        pk, sk = keys[c]
        p = (rng.randbytes(32), rng.randbytes(32))
        t = 1.7e9 + i * 1e-3
        msg = pickle.dumps((None, p, t, pk))
        sig = nb.crypto_sign(msg, sk)[:64]
        pre = pickle.dumps(Event(None, p, t, pk, sig))
        id_ = hashlib.blake2b(pre, digest_size=32).digest()
        if rng.random() < 0.01:
            b = bytearray(sig)
            b[rng.randrange(64)] ^= 1 << rng.randrange(8)
            sig = bytes(b)
        out.append((c, sig, msg, pre, id_))
    return out


def _nacl(args):
    """libsodium's verdict on each (sig, msg, pk)."""
    out = []
    for sig, msg, pk in args:
        try:
            nb.crypto_sign_open(sig + msg, pk)
            out.append(1)
        except nexc.CryptoError:
            out.append(0)
    return out


def _chunks(n, k):
    step = (n + k - 1) // k
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def card():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:            # (the power limit is part of the number: say that it could not be read)
        return "unknown (%s)" % ex


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--members", type=int, default=64)
    ap.add_argument("--subset", type=int, default=20000, help="events libsodium verifies on one core")
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default="", help="directory for bench_verify.json (the JSON line is printed either way)")
    ap.add_argument("--profile", action="store_true", help="then one more call under torch.profiler: kernel and copy times")
    a = ap.parse_args()
    from swirld_b200 import engine
    N, M = a.n, a.members
    cores = os.cpu_count() or 1
    res = {"card": card(), "n": N, "members": M, "host_cores": cores}

    t0 = time.perf_counter()
    with mp.Pool(cores) as pool:
        evs = [e for part in pool.map(_make, [(a.seed, M, lo, hi) for lo, hi in _chunks(N, 4 * cores)]) for e in part]
    res["s_make"] = time.perf_counter() - t0
    pks = [k[0] for k in _keys(a.seed, M)]
    triples = [(sig, msg, pks[c]) for c, sig, msg, _, _ in evs]

    # libsodium: one core over a subset, all cores over every event (the verdicts the GPU's are checked against)
    sub = triples[:a.subset]
    t0 = time.perf_counter()
    _nacl(sub)
    res["nacl_1core_ev_per_s"] = len(sub) / (time.perf_counter() - t0)
    t0 = time.perf_counter()
    with mp.Pool(cores) as pool:
        want_sig = [v for part in pool.map(_nacl, [triples[lo:hi] for lo, hi in _chunks(N, 4 * cores)]) for v in part]
    res["nacl_allcores_ev_per_s"] = N / (time.perf_counter() - t0)
    t0 = time.perf_counter()
    digests = [hashlib.blake2b(pre, digest_size=32).digest() for _, _, _, pre, _ in evs]
    res["blake2b_1core_ev_per_s"] = N / (time.perf_counter() - t0)
    want = np.array([s | (int(d == e[4]) << 1) for s, d, e in zip(want_sig, digests, evs)], np.uint8)
    res["tampered"] = int((want != 3).sum())

    # the GPU call on prepacked columns (what a host that batches a sync's events hands over)
    e = engine.Engine(M, 16)
    e.set_member_keys(pks)
    cr = np.array([x[0] for x in evs], np.int32)
    sig = np.frombuffer(b"".join(x[1] for x in evs), np.uint8)
    (msg, moff), (pre, poff) = engine._packed([x[2] for x in evs]), engine._packed([x[3] for x in evs])
    ids = np.frombuffer(b"".join(x[4] for x in evs), np.uint8)
    out = np.zeros(N, np.uint8)
    P = engine._ptr

    def call():
        e._chk(e._lib.sw_verify_events(e._h, N, P(cr), P(sig), P(msg), P(moff), P(pre), P(poff), P(ids), P(out)))

    call()                                                   # warm-up (module load, buffer growth)
    host_ms, dev_ms, ok = [], [], True
    for _ in range(a.calls):
        out[:] = 0
        e.record(0)
        t0 = time.perf_counter()
        call()
        host_ms.append((time.perf_counter() - t0) * 1e3)
        e.record(1)
        dev_ms.append(e.elapsed_ms(0, 1))
        ok &= bool(np.array_equal(out, want))
    res["verdicts_equal_libsodium"] = ok
    res["bytes_in_per_call"] = int(msg.size + pre.size + sig.size + ids.size + cr.size * 4 + (moff.size + poff.size) * 8)
    for k, v in (("host_ms", host_ms), ("device_ms", dev_ms)):
        res[k] = {"median": statistics.median(v), "min": min(v), "max": max(v), "all": v}
    res["gpu_ev_per_s_end_to_end"] = N / (res["host_ms"]["median"] / 1e3)
    res["gpu_over_nacl_1core"] = res["gpu_ev_per_s_end_to_end"] / res["nacl_1core_ev_per_s"]
    res["gpu_over_nacl_allcores"] = res["gpu_ev_per_s_end_to_end"] / res["nacl_allcores_ev_per_s"]
    res["stats"] = e.stats()
    if a.profile:                                            # a run of its own, after the timed calls
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            call()
        dev = {}
        for ev in prof.events():
            if ev.device_type.name == "CUDA":
                dev[ev.name] = dev.get(ev.name, 0.0) + ev.time_range.elapsed_us() / 1e3
        res["profile_device_ms"] = dev
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_verify.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    if not ok:
        sys.exit("sw_verify_events disagrees with libsodium")


if __name__ == "__main__":
    main()
