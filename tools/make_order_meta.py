"""Generate tests/golden/meta_<spec>.npz: the consensus timestamp and round received of every event the UNMODIFIED
reference (py-swirld's swirld.py, imported in place through oracle/ref_harness.py) orders, on a subset of the traces and
call schedules of oracle/golden_specs.py.

    SWIRLD_REFERENCE=<checkout of py-swirld> python tools/make_order_meta.py [name ...]

The reference keeps neither: `ts` and `r` are locals of its find_order (swirld.py:281-306).  They are captured without
editing a line of it, through a module-level `sorted` installed in the imported module's namespace: the un-keyed call
`sorted(new_c)` (:283) gives the rounds, and the k-th keyed call `sorted(seen, key=...)` (:306) belongs to the k-th of
them, with `key(x)[0]` = ts[x].  Each fixture holds transactions[], consensus_time[] (f64) and round_received[] (int32),
parallel, in index space.
"""
from __future__ import annotations

import builtins
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

import golden_specs as gs  # noqa: E402
import ref_harness as rh   # noqa: E402

# K = 1 cadence, stakes (zero included, and the largest total), tied times, the late joiner, two-word masks, wide, other
# value columns: specs the reference runs in seconds to a minute
SPECS = ["g1_m4_n2000_s1_k1", "g2_m8_n6000_s2_k1",
         "g1_m5_n1500_s4_k11_stake", "g1_m7_n3000_s4_k11_stake", "g1_m80_n8000_s4_k999_stake",
         "g1_m16_n8000_s1_tied8_k1000", "g4_m9_n6000_join3000_s77_k2500",
         "g1_m33_n6000_s7_k640", "g1_m64_n20000_s1_k2000",
         "g1_m96_n20000_s3_k3000", "g3_m128_n12000_s1_k2048"] + \
    [n for n in gs.SPECS if n.startswith("rs_")] + ["g1_m4_n600_s31_k7_bigstake"]


def path(name):
    return os.path.join(gs.GOLDEN_DIR, "meta_%s.npz" % name)


class Capture:
    """The module-level `sorted` of the reference while a run is in progress."""

    def __init__(self):
        self.rounds, self.k, self.ts, self.rr = [], 0, {}, {}

    def __call__(self, it, key=None, reverse=False):
        if key is None:                                   # sorted(new_c), swirld.py:283
            out = builtins.sorted(it, reverse=reverse)
            self.rounds, self.k = out, 0
            return out
        items = list(it)                                  # sorted(seen, key=...), swirld.py:306
        r = self.rounds[self.k]
        self.k += 1
        for x in items:
            self.ts[x] = key(x)[0]
            self.rr[x] = r
        return builtins.sorted(items, key=key, reverse=reverse)


def main(names):
    swirld = rh.load_reference()
    for name in names:
        tr, K, stake = gs.make_trace(name)
        cap = Capture()
        swirld.sorted = cap
        t0 = time.time()
        try:
            r = rh.run_reference(tr, K, stake)
        finally:
            del swirld.sorted
        tx = r["transactions"]
        assert set(cap.ts) == set(tx.tolist()), (name, len(cap.ts), len(tx))
        ts = np.array([cap.ts[int(x)] for x in tx], np.float64)
        rr = np.array([cap.rr[int(x)] for x in tx], np.int32)
        np.savez_compressed(path(name), transactions=tx, consensus_time=ts, round_received=rr)
        print("%-32s ordered=%d rounds received %d..%d  (%.1fs)" % (
            name, len(tx), rr.min() if rr.size else -1, rr.max() if rr.size else -1, time.time() - t0), flush=True)


if __name__ == "__main__":
    if not rh.reference_available():
        sys.exit("set SWIRLD_REFERENCE to a checkout of py-swirld")
    main(sys.argv[1:] or SPECS)
