"""ctypes binding of oracle/liboracle.so (the literal C restatement of the
reference's hot path).  TEST INFRASTRUCTURE: importable only from tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle.so")

_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
_i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(np.float64, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_i8p = np.ctypeslib.ndpointer(np.int8, flags="C_CONTIGUOUS")


def build(force: bool = False) -> str:
    src = os.path.join(HERE, "swirld_oracle.c")
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", HERE, "-s", "liboracle.so"])
    return LIB


_lib = None

# the branch counters of or_coverage, in the order of OR_COV_* in swirld_oracle.c
COVERAGE = ("coin_votes", "coin_ones", "coin_super", "decide_after_c", "decisions", "majority_empty",
            "median_odd", "median_even", "single_seer", "tied")


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            build()
        L = C.CDLL(LIB)
        L.or_create.restype = C.c_void_p
        L.or_create.argtypes = [C.c_int, _i64p, C.c_int]
        L.or_destroy.argtypes = [C.c_void_p]
        L.or_append.argtypes = [C.c_void_p, C.c_int, _i32p, _i32p, _i32p, _f64p, _u8p]
        L.or_divide_rounds.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.or_decide_fame.argtypes = [C.c_void_p, _i32p, C.c_int]
        L.or_find_order.argtypes = [C.c_void_p, _i32p, C.c_int]
        for f in ("or_n_events", "or_max_round", "or_n_transactions"):
            getattr(L, f).argtypes = [C.c_void_p]
        L.or_get_round.argtypes = [C.c_void_p, _i32p]
        L.or_get_famous.argtypes = [C.c_void_p, _i8p]
        L.or_get_idx.argtypes = [C.c_void_p, _i32p]
        L.or_get_height.argtypes = [C.c_void_p, _i32p]
        L.or_get_transactions.argtypes = [C.c_void_p, _i32p]
        L.or_get_can_see.argtypes = [C.c_void_p, C.c_int, C.c_int, _i32p]
        L.or_get_witness.argtypes = [C.c_void_p, _u8p]
        L.or_get_witness_table.argtypes = [C.c_void_p, _i32p]
        L.or_get_consensus.argtypes = [C.c_void_p, _i32p, C.c_int]
        L.or_coverage.argtypes = [C.c_void_p, _i64p]
        _lib = L
    return _lib


class Oracle:
    """One node-view of the oracle; same call surface as the engine."""

    def __init__(self, M: int, stake=None, coin_period: int = 6):
        self.M = M
        st = np.ones(M, dtype=np.int64) if stake is None else np.ascontiguousarray(stake, dtype=np.int64)
        self._h = lib().or_create(M, st, coin_period)
        if not self._h:
            raise ValueError("or_create failed")

    def close(self):
        if self._h:
            lib().or_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _chk(rc):
        if rc == -2:
            raise IndexError("list index out of range (swirld.py:305)")
        if rc == -3:
            raise KeyError("missing key (reference would raise KeyError)")
        if rc < 0:
            raise ValueError("oracle error %d" % rc)
        return rc

    def append(self, tr):
        self._chk(lib().or_append(
            self._h, tr.N, np.ascontiguousarray(tr.p0, np.int32),
            np.ascontiguousarray(tr.p1, np.int32), np.ascontiguousarray(tr.creator, np.int32),
            np.ascontiguousarray(tr.t, np.float64), np.ascontiguousarray(tr.sig, np.uint8)))

    def divide_rounds(self, first, n):
        self._chk(lib().or_divide_rounds(self._h, first, n))

    def decide_fame(self):
        buf = np.empty(max(16, self.max_round + 2), dtype=np.int32)
        n = self._chk(lib().or_decide_fame(self._h, buf, buf.size))
        return buf[:n].tolist()

    def find_order(self, new_c):
        a = np.ascontiguousarray(sorted(new_c), dtype=np.int32)
        if a.size == 0:
            a = np.zeros(1, dtype=np.int32)
            self._chk(lib().or_find_order(self._h, a, 0))
        else:
            self._chk(lib().or_find_order(self._h, a, a.size))

    @property
    def n(self):
        return lib().or_n_events(self._h)

    @property
    def max_round(self):
        return lib().or_max_round(self._h)

    @property
    def n_transactions(self):
        return lib().or_n_transactions(self._h)

    def results(self):
        n, M = self.n, self.M
        rnd = np.empty(n, np.int32); lib().or_get_round(self._h, rnd)
        fam = np.empty(n, np.int8); lib().or_get_famous(self._h, fam)
        wit = np.empty(n, np.uint8); lib().or_get_witness(self._h, wit)
        wt = np.empty((self.max_round + 1, M), np.int32); lib().or_get_witness_table(self._h, wt)
        cons = np.empty(self.max_round + 2, np.int32)
        nc = lib().or_get_consensus(self._h, cons, cons.size)
        tx = np.empty(lib().or_n_transactions(self._h), np.int32)
        if tx.size:
            lib().or_get_transactions(self._h, tx)
        return {"round": rnd, "witness": wit, "witness_table": wt, "famous": fam,
                "consensus": cons[:nc].copy(), "transactions": tx}

    def can_see(self, first=0, n=None):
        n = self.n - first if n is None else n
        out = np.empty((n, self.M), np.int32)
        lib().or_get_can_see(self._h, first, n, out)
        return out

    def coverage(self):
        """How often this view took each rarely taken branch so far: {name in COVERAGE: count}."""
        out = np.zeros(len(COVERAGE), np.int64)
        assert lib().or_coverage(self._h, out) == len(COVERAGE)
        return dict(zip(COVERAGE, out.tolist()))


def run_oracle(tr, K, stake=None, coin_period=6, timing=None):
    """Feed a trace in chunks of K (the schedule) and return results()."""
    import time
    from swirld_b200.traces import chunks
    o = Oracle(tr.M, stake, coin_period)
    o.append(tr)
    new_c_per_call = []
    t_dr = t_df = t_fo = 0.0
    for first, cnt in chunks(tr.N, K):
        a = time.perf_counter()
        o.divide_rounds(first, cnt)
        b = time.perf_counter()
        nc = o.decide_fame()
        c = time.perf_counter()
        o.find_order(nc)
        d = time.perf_counter()
        t_dr += b - a; t_df += c - b; t_fo += d - c
        new_c_per_call.append(sorted(nc))
    res = o.results()
    res["new_c_per_call"] = new_c_per_call
    res["t_divide_rounds"] = t_dr
    res["t_decide_fame"] = t_df
    res["t_find_order"] = t_fo
    res["coverage"] = o.coverage()
    res["oracle"] = o
    return res
