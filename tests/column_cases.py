"""Named traces for find_order and the coin on other value columns (swirld_b200.traces.restamped), each with what its
oracle run must reach.

Every other trace of the suite has t[i] = i (or i // tied) and BLAKE2b signatures, so integer times that float32 holds
exactly decide every order, and whitened signatures differ in byte 0 for 255 of every 256 ties.  The cases here give
the order kernels fractional, negative, permuted, constant, overflowing and subnormal times, signatures that share
their first P bytes (so a tie is decided by key word P // 8 of (ts, white ^ sig), swirld.py:306), and coins that all
agree.  ``tests/test_column_cases.py`` checks on the CPU that each case reaches what it needs; ``tests/test_gpu_columns.py``
runs them on the engine.

The counters (``analyse``):
  word0 .. word7  adjacent pairs of one round received with equal consensus time whose sort key first differs in key word
                  k (the 64-bit big-endian words of white ^ sig; swirld_kernels.cuh order_less)
  neg / inf       ordered events with a negative / +inf consensus time
  inexact         consensus times .5 * (a + b) that are not the exact mean of the two median times (rounded sum or half)
  coin_votes / coin_ones   the oracle's coin counters (fame_cases.py)
  coin_same       1 when the coin voted and every vote came up the same (coin0 / coin1)
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

import fame_cases as fc
from fame_cases import RAGGED, Case


def rs(base, times, sigs, seed, **kw):
    return dict(base=base, times=times, sigs=sigs, seed=seed, **kw)


def _w(P):
    return "word%d" % (P // 8)


CASES = {
    # ---- one-word masks of the M <= 64 kernels
    "wall_m4_p56_k1": Case("restamped", rs("gossip", "wall", "prefix56", 21, M=4, N=1500), 1, None, 6,
                           (_w(56), "inexact")),
    "const_m5_p32_ragged": Case("restamped", rs("gossip", "const", "prefix32", 22, M=5, N=1500), RAGGED, None, 6,
                                (_w(32),)),
    "neg_m16_p16_k250": Case("restamped", rs("gossip", "neg", "prefix16", 23, M=16, N=4000), 250, None, 6,
                             (_w(16), "neg", "inexact")),
    "tiny_m16_p60c_batch": Case("restamped", rs("gossip", "tiny", "prefix60_coin", 24, M=16, N=6000), 3000, None, 6,
                                ("word0", _w(60), "inexact")),
    # ---- two-word masks
    "huge_m33_p8_k640": Case("restamped", rs("gossip", "huge", "prefix8", 25, M=33, N=6000), 640, None, 6,
                             (_w(8), "inf", "inexact")),
    "shuffle_m64_p56_batch": Case("restamped", rs("gossip", "shuffle", "prefix56", 26, M=64, N=12000), 4096, None, 6,
                                  (_w(56),)),
    "coin1_m40_adv_c2": Case("restamped", rs("adversarial", "wall", "coin1", 24, M=40, N=9000, p_cross=0.02,
                                             p_stale=0.4), 2048, None, 2, ("coin_votes", "coin_same", "inexact")),
    "coin0_m64_adv_c2": Case("restamped", rs("adversarial", "neg", "coin0", 26, M=64, N=12000, p_cross=0.1,
                                             p_stale=0.3), 4096, None, 2, ("coin_votes", "coin_same", "neg")),
    # ---- any-M kernels: the radix-select median of swirld_wide.cuh
    "neg_m80_p16_k999": Case("restamped", rs("gossip", "neg", "prefix16", 27, M=80, N=8000), 999, None, 6,
                             (_w(16), "neg")),
    "wall_m96_p60_k3000": Case("restamped", rs("gossip", "wall", "prefix60", 28, M=96, N=12000), 3000, None, 6,
                               (_w(60), "inexact")),
    "huge_m96_p32c_ragged": Case("restamped", rs("gossip", "huge", "prefix32_coin", 29, M=96, N=10000), RAGGED, None, 6,
                                 ("word0", _w(32), "inf")),
    "coin1_m96_adv_c2": Case("restamped", rs("adversarial", "shuffle", "coin1", 68, M=96, N=12000), 3000, None, 2,
                             ("coin_votes", "coin_same")),
    "tiny_m129_p16_k2000": Case("restamped", rs("gossip", "tiny", "prefix16", 30, M=129, N=12000), 2000, None, 6,
                                (_w(16), "inexact")),
}

COUNTERS = tuple("word%d" % k for k in range(8)) + ("tied", "neg", "inf", "inexact", "coin_votes", "coin_ones",
                                                    "coin_same", "ordered")


def run_oracle(case, tr=None):
    """The oracle's order, consensus times, rounds received, median times, results() and coverage() over the case's
    schedule."""
    import order_meta
    tr = case.trace() if tr is None else tr
    return order_meta.run_oracle_meta(tr, [c for _, c in case.schedule(tr.N)], case.stakes(), case.C, extra=True)


def _key(white, sig):
    return int.from_bytes(bytes(white ^ sig), "big")


def analyse(tr, r):
    """The counters of the module docstring, from an oracle run (run_oracle) on trace tr."""
    tx, ts, rr, med = r["transactions"], r["consensus_time"], r["round_received"], r["median"]
    wt, fam = r["results"]["witness_table"], r["results"]["famous"]
    out = dict.fromkeys(COUNTERS, 0)
    white = {}
    for rnd in np.unique(rr).tolist():
        w = np.zeros(64, np.uint8)
        for x in wt[rnd][wt[rnd] >= 0]:
            if fam[x] == 1:
                w ^= tr.sig[x]
        white[rnd] = w
    for i in range(1, len(tx)):
        if rr[i] != rr[i - 1] or ts[i] != ts[i - 1]:
            continue
        w = white[int(rr[i])]
        a, b = w ^ tr.sig[tx[i - 1]], w ^ tr.sig[tx[i]]
        assert _key(w, tr.sig[tx[i - 1]]) < _key(w, tr.sig[tx[i]]), "the oracle's order is not by (ts, white ^ sig)"
        first = int(np.nonzero(a != b)[0][0])
        out["word%d" % (first // 8)] += 1
        out["tied"] += 1
    out["neg"] = int((ts < 0).sum())
    out["inf"] = int(np.isinf(ts).sum())
    for (a, b), t in zip(med.tolist(), ts.tolist()):
        if np.isfinite(t) and (Fraction(a) + Fraction(b)) / 2 != Fraction(t):
            out["inexact"] += 1
    cov = r["coverage"]
    out["coin_votes"], out["coin_ones"] = cov["coin_votes"], cov["coin_ones"]
    out["coin_same"] = int(cov["coin_votes"] > 0 and cov["coin_ones"] in (0, cov["coin_votes"]))
    out["ordered"] = len(tx)
    return out


def missing(case, counters):
    return [k for k in case.needs if counters[k] == 0]


__all__ = ["CASES", "COUNTERS", "RAGGED", "analyse", "fc", "missing", "run_oracle"]
