"""Named traces for the fame and order kernels, each with the oracle branch counters it must reach.

A parity case only tests a branch if its trace takes it.  Every case below names the branches it is there for
(``needs``: counters of ``oracle.COVERAGE`` that must be non-zero); ``tests/test_fame_cases.py`` checks them on the
CPU, so a change of a generator cannot quietly empty a case, and ``tests/test_gpu_fame_order.py`` runs the same
cases on the engine and checks the same counters from its own oracle run.

The counters (oracle/swirld_oracle.c, OR_COV_*):
  coin_votes / coin_ones  votes cast by the coin (swirld.py:272), and how many of them were 1
  coin_super              supermajority votes in a coin round (:268-269)
  decide_after_c          decisions more than C rounds after the candidate's round
  majority_empty          majority() over an empty strongly-seen set (:260)
  median_odd/median_even  find_order medians over an odd / even number of times (:305)
  single_seer             the IndexError of :305 (one famous witness sees the event)
  tied                    adjacent events of a round's final order with equal consensus time (:306, the tie-break
                          by the whitened signature)

The member counts sit at the mask widths of the wide kernels: NJ = 32-bit words per member mask, a power of two
(M 65-128: NJ = 4, 129-256: 8, 257-512: 16, 513-1024: 32), and M = 33-64 is the two-word path of the M <= 64
kernels.  M = 97, 129, 257 and 513 leave one or a few live bits in the last word.
"""
from __future__ import annotations

from dataclasses import dataclass

# the ragged schedule of test_engine_edge_cases: calls of at most 16 events take the one-launch streaming kernel
# (swirld_stream.cuh), the others the batch kernels
RAGGED = (1, 2, 3, 5, 64, 1, 1, 700, 31, 33)


def stake_of(kind, M):
    """None (unit stake), "mixed" (1..4), "zero" (every sixth member has none, the others 1 or 2) or a list."""
    if kind is None or isinstance(kind, list):
        return kind
    if kind == "mixed":
        return [1 + (i % 5 == 0) + 2 * (i % 7 == 3) for i in range(M)]
    if kind == "zero":
        return [0 if i % 6 == 5 else 1 + (i % 5 == 0) for i in range(M)]
    raise ValueError(kind)


@dataclass(frozen=True)
class Case:
    gen: str                  # a generator of swirld_b200.traces
    kw: dict                  # its arguments
    K: object                 # chunk size of the call schedule, or a tuple of sizes used in turn
    stake: object = None      # see stake_of
    C: int = 6                # coin period
    needs: tuple = ()         # counters of oracle.COVERAGE that must be > 0
    slice_to: int = 0         # use only the first slice_to events (0: all)

    @property
    def M(self):
        return self.kw["M"]

    def trace(self):
        from swirld_b200 import traces
        tr = getattr(traces, self.gen)(**self.kw)
        return tr.slice(0, self.slice_to) if self.slice_to else tr

    def stakes(self):
        return stake_of(self.stake, self.M)

    def schedule(self, n):
        """[(first, count)] of the calls."""
        sizes = self.K if isinstance(self.K, tuple) else (self.K,)
        out, first, i = [], 0, 0
        while first < n:
            cnt = min(sizes[i % len(sizes)], n - first)
            out.append((first, cnt))
            first += cnt
            i += 1
        return out


COIN = ("coin_votes", "coin_ones", "coin_super", "decide_after_c")

CASES = {
    # ---- coin rounds above 64 members, one or more per mask width
    "coin_nj4_m96_adv_c2": Case("adversarial", dict(M=96, N=12000, seed=68), 3000, None, 2, COIN),
    "coin_nj4_m97_adv_c2_zero": Case("adversarial", dict(M=97, N=12000, seed=68), 3000, "zero", 2, COIN),
    "coin_nj4_m100_gossip_c2": Case("gossip", dict(M=100, N=16000, seed=62), 4000, None, 2,
                                    COIN + ("median_odd", "median_even", "tied")),
    "coin_nj4_m128_adv_c3": Case("adversarial", dict(M=128, N=30000, seed=5, p_cross=0.002, p_stale=0.3), 8192,
                                 None, 3, COIN + ("majority_empty", "median_odd", "median_even")),
    "coin_nj8_m129_gossip_c2": Case("gossip", dict(M=129, N=20000, seed=9), 4000, None, 2,
                                    COIN + ("median_odd", "median_even", "tied")),
    "coin_nj8_m160_adv_c2_zero": Case("adversarial", dict(M=160, N=30000, seed=5, p_cross=0.002, p_stale=0.3), 8192,
                                      "zero", 2, COIN + ("majority_empty",)),
    "coin_nj16_m257_gossip_c2": Case("gossip", dict(M=257, N=40000, seed=7), 8192, None, 2,
                                     COIN + ("median_odd", "median_even")),
    "coin_nj16_m300_adv_c2_zero": Case("adversarial", dict(M=300, N=40000, seed=5, p_cross=0.002, p_stale=0.3), 8192,
                                       "zero", 2, COIN),
    # NJ = 32: gossip at M = 513 needs about 60 000 events for enough rounds (11 at C = 2, no consensus yet); the
    # oracle takes over a minute
    "coin_nj32_m513_gossip_np_c2": Case("gossip_np", dict(M=513, N=60000, seed=3), 12000, None, 2, COIN),
    # the reference's cadence: the streaming divide_rounds kernel feeds the wide fame kernel
    "coin_nj4_m96_adv_c2_ragged": Case("adversarial", dict(M=96, N=12000, seed=68), RAGGED, None, 2, COIN),
    # ---- coin rounds on the two-word masks of the M <= 64 kernels (all four implementations)
    "coin_m40_adv_c3": Case("adversarial", dict(M=40, N=9000, seed=24, p_cross=0.02, p_stale=0.4), 2048, None, 3,
                            COIN + ("median_odd", "median_even", "tied")),
    "coin_m64_adv_c3": Case("adversarial", dict(M=64, N=12000, seed=25, p_cross=0.03, p_stale=0.3), 4096, None, 3,
                            COIN + ("median_odd", "median_even", "tied")),
    # ---- tied consensus times above 64 members: the radix-select median and the bisection for "received" of the
    # wide order kernels meet equal keys (t = index // tied)
    "tied_m96_gossip": Case("gossip", dict(M=96, N=12000, seed=3, tied=16), 3000, None, 6, ("tied", "median_odd", "median_even")),
    "tied_m96_adv": Case("adversarial", dict(M=96, N=12000, seed=4, p_cross=0.02, p_stale=0.3, tied=16), 3000, None, 6,
                         ("tied", "median_odd", "median_even")),
    "tied_m129_gossip_c3": Case("gossip", dict(M=129, N=12000, seed=9, tied=16), 2000, None, 3,
                                COIN + ("tied", "median_odd", "median_even")),
    "tied_m300_gossip": Case("gossip", dict(M=300, N=36000, seed=5, tied=32), 9000, None, 6,
                             ("tied", "median_odd", "median_even")),
}

# A single famous witness sees an event with more than half the stake: swirld.py:305 raises IndexError (zero-stake
# members make it likely).  The reference has already ordered the earlier rounds of sorted(new_c) when it raises,
# so what a view holds after the raise is undefined; the tests compare everything up to the raise and the raise.
SEER_CASES = {
    "seer_m4": Case("gossip", dict(M=4, N=1000, seed=1), 20, [1, 0, 0, 0], 6, ("single_seer",)),
    "seer_m6": Case("gossip", dict(M=6, N=2000, seed=2), 20, [2, 1, 0, 0, 0, 0], 6, ("single_seer",)),
    "seer_m80": Case("gossip", dict(M=80, N=6000, seed=2), 500, [1] + [0] * 79, 6, ("single_seer",)),
    "seer_m70_k1": Case("gossip", dict(M=70, N=6000, seed=3), 1, [3, 1] + [0] * 68, 6, ("single_seer",)),
}

ALL_CASES = {**CASES, **SEER_CASES}


def run_oracle(case, tr=None):
    """The oracle over the case's schedule: results(), new_c per call, coverage(), and the index of the call whose
    find_order raised IndexError (-1: none; the run stops there)."""
    import oracle as orc
    tr = case.trace() if tr is None else tr
    o = orc.Oracle(tr.M, case.stakes(), case.C)
    o.append(tr)
    ncs, raised = [], -1
    for i, (first, cnt) in enumerate(case.schedule(tr.N)):
        o.divide_rounds(first, cnt)
        nc = o.decide_fame()
        ncs.append(sorted(nc))
        try:
            o.find_order(nc)
        except IndexError:
            raised = i
            break
    res = o.results()
    res.update(new_c_per_call=ncs, coverage=o.coverage(), raised_at=raised, oracle=o)
    return res


def missing(case, coverage):
    """The counters the case needs that its run left at zero."""
    return [k for k in case.needs if coverage[k] == 0]
