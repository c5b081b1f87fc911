"""Named traces that fill the fixed-size windows of the round kernels and run the second trips of the fame and order
kernels' loops, each with the sizes its oracle run must exceed.

A size test only tests a size if its trace reaches it.  Every case below names the sizes it is there for (``needs``:
pairs (size, threshold), the size must be > threshold); ``tests/test_shape_cases.py`` checks them on the CPU, so a
change of a generator or schedule cannot quietly shrink a case, and ``tests/test_gpu_partition.py`` runs the same cases
on the engine.  The sizes (``sizes()``), all from the oracle over the case's schedule:
  run       the longest run of one member's consecutive events with equal round
  ring_gap  at a call start, the most events of one member from its latest witness (included) to the call: more than
            RB_RING and the witness has left the member's ring of recent events
  behind    at a call start, the largest round difference between two members' latest events
  segment   the most events one consensus round orders (find_order replayed one round at a time)
  new_c     the most new consensus rounds one decide_fame call returns
  open      the most rounds one decide_fame call looks at: max_r - max_c + 1
The thresholds that depend on the device (more open rounds than k_fame_rounds' 2 * n_sm CTAs, more views than SMs) are
asserted by the GPU tests.
"""
from __future__ import annotations

import numpy as np

from fame_cases import RAGGED, Case

# the sizes the kernels are built around (DESIGN.md section 2)
RB_RING = 256     # swirld_rounds.cuh RB_RING, swirld_wide.cuh RW_RING: a member's ring of the events before the chunk
RC_WN = 128       # swirld_rcluster.cuh: rows per chain in the cluster round kernel's shared window
RB_WR = 32        # rounds of Wf mirrored in shared memory; chains further apart make the cluster kernel hand over
SPEC = 1024       # sw_decide_fame copies this many new rounds back with the scalars, the rest in a second copy
SORT_BLOCK = 1024  # k_order_sort: the one 1024-thread CTA that sorts all events of one consensus round

STALL = (("run", RB_RING), ("run", RC_WN), ("ring_gap", RB_RING), ("segment", SORT_BLOCK))
BEHIND = (("behind", RB_WR),)
# side A (members 0..3) holds 4 of the 5 units of stake: more than 2/3 on half the members.  (A round advances when
# the NUMBER of strongly seen members exceeds 2/3 of the total stake, swirld.py:216-219, so the total stays small.)
STAKE_SPLIT = [2, 1, 1, 0, 1, 0, 0, 0]
STAKE_MIXED_33 = [2, 0] * 4 + [1] * 25         # stakes 0, 1 and 2, total 33

CASES = {
    # ---- M <= 64: every case runs on all four implementations
    # an even split: both sides stall in one round for 15 000 events; calls of 4096 events end inside the stall
    "part_m8_even": Case("partition", dict(M=8, N=30000, seed=1, split=4, start=5000, end=20000), 4096,
                         needs=STALL),
    # a majority split: side A keeps advancing, side B falls more than RB_WR rounds behind
    "part_m8_major": Case("partition", dict(M=8, N=30000, seed=1, split=6, start=5000, end=20000), 4096,
                          needs=STALL + BEHIND),
    # the reference's cadence through a stall: calls of at most 16 events take the one-launch streaming kernel, the
    # others the batch kernels, which then start with the stalled chains' witnesses out of the ring
    "part_m8_even_ragged": Case("partition", dict(M=8, N=12000, seed=2, split=4, start=2000, end=10000), RAGGED,
                                needs=(("run", RB_RING), ("ring_gap", RB_RING), ("segment", SORT_BLOCK))),
    # integer stakes: four members each side, side A holds 4/5 of the stake, so only side B stalls; the kernels with
    # the exact per-column count (UNIT = false)
    "part_m8_stake": Case("partition", dict(M=8, N=30000, seed=3, split=4, start=5000, end=20000), 4096,
                          STAKE_SPLIT, needs=STALL + BEHIND),
    # two-word masks
    "part_m40_even": Case("partition", dict(M=40, N=50000, seed=1, split=20, start=10000, end=40000), 8192,
                          needs=STALL),
    "part_m64_even": Case("partition", dict(M=64, N=120000, seed=1, split=32, start=20000, end=80000), 16384,
                          needs=STALL),
    "part_m64_major": Case("partition", dict(M=64, N=120000, seed=1, split=48, start=20000, end=80000), 16384,
                           needs=STALL + BEHIND),
    # ---- above 64 members: the wide kernels (RW_RING; they mirror no rounds, so how far behind is not a size here)
    "part_m97_even": Case("partition", dict(M=97, N=60000, seed=1, split=48, start=10000, end=45000), 8192,
                          needs=STALL),
    "part_m97_major": Case("partition", dict(M=97, N=60000, seed=1, split=70, start=10000, end=45000), 8192,
                           needs=STALL),
    "part_m129_even": Case("partition", dict(M=129, N=80000, seed=1, split=64, start=10000, end=60000), 8192,
                           needs=STALL),
    "part_m129_major": Case("partition", dict(M=129, N=80000, seed=1, split=90, start=10000, end=60000), 8192,
                            needs=STALL),
    # ---- calls larger than one launch: one call over the whole trace
    "big_m4_one_call": Case("gossip", dict(M=4, N=40000, seed=3), 40000, needs=(("new_c", SPEC),)),
    "big_m33_one_call": Case("gossip", dict(M=33, N=400000, seed=3), 400000, needs=(("new_c", SPEC),)),
    "big_m33_one_call_stake": Case("gossip", dict(M=33, N=400000, seed=3), 400000, STAKE_MIXED_33,
                                   needs=(("new_c", SPEC),)),
    "big_m65_one_call": Case("gossip", dict(M=65, N=250000, seed=3), 250000),
    # the backlog arrives late: calls of 1000 events for the first half, then the other half in one call, so that
    # max_c is far from zero when the fame kernels meet more open rounds than CTAs
    "big_m4_backlog": Case("gossip", dict(M=4, N=40000, seed=3), (1000,) * 20 + (20000,), needs=(("new_c", SPEC),)),
}


def sizes(case, tr=None):
    """The oracle over the case's schedule with find_order replayed one consensus round at a time (the same order:
    find_order takes sorted(new_c) one round after the other).  Returns the oracle's results() and the sizes above,
    with per-call lists of some of them ("<size>_per_call"), max_c at every call, new_c per call and the oracle."""
    import oracle as orc
    tr = case.trace() if tr is None else tr
    o = orc.Oracle(tr.M, case.stakes(), case.C)
    o.append(tr)
    sched = case.schedule(tr.N)
    ncs, opens, maxcs, segs = [], [], [], []
    cons, max_c = set(), 0
    for first, cnt in sched:
        o.divide_rounds(first, cnt)
        nc = sorted(o.decide_fame())
        opens.append(o.max_round - max_c + 1)
        maxcs.append(max_c)
        ncs.append(nc)
        for r in nc:
            n0 = o.n_transactions
            o.find_order([r])
            segs.append(o.n_transactions - n0)
        cons.update(nc)
        while max_c in cons:
            max_c += 1
    res = o.results()
    rnd, wit = res["round"], res["witness"].astype(bool)
    starts = np.array([first for first, _ in sched], np.int64)
    run = 0
    gap = np.zeros(len(starts), np.int64)
    last_r = np.full((tr.M, len(starts)), -1, np.int64)
    for c in range(tr.M):
        chain = np.flatnonzero(tr.creator == c)
        if chain.size == 0:
            continue
        r = rnd[chain]
        edges = np.concatenate([[-1], np.flatnonzero(np.diff(r) != 0), [r.size - 1]])
        run = max(run, int(np.diff(edges).max()))
        before = np.searchsorted(chain, starts)                     # the member's events below each call start
        lastw = np.maximum.accumulate(np.where(wit[chain], np.arange(chain.size), -1))
        has = before > 0
        gap[has] = np.maximum(gap[has], before[has] - lastw[before[has] - 1])
        last_r[c, has] = r[before[has] - 1]
    live = last_r >= 0
    behind = np.where(live.any(0), np.where(live, last_r, -1).max(0) - np.where(live, last_r, 1 << 30).min(0), 0)
    out = dict(res)
    out.update(run=run, ring_gap=int(gap.max()), behind=int(behind.max()), segment=max(segs, default=0),
               new_c=max(len(x) for x in ncs), open=max(opens), ring_gap_per_call=gap.tolist(),
               behind_per_call=behind.tolist(), open_per_call=opens, max_c_per_call=maxcs, new_c_per_call=ncs, oracle=o)
    return out


def short(s):
    """The maxima only, for printing."""
    return {k: s[k] for k in ("run", "ring_gap", "behind", "segment", "new_c", "open")}


def missing(case, s):
    """The (size, threshold) pairs the case needs that its run does not exceed."""
    return [(k, t) for k, t in case.needs if not s[k] > t]
