"""Named node views: one member's own view of a generator trace (traces.node_view), each with the sizes it must exceed.

A node's view is the input the engine is built for (the reference's Node.main, swirld.py:315-328): what every sync
brought, parents first, then the node's own new event, and one divide_rounds call per sync.  It differs from the
generator traces in index order: roots arrive out of member order and late, other-parents are often stale (not their
member's latest event when they arrive) and sit many chain steps, can_see blocks and calls below the event that reads
them, and calls of a few events alternate with bursts of thousands.  Every case names the sizes it is there for
(``needs``: pairs (size, threshold), the size must be > threshold); ``tests/test_view_cases.py`` checks them on the CPU
and ``tests/test_gpu_node_views.py`` runs the cases on the engine.

The schedule is "sync" (the view's own call sizes; ``merge`` joins runs of them into one call: a node that divides
several syncs at once, e.g. after it was busy) or ("resident", K): the whole view appended first, then calls of K.
The sizes, from the view and its schedule alone (``view_sizes``):
  stale             stale other-parents
  stale_depth       the deepest one, in chain steps behind its member's latest event when it arrives
  stale_prev_call   stale other-parents that lie below the can_see scan that reads them
  stale_prev_block  stale other-parents in an earlier block of the same scan (blocks as cs_blocks cuts them)
  tile_stale        the most stale other-parents in one 128-event tile of a scan (> CS_SV: the tile's prefetch slots
                    are full and the rest are read in the walk)
  root_last         the largest index of a root; roots_permuted: 1 if the roots are not in member order
  small_calls       calls of at most 16 events (the one-launch streaming kernel)
  large_calls       calls of at least 2048 events (the cluster round kernel and the round stream at M <= 64)
  eager             appends of at least 4096 events (sw_append scans them at once)
  slow_rows         resident cases: rows of the one scan of the whole view that fail the finality check
  slow_waves        ... and the waves that finish them (more than 2: k_cs_slow_rest finishes the rest)
The scans: one per call of a "sync" schedule (each call appends its own events), one over the whole view for a
resident one.  run, ring_gap, behind and segment are shape_cases.sizes over the case's calls.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

import fame_cases as fc
import shape_cases as sc

CS_TILE = 128     # swirld_cansee.cuh: events per tile of a can_see block
CS_SV = 64        # ... and the prefetch slots for a tile's stale other-parents
SMALL = 16        # calls up to this size take the one-launch streaming kernel
LARGE = 2048      # calls from this size take the cluster round kernel (SW_RC_MIN_N) at M <= 64
EAGER = 4096      # appends from this size are scanned by sw_append


@functools.lru_cache(maxsize=None)
def _view(gen, kw_items, node):
    from swirld_b200 import traces
    return traces.node_view(getattr(traces, gen)(**dict(kw_items)), node)


@dataclass(frozen=True)
class ViewCase:
    gen: str                  # a generator of swirld_b200.traces: the base trace
    kw: dict                  # its arguments
    node: int                 # the member whose view this is
    sched: object = "sync"    # "sync", or ("resident", K)
    stake: object = None      # see fame_cases.stake_of
    C: int = 6                # coin period
    needs: tuple = ()         # (size, threshold): the size must be > threshold
    merge: tuple = ()         # "sync": (a, b) pairs, calls a..b-1 of the view become one call

    @property
    def M(self):
        return self.kw["M"]

    @property
    def resident(self):
        return self.sched != "sync"

    def view(self):
        """(view trace, the sizes of its syncs)."""
        return _view(self.gen, tuple(sorted(self.kw.items())), self.node)

    def trace(self):
        return self.view()[0]

    def stakes(self):
        return fc.stake_of(self.stake, self.M)

    def calls(self):
        """The divide_rounds call sizes."""
        tr, sizes = self.view()
        if self.resident:
            return [c for _, c in fc.Case(self.gen, self.kw, self.sched[1]).schedule(tr.N)]
        out, i = [], 0
        for a, b in sorted(self.merge):
            out += sizes[i:a] + [sum(sizes[a:b])]
            i = b
        return out + sizes[i:]

    def schedule(self, n=None):
        """[(first, count)] of the calls."""
        out, first = [], 0
        for c in self.calls():
            out.append((first, c))
            first += c
        assert n is None or first == n
        return out

    def as_case(self):
        """The same trace and calls as a fame_cases.Case (a tuple K of the call sizes replays them once)."""
        return fc.Case(self.gen, self.kw, tuple(self.calls()), self.stake, self.C)


G = "gossip"
P = "partition"
CASES = {
    # ---- views of gossip: out-of-order roots, stale other-parents from earlier calls.  A gossip node's syncs are
    # small (a few dozen events), so above 32 members a run of them is divided at once: calls of >= 2048 events
    # among calls of <= 16
    "view_g_m4_n2": ViewCase(G, dict(M=4, N=3000, seed=51), 2,
                             needs=(("stale", 100), ("small_calls", 100), ("stale_prev_call", 50), ("roots_permuted", 0))),
    "view_g_m8_n5": ViewCase(G, dict(M=8, N=6000, seed=52), 5,
                             needs=(("stale", 300), ("small_calls", 100), ("stale_prev_call", 100), ("root_last", 7))),
    "view_g_m31_n30": ViewCase(G, dict(M=31, N=8000, seed=53), 30,
                               needs=(("stale", 500), ("small_calls", 10), ("stale_depth", 4), ("root_last", 30))),
    "view_g_m33_n11": ViewCase(G, dict(M=33, N=12000, seed=54), 11, merge=((60, 140), (150, 229)),
                               needs=(("small_calls", 10), ("large_calls", 1), ("stale_prev_block", 10),
                                      ("root_last", 32))),
    "view_g_m64_n3": ViewCase(G, dict(M=64, N=20000, seed=55), 3, merge=((40, 90), (150, 200)),
                              needs=(("small_calls", 10), ("large_calls", 1), ("stale_prev_block", 10),
                                     ("stale_depth", 8), ("root_last", 63))),
    # ---- views of partitions: a heal burst of thousands of events, stale parents thousands of events behind
    "view_p_m8_even_n0": ViewCase(P, dict(M=8, N=30000, seed=1, split=4, start=5000, end=20000), 0,
                                  needs=(("stale_depth", 1000), ("large_calls", 0), ("eager", 0), ("small_calls", 100),
                                         ("behind", 0))),
    "view_p_m8_even_n5": ViewCase(P, dict(M=8, N=30000, seed=1, split=4, start=5000, end=20000), 5,
                                  needs=(("stale_depth", 1000), ("large_calls", 0), ("eager", 0), ("small_calls", 100),
                                         ("behind", 0))),
    "view_p_m8_major_n7": ViewCase(P, dict(M=8, N=30000, seed=1, split=6, start=5000, end=20000), 7,
                                   needs=(("stale_depth", 1000), ("large_calls", 0), ("eager", 0),
                                          ("behind", sc.RB_WR))),
    "view_p_m64_n40": ViewCase(P, dict(M=64, N=60000, seed=2, split=32, start=10000, end=40000), 40,
                               needs=(("stale_depth", 100), ("large_calls", 0), ("eager", 0), ("small_calls", 100),
                                      ("behind", 0))),
    # ---- two cliques with rare cross links: long bursts, slow rows of the scan over the whole view
    "view_a_m16_n0": ViewCase("adversarial", dict(M=16, N=12000, seed=3, p_cross=0.002, p_stale=0.0), 0,
                              needs=(("stale_depth", 64), ("small_calls", 100), ("segment", 1000))),
    "view_a_m16_n0_resident": ViewCase("adversarial", dict(M=16, N=12000, seed=3, p_cross=0.002, p_stale=0.0), 0,
                                       ("resident", 2048),
                                       needs=(("slow_rows", 100), ("slow_waves", 2), ("stale_prev_block", 100))),
    # ---- a member whose root arrives thousands of events late
    "view_late_m9_n0": ViewCase("late_joiner", dict(M=9, N=6000, join_at=3000, seed=77), 0,
                                needs=(("root_last", 2000), ("small_calls", 100))),
    # ---- integer stakes with zero-stake members, and coin rounds
    "view_g_m10_n4_zero": ViewCase(G, dict(M=10, N=6000, seed=56), 4, "sync", "zero",
                                   needs=(("stale", 300), ("small_calls", 100))),
    "view_a_m8_n1_c2": ViewCase("adversarial", dict(M=8, N=6000, seed=57, p_cross=0.05, p_stale=0.3), 1, C=2,
                                needs=(("stale_depth", 8), ("small_calls", 100), ("coin_votes", 0))),
    # ---- full tiles of deep stale parents, in one scan over the whole view
    "view_a_m16_stale_resident": ViewCase("adversarial", dict(M=16, N=12000, seed=58, p_cross=0.002, p_stale=0.95), 2,
                                          ("resident", 4096),
                                          needs=(("tile_stale", CS_SV), ("stale_depth", 64), ("stale_prev_block", 100))),
    # ---- above 64 members: the wide kernels
    "view_g_m65_n64": ViewCase(G, dict(M=65, N=12000, seed=59), 64, needs=(("stale", 1000), ("small_calls", 10))),
    "view_g_m97_n1": ViewCase(G, dict(M=97, N=12000, seed=60), 1, needs=(("stale", 1000), ("small_calls", 10))),
    "view_g_m129_n100": ViewCase(G, dict(M=129, N=16000, seed=61), 100, needs=(("stale", 1000), ("small_calls", 5))),
    "view_g_m100_n3_c2": ViewCase(G, dict(M=100, N=16000, seed=62), 3, C=2,
                                  needs=(("stale", 1000), ("small_calls", 10), ("coin_votes", 0), ("segment", 1000))),
}


def cs_block_len(M):
    """cs_blocks: the block length of the can_see scan."""
    return (max(256, min((16 if M <= 64 else 32) * M, 1 << 15)) + 3) & ~3


def cs_block_starts(M, first, n):
    """The starts of the blocks of the scan of [first, first+n) (n > 24), as cs_blocks cuts them."""
    B = cs_block_len(M)
    fa = first & ~3
    nb = 1 if first + n <= fa + B else 1 + (first + n - (fa + B) + B - 1) // B
    if nb > 1 and first + n - (fa + (nb - 1) * B) < 3 * B // 4:
        nb -= 1
    return [first] + [fa + j * B for j in range(1, nb)]


def stale_info(tr):
    """(stale[N] bool, depth[N]): the other-parent is not its member's latest event when the event arrives (sw_append's
    h_stale), and how many of that member's events arrived after it."""
    N = tr.N
    p1 = tr.p1.astype(np.int64)
    seq = np.zeros(N, np.int64)
    depth = np.zeros(N, np.int64)
    has = p1 >= 0
    cb = np.where(has, tr.creator[np.maximum(p1, 0)], -1)
    for c in range(tr.M):
        ev = np.flatnonzero(tr.creator == c)
        seq[ev] = np.arange(ev.size)
        mine = np.flatnonzero(cb == c)
        head = np.searchsorted(ev, mine) - 1             # c's latest event below each event that names one of c's
        depth[mine] = head - seq[p1[mine]]
    return depth > 0, depth


def scan_ranges(case, tr):
    """The ranges the can_see scans cover: one per call of a "sync" schedule, the whole view for a resident one."""
    return [(0, tr.N)] if case.resident else case.schedule(tr.N)


def view_sizes(case, tr=None):
    """The sizes above, from the view and its schedule."""
    tr = case.trace() if tr is None else tr
    st, depth = stale_info(tr)
    calls = np.array(case.calls(), np.int64)
    sidx = np.flatnonzero(st)
    p1 = tr.p1.astype(np.int64)
    prev_call = prev_block = tile = 0
    for first, n in scan_ranges(case, tr):
        inr = sidx[(sidx >= first) & (sidx < first + n)]
        prev_call += int((p1[inr] < first).sum())
        if n <= 24:
            continue
        starts = np.array(cs_block_starts(tr.M, first, n), np.int64)
        blk = np.searchsorted(starts, inr, side="right") - 1
        bb = p1[inr]
        prev_block += int(((bb >= first) & (np.searchsorted(starts, bb, side="right") - 1 < blk)).sum())
        tstart = starts[blk] + (inr - starts[blk]) // CS_TILE * CS_TILE
        if inr.size:
            tile = max(tile, int(np.unique(tstart, return_counts=True)[1].max()))
    roots = np.flatnonzero(tr.p0 < 0)
    return dict(stale=int(st.sum()), stale_depth=int(depth.max(initial=0)), stale_prev_call=prev_call,
                stale_prev_block=prev_block, tile_stale=tile, root_last=int(roots.max()),
                roots_permuted=int(not np.all(np.diff(tr.creator[roots]) > 0)),
                small_calls=int((calls <= SMALL).sum()), large_calls=int((calls >= LARGE).sum()),
                eager=(int(tr.N >= EAGER) if case.resident else int((calls >= EAGER).sum())))


def slow_sizes(case, tr=None):
    """slow_rows and slow_waves of the scan over the whole view (the model of test_cansee2_model)."""
    from test_cansee2_model import scan_launch
    tr = case.trace() if tr is None else tr
    st, _ = stale_info(tr)
    row = np.full((tr.N, tr.M), -1, np.int64)
    stats = {"fast": 0, "slow": 0, "table": 0, "p1_rows": 0, "waves": 0}
    scan_launch(tr, st, 0, tr.N, cs_block_len(tr.M), row, np.full(tr.M, -1, np.int64), stats)
    return dict(slow_rows=stats["slow"], slow_waves=stats["waves"]), row


def missing(case, s):
    """The (size, threshold) pairs the case needs that it does not exceed."""
    return [(k, t) for k, t in case.needs if not s[k] > t]
