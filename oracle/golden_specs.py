"""Trace + call-schedule specs of the committed golden fixtures (tests/golden).
Shared by oracle/make_golden.py (which runs the unmodified reference on them)
and by the tests (which rebuild the same trace and compare)."""
from __future__ import annotations

import os

SPECS = {
    # name: (generator, kwargs, K, stake or None)
    # config 1 of BASELINE.json: 4-member 2000-event gossip, the sim's cadence K=1
    "g1_m4_n2000_s1_k1":    ("gossip", dict(M=4, N=2000, seed=1), 1, None),
    "g1_m4_n2000_s1_k50":   ("gossip", dict(M=4, N=2000, seed=1), 50, None),
    "g1_m4_n2000_s1_k2000": ("gossip", dict(M=4, N=2000, seed=1), 2000, None),
    "g1_m4_n2000_s2_k1":    ("gossip", dict(M=4, N=2000, seed=2), 1, None),
    "g1_m4_n2000_s2_k50":   ("gossip", dict(M=4, N=2000, seed=2), 50, None),
    "g1_m4_n2000_s3_k7":    ("gossip", dict(M=4, N=2000, seed=3), 7, None),
    "g1_m4_n2000_s3_k2000": ("gossip", dict(M=4, N=2000, seed=3), 2000, None),
    "g1_m7_n3000_s5_k37":   ("gossip", dict(M=7, N=3000, seed=5), 37, None),
    # integer stakes (stake dict of swirld.py:42); the first never leaves round 0
    # because promotion compares a member COUNT with the STAKE threshold (quirk Q3)
    "g1_m5_n1500_s4_k11_stake": ("gossip", dict(M=5, N=1500, seed=4), 11, [1, 2, 3, 1, 2]),
    "g1_m7_n3000_s4_k11_stake": ("gossip", dict(M=7, N=3000, seed=4), 11, [1, 1, 2, 1, 1, 1, 0]),
    "g1_m10_n3000_s4_k64_stake": ("gossip", dict(M=10, N=3000, seed=4), 64, [1, 1, 1, 1, 1, 1, 1, 1, 2, 0]),
    "g2_m8_n6000_s2_k1":    ("adversarial", dict(M=8, N=6000, seed=2, p_cross=0.05, p_stale=0.3), 1, None),
    "g1_m16_n20000_s1_k1000": ("gossip", dict(M=16, N=20000, seed=1), 1000, None),
    "g2_m16_n12000_s1_k500":  ("adversarial", dict(M=16, N=12000, seed=1, p_cross=0.02, p_stale=0.3), 500, None),
    "g1_m16_n8000_s1_tied8_k1000": ("gossip", dict(M=16, N=8000, seed=1, tied=8), 1000, None),
    "g3_m16_n6000_s1_k700": ("tick", dict(M=16, N=6000, seed=1), 700, None),
    "g3_m32_n8000_s2_k512": ("tick", dict(M=32, N=8000, seed=2), 512, None),
    "g1_m33_n6000_s7_k640": ("gossip", dict(M=33, N=6000, seed=7), 640, None),
    "g2_m64_n16000_s3_k4096": ("adversarial", dict(M=64, N=16000, seed=3, p_cross=0.03, p_stale=0.3), 4096, None),
    "g1_m64_n20000_s1_k2000": ("gossip", dict(M=64, N=20000, seed=1), 2000, None),
    # config 2 of BASELINE.json in full, config 3 as a prefix (same K as the bench)
    "g1_m16_n100000_s1_k4096": ("gossip", dict(M=16, N=100000, seed=1), 4096, None),
    "g1_m64_n131072_s1_k65536": ("gossip", dict(M=64, N=131072, seed=1), 65536, None),
    # beyond 64 members (multi-word member masks): prefixes of BASELINE.json's configs 4 and 5 and mid sizes
    "g1_m96_n20000_s3_k3000": ("gossip", dict(M=96, N=20000, seed=3), 3000, None),
    "g1_m80_n8000_s4_k999_stake": ("gossip", dict(M=80, N=8000, seed=4), 999, [1 + (i % 3 == 0) for i in range(80)]),
    "g2_m128_n40000_s2_k8192": ("adversarial", dict(M=128, N=40000, seed=2, p_cross=0.02, p_stale=0.3), 8192, None),
    "g3_m128_n12000_s1_k2048": ("tick", dict(M=128, N=12000, seed=1), 2048, None),
    "g1_m256_n60000_s1_k16384": ("gossip", dict(M=256, N=60000, seed=1), 16384, None),
    "g1_m1024_n20000_s1_k8192": ("gossip", dict(M=1024, N=20000, seed=1), 8192, None),
    # a member whose root arrives ~48 rounds late (its chain starts further behind than the round kernels' mirror)
    "g4_m9_n6000_join3000_s77_k2500": ("late_joiner", dict(M=9, N=6000, join_at=3000, seed=77), 2500, None),
    # short gossip and adversarial traces at the reference's own cadences (tests/test_oracle_golden.py, LIVE)
    "g1_m4_n600_s11_k1": ("gossip", dict(M=4, N=600, seed=11), 1, None),
    "g2_m4_n600_s11_k1": ("adversarial", dict(M=4, N=600, seed=11, p_cross=0.05, p_stale=0.3), 1, None),
    "g1_m5_n900_s12_k13": ("gossip", dict(M=5, N=900, seed=12), 13, None),
    "g2_m5_n900_s12_k13": ("adversarial", dict(M=5, N=900, seed=12, p_cross=0.05, p_stale=0.3), 13, None),
    "g1_m16_n3000_s13_k250": ("gossip", dict(M=16, N=3000, seed=13), 250, None),
    "g2_m16_n3000_s13_k250": ("adversarial", dict(M=16, N=3000, seed=13, p_cross=0.05, p_stale=0.3), 250, None),
    # other value columns (traces.restamped): fractional, negative, constant, overflowing and subnormal times, and
    # signatures that share their first P bytes, so ties of the order are decided at byte P or later
    "rs_g1_m4_n1500_s21_k1_wall_p56": ("restamped", dict(base="gossip", times="wall", sigs="prefix56", seed=21, M=4, N=1500), 1, None),
    "rs_g1_m5_n1500_s22_k13_const_p32": ("restamped", dict(base="gossip", times="const", sigs="prefix32", seed=22, M=5, N=1500), 13, None),
    "rs_g2_m16_n4000_s23_k250_neg_p16": ("restamped", dict(base="adversarial", times="neg", sigs="prefix16", seed=23, M=16, N=4000,
                                                           p_cross=0.05, p_stale=0.3), 250, None),
    "rs_g1_m33_n6000_s25_k640_huge_p8": ("restamped", dict(base="gossip", times="huge", sigs="prefix8", seed=25, M=33, N=6000), 640, None),
    "rs_g1_m64_n12000_s24_k2048_tiny_p60c": ("restamped", dict(base="gossip", times="tiny", sigs="prefix60_coin", seed=24, M=64,
                                                               N=12000), 2048, None),
    "rs_g1_m96_n12000_s28_k3000_wall_p60": ("restamped", dict(base="gossip", times="wall", sigs="prefix60", seed=28, M=96, N=12000), 3000, None),
    "rs_g1_m80_n8000_s27_k999_shuffle_p16": ("restamped", dict(base="gossip", times="shuffle", sigs="prefix16", seed=27, M=80, N=8000), 999,
                                             [1 + (i % 3 == 0) for i in range(80)]),
    # the largest stake total B = (2**63 - 1) // 3 whose triple fits in int64: a member count never exceeds 2/3 of it
    # (quirk Q3), so every event stays in round 0 and nothing is ordered
    "g1_m4_n600_s31_k7_bigstake": ("gossip", dict(M=4, N=600, seed=31), 7, [2 ** 61, (2 ** 63 - 1) // 3 - 2 ** 61 - 1, 1, 0]),
}

# the arrival traces and call schedules of two nodes of one gossip simulation over tests/host_sim.py (4 nodes,
# 400 turns, real signatures, so not reproducible from a seed: the fixture stores the trace itself)
NODE_FIXTURES = ["node_m4_t400_s5_n0", "node_m4_t400_s5_n1"]

# node views of generator traces (traces.node_view: one member's arrival order, one call per sync), stored like
# NODE_FIXTURES with the reference's replay: name -> (generator, kwargs, node)
VIEW_FIXTURES = {
    # a partition that heals: the node's syncs after the heal bring thousands of events, stale parents far behind
    "view_g5_m8_n12000_s3_x0": ("partition", dict(M=8, N=12000, seed=3, split=4, start=2000, end=9000), 0),
    # the two-word masks, roots out of member order
    "view_g1_m33_n6000_s7_x5": ("gossip", dict(M=33, N=6000, seed=7), 5),
    # two cliques with rare cross links: long bursts from the other clique (at p_cross = 0.002 no round of an 8000-event
    # view reaches consensus)
    "view_g2_m16_n8000_s1_x0": ("adversarial", dict(M=16, N=8000, seed=1, p_cross=0.004, p_stale=0.3), 0),
}

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                          "tests", "golden")


def make_trace(name):
    from swirld_b200 import traces
    gen, kw, K, stake = SPECS[name]
    return getattr(traces, gen)(**kw), K, stake


def path(name):
    return os.path.join(GOLDEN_DIR, name + ".npz")


def make_view(name):
    """(view trace, call sizes) of VIEW_FIXTURES[name]."""
    from swirld_b200 import traces
    gen, kw, node = VIEW_FIXTURES[name]
    return traces.node_view(getattr(traces, gen)(**kw), node)
