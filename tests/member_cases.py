"""Named cases at every member count the kernels branch on, each with what its oracle run must reach.

Nearly every kernel is shaped by the member count M:
  M <= 64     the kernels of swirld_rounds.cuh / swirld_rcluster.cuh / swirld_kernels.cuh, instantiated for NC =
              ceil(M / 32) in {1, 2} words per mask, with unit stakes (UNIT: a bit-sliced count compared with the
              threshold floor(2 M / 3) plane by plane) or integer ones (UNIT = false: exact per-column sums)
  M > 64      the wide kernels of swirld_wide.cuh, instantiated for NJ = the next power of two >= ceil(M / 32)
              (65-128: 4, 129-256: 8, 257-512: 16, 513-1024: 32); the streaming kernel and k_cs_small run
              round_up(M, 32) threads and zero the mask words between ceil(M / 32) and NJ
  can_see     the scan cuts a call into blocks of cs_block_len(M) events and tiles the members CT = 32, 16 or 8
              columns wide, CT chosen from M, the number of blocks and the device's SM count (cs_tile_width)

NARROW runs every M from 2 to 64, with unit stakes (every threshold floor(2 M / 3) from 1 to 42; M = 1, threshold 0,
is tests/test_gpu_member_counts.py's own test) and with "zero" stakes (fame_cases.stake_of), through a call schedule
that takes the streaming kernel, the grid-wide round kernel and the cluster round kernel in turn.  WIDE holds every
NJ bucket's lower and upper edge and member counts one short of a full last mask word (M = 32 k - 1) and one past it
(32 k + 1).  SCAN holds multi-block scans above 256 members with full oracle runs, and SCAN_CT candidates for the
narrow tiles, whose can_see only the GPU test checks (against traces.can_see_rows) on the cases its SM count picks.

Every oracle case names what it must reach (``needs``: (size, threshold), the size must be > threshold, or (size,
"==", value)); tests/test_member_cases.py checks them on the CPU and tests/test_gpu_member_counts.py runs the cases on
the engine.  The sizes (``sizes()``):
  consensus   rounds that reached consensus
  max_round   the largest round of any event
  blocks      the most can_see blocks one call's scan has (cs_blocks)
  stale       other-parents that are not their member's latest event when they arrive (the scan's SV = 64 layout)
"""
from __future__ import annotations

import fame_cases as fc
import view_cases as vc

# calls of at most 16 events (the one-launch streaming kernel), 17..2047 (the grid-wide round kernel) and >= 2048
# (the cluster round kernel under the default configuration), in turn
NARROW_K = (1, 7, 16, 300, 2048, 3, 1000, 2600, 12, 40)
# above 64 members: calls of at most 16 events (the streaming kernel) between calls of thousands (the wide kernels)
WIDE_K = (16, 6000, 1, 2500, 7)

MIN_CONSENSUS = 5     # what every narrow case that can reach consensus must reach


def _narrow():
    out = {}
    for M in range(2, 65):
        for stake in (None, "zero"):
            if stake is None and M <= 3 or stake == "zero" and M == 2:
                # quirk Q3: promotion compares a COUNT of strongly seen members with the STAKE threshold floor(2 tot / 3).
                # Unit stakes, M = 2 and 3: rounds advance but no round is ever decided.  Stakes [2, 1]: two members
                # never exceed floor(6 / 3) = 2, so every event stays in round 0
                needs = (("consensus", "==", 0),) + ((("max_round", 49),) if stake is None else (("max_round", "==", 0),))
            else:
                needs = (("consensus", MIN_CONSENSUS - 1),)
            name = "narrow_m%02d_%s" % (M, "unit" if stake is None else stake)
            out[name] = fc.Case("gossip", dict(M=M, N=max(3000, 200 * M), seed=1000 + M), NARROW_K, stake, needs=needs)
    return out


NARROW = _narrow()


def _wide(M, N, stake=None, needs=None, gen="gossip"):
    """Up to about 300 members: at least 2 consensus rounds.  Above, the oracle costs about N M^2, so the cases stay
    short and need rounds only: round 2 up to 512 members, round 1 up to 767.  At 1023 and 1024 members every event
    of a case this short stays in round 0 (round 1 takes about 20 000 events, 37 s of oracle): those two test the
    scan, the round-0 masks and witnesses and the empty fame at NJ = 32 with a full and a nearly full last word."""
    if needs is None:
        needs = ((("consensus", 1),) if M <= 300 else (("max_round", 1),) if M <= 512 else
                 (("max_round", 0),) if M < 1000 else (("max_round", "==", 0),))
    return fc.Case(gen, dict(M=M, N=N, seed=2000 + M), WIDE_K, stake, needs=needs)


WIDE = {
    # NJ = 4 (65-128 members)
    "wide_m65": _wide(65, 8000),
    "wide_m95": _wide(95, 10000),
    "wide_m95_zero": _wide(95, 10000, "zero"),
    "wide_m97": _wide(97, 10000),
    "wide_m127": _wide(127, 12000),
    "wide_m128": _wide(128, 12000),
    # NJ = 8 (129-256)
    "wide_m129": _wide(129, 12000),
    "wide_m159": _wide(159, 14000),
    "wide_m161": _wide(161, 14000),
    "wide_m191": _wide(191, 16000),
    "wide_m192": _wide(192, 16000),
    "wide_m193": _wide(193, 16000),
    "wide_m193_zero": _wide(193, 16000, "zero"),
    "wide_m255": _wide(255, 18000),
    "wide_m256": _wide(256, 18000),
    # NJ = 16 (257-512)
    "wide_m257": _wide(257, 18000),
    "wide_m383": _wide(383, 14000),
    "wide_m383_zero": _wide(383, 14000, "zero"),
    "wide_m384": _wide(384, 14000),
    "wide_m385": _wide(385, 14000),
    "wide_m511": _wide(511, 16000),
    "wide_m512": _wide(512, 16000),
    # NJ = 32 (513-1024)
    "wide_m513": _wide(513, 12000),
    "wide_m767": _wide(767, 12000),
    "wide_m1023": _wide(1023, 12000),
    "wide_m1024": _wide(1024, 12000),
}

# ---- the can_see scan above 256 members: calls of 3 blocks (B = cs_block_len(300) = 9600 events) that start off the
# 4-event alignment, with and without stale other-parents (SV = 0 / 64)
SCAN_K = (1003, 28000, 16, 2981)
SCAN = {
    "scan_m300_gossip": fc.Case("gossip_np", dict(M=300, N=32000, seed=31), SCAN_K,
                                needs=(("blocks", 2), ("consensus", 0))),
    "scan_m300_adv_stale": fc.Case("adversarial_np", dict(M=300, N=32000, seed=32, p_cross=0.05, p_stale=0.3), SCAN_K,
                                   needs=(("blocks", 2), ("stale", 1000), ("consensus", 0))),
}

# ---- narrow tiles: one call over the whole trace (appended at once, so sw_append scans it); which CT the host picks
# depends on the SM count, so the GPU test takes, for each width, the first candidate that picks it on its device
SCAN_CT = {
    "ct_m1000_gossip": fc.Case("gossip_np", dict(M=1000, N=200000, seed=41), 200000),
    "ct_m513_adv_stale": fc.Case("adversarial_np", dict(M=513, N=262144, seed=43), 262144),
    "ct_m1024_adv_stale": fc.Case("adversarial_np", dict(M=1024, N=200000, seed=42), 200000),
    "ct_m700_gossip": fc.Case("gossip_np", dict(M=700, N=300000, seed=44), 300000),
    "ct_m700_adv_stale": fc.Case("adversarial_np", dict(M=700, N=300000, seed=45), 300000),
}
CS_TILE = vc.CS_TILE
CS_SV = vc.CS_SV
CS_SMEM = 220 << 10        # the shared memory one SM gives the scan's CTAs, as cansee_scan counts it


def cs_blocks(M, first, n):
    """swirld_b200.cu cs_blocks: the number of blocks of the scan of [first, first+n) (n > 24)."""
    return len(vc.cs_block_starts(M, first, n))


def cs_tile_width(M, nb, stale, n_sm):
    """swirld_b200.cu cansee_scan, the loop that picks CT: the width in 32, 16, 8 whose grid of nb x ceil(M / CT)
    CTAs finishes in the fewest waves, at as many CTAs per SM as the per-member cache val[M + SV][CT] lets fit (at most
    32); a tie keeps the wider tile."""
    sv = CS_SV if stale else 0
    best, CT = -1, 32
    for ct in (32, 16, 8):
        smem = (M + sv) * ct * 4 + CS_TILE * 16 + 3 * CS_TILE
        conc = max(1, min(32, CS_SMEM // smem))
        ctas = nb * ((M + ct - 1) // ct)
        waves = (ctas + n_sm * conc - 1) // (n_sm * conc)
        if best < 0 or waves < best:
            best, CT = waves, ct
    return CT


def scan_shape(case, tr, n_sm):
    """(CT, blocks) of the scan of a SCAN_CT case's one call."""
    nb = cs_blocks(case.M, 0, tr.N)
    return cs_tile_width(case.M, nb, bool(vc.stale_info(tr)[0].any()), n_sm), nb


def pick_ct(n_sm, ct, stale):
    """The first SCAN_CT case whose scan picks tiles ct wide on n_sm SMs, with or without stale parents; None if none.
    (The graph is not needed: a case has stale parents iff its generator draws them.)"""
    for name, case in SCAN_CT.items():
        if (case.gen == "adversarial_np") != stale:
            continue
        if cs_tile_width(case.M, cs_blocks(case.M, 0, case.kw["N"]), stale, n_sm) == ct:
            return name
    return None


ORACLE_CASES = {**NARROW, **WIDE, **SCAN}


def sizes(case, tr=None):
    """fame_cases.run_oracle over the case's schedule, with the sizes above."""
    tr = case.trace() if tr is None else tr
    res = fc.run_oracle(case, tr)
    blocks = max((cs_blocks(tr.M, f, n) for f, n in case.schedule(tr.N) if n > 24), default=0)
    res.update(consensus_rounds=len(res["consensus"]), max_round=int(res["round"].max()), blocks=blocks,
               stale=int(vc.stale_info(tr)[0].sum()))
    return res


def short(s):
    return {"consensus": s["consensus_rounds"], "max_round": s["max_round"], "blocks": s["blocks"], "stale": s["stale"]}


def missing(case, s):
    """The needs the case's sizes do not meet."""
    s = short(s)
    return [n for n in case.needs if not (s[n[0]] == n[2] if len(n) == 3 else s[n[0]] > n[1])]
