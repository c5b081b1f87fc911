"""The member-count cases of tests/member_cases.py reach what they are there for.  Oracle and model only (no GPU): a
change of a generator, a schedule or the cases that shrinks one, or drops a member count, a threshold or a scan shape
from the sweep, fails here.  Run with -rA or -s to see each case's sizes."""
import pytest

import member_cases as mc

H100_SXM_SMS = 132


@pytest.mark.parametrize("name", list(mc.ORACLE_CASES))
def test_case_reaches_its_needs(name):
    case = mc.ORACLE_CASES[name]
    s = mc.sizes(case)
    print("%s: N=%d %s" % (name, case.kw["N"], mc.short(s)))
    assert not mc.missing(case, s), "%s no longer reaches %s (has %s)" % (name, mc.missing(case, s), mc.short(s))


def test_narrow_sweep_covers_every_member_count_and_threshold():
    """Every M from 2 to 64 with unit and with "zero" stakes, and, with M = 1, every unit-stake threshold
    floor(2 M / 3) from 0 to 42; every schedule takes the streaming, grid-wide and cluster round kernels."""
    unit = sorted(c.M for c in mc.NARROW.values() if c.stake is None)
    zero = sorted(c.M for c in mc.NARROW.values() if c.stake == "zero")
    assert unit == zero == list(range(2, 65))
    assert {2 * M // 3 for M in [1] + unit} == set(range(43))
    for case in mc.NARROW.values():
        calls = [n for _, n in case.schedule(case.kw["N"])]
        assert min(calls) <= 16 and any(16 < n < 2048 for n in calls) and max(calls) >= 2048, case


def test_wide_cases_hold_every_mask_edge():
    """Each NJ bucket has a case at its lower and upper edge, one with M = 32 k - 1 (one member short of a full last
    word) and one with M = 32 k + 1 (one live bit in it), and a case with "zero" stakes below 513 members."""
    Ms = {c.M for c in mc.WIDE.values()}
    for lo, hi in ((65, 128), (129, 256), (257, 512), (513, 1024)):
        have = sorted(M for M in Ms if lo <= M <= hi)
        assert lo in have and hi in have, (lo, hi, have)
        assert any(M % 32 == 31 for M in have) and any(M % 32 == 1 for M in have), (lo, hi, have)
        if hi <= 512:
            assert any(c.stake == "zero" and lo <= c.M <= hi for c in mc.WIDE.values()), (lo, hi)
    assert {95, 127, 159, 161, 191, 192, 193, 255, 383, 384, 385, 511, 512, 767, 1023} <= Ms


def test_scan_shape_model():
    """The restatement of cs_blocks and of the CT loop: block counts at the edges of the short-tail rule, the tile
    widths the wide members and stale parents push it to, and at H100 SXM's 132 SMs a candidate for CT = 16 with and
    without stale parents and one for CT = 8, each a scan of several blocks."""
    B = mc.vc.cs_block_len(300)
    assert B == 9600 and mc.vc.cs_block_len(1024) == 1 << 15 and mc.vc.cs_block_len(64) == 1024
    assert mc.cs_blocks(300, 0, B) == 1 and mc.cs_blocks(300, 0, B + 3 * B // 4 - 1) == 1
    assert mc.cs_blocks(300, 0, B + 3 * B // 4) == 2
    assert mc.cs_blocks(300, 1003, 28000) == 3
    assert mc.cs_tile_width(64, 1, False, H100_SXM_SMS) == 32
    picks = {(ct, st): mc.pick_ct(H100_SXM_SMS, ct, st) for ct, st in ((16, False), (16, True), (8, False))}
    assert all(picks.values()), picks
    for (ct, st), name in picks.items():
        case = mc.SCAN_CT[name]
        nb = mc.cs_blocks(case.M, 0, case.kw["N"])
        assert nb > 1 and mc.cs_tile_width(case.M, nb, st, H100_SXM_SMS) == ct, (name, nb)


@pytest.mark.parametrize("name", list(mc.SCAN_CT))
def test_scan_ct_case_has_stale_parents_as_named(name):
    """pick_ct tells the stale cases by their generator: the trace must agree."""
    from swirld_b200 import traces
    case = mc.SCAN_CT[name]
    tr = getattr(traces, case.gen)(**case.kw)
    stale = int(mc.vc.stale_info(tr)[0].sum())
    assert (stale > 1000) if case.gen == "adversarial_np" else stale == 0, stale
    ct, nb = mc.scan_shape(case, tr, H100_SXM_SMS)
    print("%s: %d stale, %d blocks, CT %d at %d SMs" % (name, stale, nb, ct, H100_SXM_SMS))
