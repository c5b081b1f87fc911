"""decide_fame and find_order on the branches the broad parity suite rarely or never reaches: coin rounds at every
mask width, a single seer (swirld.py:305 IndexError), tied consensus times above 64 members, and a checkpoint that
has to carry stakes and coin bits.  The cases and the oracle branch counters each relies on are in
tests/fame_cases.py; every test asserts those counters from its own oracle run, then compares the engine with the
oracle bit for bit (per-call new_c included) and can_see."""
import dataclasses

import numpy as np
import pytest

import fame_cases as fc
import oracle as orc
from test_gpu_parity import _check_round_kernel, impl  # noqa: F401  (impl: the four M <= 64 implementations)
from util import assert_same

pytestmark = pytest.mark.gpu

WIDE_COIN = [n for n, c in fc.CASES.items() if n.startswith("coin") and c.M > 64]
TWO_WORD_COIN = [n for n, c in fc.CASES.items() if n.startswith("coin") and c.M <= 64]
TIED = [n for n in fc.CASES if n.startswith("tied")]
SEER_NARROW = [n for n, c in fc.SEER_CASES.items() if c.M <= 64]
SEER_WIDE = [n for n, c in fc.SEER_CASES.items() if c.M > 64]


def _oracle(name, case, tr):
    o = fc.run_oracle(case, tr)
    assert not fc.missing(case, o["coverage"]), "%s no longer reaches %s" % (name, fc.missing(case, o["coverage"]))
    return o


def _engine(case, tr):
    from swirld_b200 import engine
    e = engine.Engine(tr.M, tr.N, case.stakes(), case.C)
    ncs = []
    for first, cnt in case.schedule(tr.N):
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    r = e.results()
    r.update(new_c_per_call=ncs, can_see=e.can_see(), stats=e.stats())
    return r


def _parity(name, case):
    tr = case.trace()
    o = _oracle(name, case, tr)
    r = _engine(case, tr)
    assert_same(o, r, what=name)
    assert np.array_equal(o["oracle"].can_see(), r["can_see"]), name + ": can_see differs"
    return r


# ---------------------------------------------------------------- coin rounds (swirld.py:267-272)
@pytest.mark.parametrize("name", WIDE_COIN)
def test_coin_rounds_wide(name):
    """k_w_fame_rounds<NJ> for NJ = 4, 8, 16 and 32, unit and zero stakes, batch and ragged schedules: counters
    coin_votes, coin_ones, coin_super, decide_after_c."""
    _parity(name, fc.CASES[name])


@pytest.mark.parametrize("name", TWO_WORD_COIN)
def test_coin_rounds_two_words(name, impl):
    """k_fame_rounds with two-word member masks (M = 33..64) on all four implementations: the coin counters."""
    case = fc.CASES[name]
    r = _parity(name, case)
    _check_round_kernel(impl, case.trace(), case.K, r)


# ---------------------------------------------------------------- tied consensus times (swirld.py:305-306)
@pytest.mark.parametrize("name", TIED)
def test_tied_times_wide(name):
    """Equal timestamps (t = index // tied) in the wide order kernels' radix-select median and received bisection:
    counters tied, median_odd, median_even."""
    _parity(name, fc.CASES[name])


# ---------------------------------------------------------------- a single seer (swirld.py:305 IndexError)
def _single_seer(name, case):
    """Engine and oracle call by call: the same new_c at every call, the IndexError at the same call, and identical
    state (rounds, witnesses, fame, consensus, order so far, can_see) when it is raised.  What a view holds after the
    raise is not compared: the reference has already ordered the earlier rounds of sorted(new_c) by then, and its
    state there is undefined."""
    from swirld_b200 import engine
    tr = case.trace()
    o = orc.Oracle(tr.M, case.stakes(), case.C)
    e = engine.Engine(tr.M, tr.N, case.stakes(), case.C)
    for i, (first, cnt) in enumerate(case.schedule(tr.N)):
        e.append_trace(tr, first, cnt)
        o.append(tr.slice(first, first + cnt))
        o.divide_rounds(first, cnt)
        e.divide_rounds(first, cnt)
        nc_o, nc_e = o.decide_fame(), e.decide_fame()
        assert sorted(nc_e) == sorted(nc_o), "%s: new_c differs at call %d" % (name, i)
        try:
            o.find_order(nc_o)
        except IndexError:
            assert_same(o.results(), e.results(), what="%s before the raise at call %d" % (name, i))
            assert np.array_equal(o.can_see(), e.can_see())
            with pytest.raises(IndexError):
                e.find_order(nc_e)
            break
        e.find_order(nc_e)
    else:
        pytest.fail("%s: the oracle never raised IndexError" % name)
    assert o.coverage()["single_seer"] == 1


@pytest.mark.parametrize("name", SEER_NARROW)
def test_single_seer_raises_at_the_same_call(name, impl):
    _single_seer(name, fc.SEER_CASES[name])


@pytest.mark.parametrize("name", SEER_WIDE)
def test_single_seer_raises_at_the_same_call_wide(name):
    _single_seer(name, fc.SEER_CASES[name])


# ---------------------------------------------------------------- checkpoint / resume with stakes and coin rounds
def test_checkpoint_resume_boundary_stake_coin(tmp_path):
    """M = 97 (NJ = 4, one live bit in the last word), zero stakes, C = 2: sw_save after half the calls, sw_load, and
    the second half on the resumed engine must use the saved stakes, coin period and coin bits (counters
    coin_votes, decide_after_c after the resume)."""
    from swirld_b200 import engine
    case = dataclasses.replace(fc.CASES["coin_nj4_m97_adv_c2_zero"], K=1500)
    tr = case.trace()
    o = _oracle("checkpoint", case, tr)
    sched = case.schedule(tr.N)
    half = len(sched) // 2
    # the oracle run of the first half alone: the second half must still cast coin votes and decide after C
    oh = orc.Oracle(tr.M, case.stakes(), case.C)
    oh.append(tr)
    for first, cnt in sched[:half]:
        oh.divide_rounds(first, cnt)
        oh.find_order(oh.decide_fame())
    cov_half = oh.coverage()
    assert o["coverage"]["coin_votes"] > cov_half["coin_votes"]
    assert o["coverage"]["decide_after_c"] > cov_half["decide_after_c"]
    e = engine.Engine(tr.M, tr.N, case.stakes(), case.C)
    ncs = []
    for first, cnt in sched[:half]:
        e.append_trace(tr, first, cnt)
        e.divide_rounds(first, cnt)
        nc = e.decide_fame()
        e.find_order(nc)
        ncs.append(sorted(nc))
    path = str(tmp_path / "ckpt.swb")
    e.save(path)
    e.close()
    e2 = engine.Engine.load(path, capacity=tr.N + 1000)
    assert e2.M == tr.M
    for first, cnt in sched[half:]:
        e2.append_trace(tr, first, cnt)
        e2.divide_rounds(first, cnt)
        nc = e2.decide_fame()
        e2.find_order(nc)
        ncs.append(sorted(nc))
    r = e2.results()
    r["new_c_per_call"] = ncs
    assert_same(o, r, what="resumed M=97 zero stakes C=2")
    assert np.array_equal(o["oracle"].can_see(), e2.can_see())
