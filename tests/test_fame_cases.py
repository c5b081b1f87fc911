"""The fame / order cases of tests/fame_cases.py reach the branches they are there for.  Runs the oracle only (no
GPU), so a generator or schedule change that empties a case fails here, before any parity run could pass vacuously.
Run with -rA or -s to see each case's counters."""
import pytest

import fame_cases as fc


@pytest.mark.parametrize("name", list(fc.ALL_CASES))
def test_case_reaches_its_branches(name):
    case = fc.ALL_CASES[name]
    r = fc.run_oracle(case)
    cov = r["coverage"]
    print("%s: %s" % (name, " ".join("%s=%d" % kv for kv in cov.items())))
    assert not fc.missing(case, cov), "%s no longer reaches %s" % (name, fc.missing(case, cov))
    if "coin_votes" in case.needs:
        assert 0 < cov["coin_ones"] < cov["coin_votes"], "%s: the coin must come up both 0 and 1" % name
    assert cov["decide_after_c"] <= cov["decisions"]
    if "single_seer" in case.needs:
        assert r["raised_at"] >= 0 and cov["single_seer"] == 1
    else:
        assert r["raised_at"] == -1 and cov["single_seer"] == 0


def test_coverage_starts_at_zero_and_is_per_view():
    import oracle as orc
    case = fc.CASES["coin_m40_adv_c3"]
    tr = case.trace()
    a = orc.Oracle(tr.M, None, case.C)
    assert set(a.coverage().values()) == {0} and tuple(a.coverage()) == orc.COVERAGE
    r = fc.run_oracle(case, tr)
    assert r["coverage"]["coin_votes"] > 0
    assert set(a.coverage().values()) == {0}
    assert r["coverage"] == orc.run_oracle(tr, case.K, None, case.C)["coverage"]
