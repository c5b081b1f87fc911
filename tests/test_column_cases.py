"""The cases of tests/column_cases.py reach what they are there for: ties decided by the key word each is named for,
negative and infinite consensus times, medians whose sum or half rounds, coins that all agree.  Runs the oracle only (no
GPU), so a change of a generator or of restamped() cannot quietly empty a case.  Run with -s to see the table."""
import pytest

import column_cases as cc


@pytest.mark.parametrize("name", list(cc.CASES))
def test_case_reaches_its_columns(name):
    case = cc.CASES[name]
    tr = case.trace()
    got = cc.analyse(tr, cc.run_oracle(case, tr))
    print("%-24s %s" % (name, " ".join("%s=%d" % kv for kv in got.items())))
    assert not cc.missing(case, got), "%s no longer reaches %s" % (name, cc.missing(case, got))
    assert got["ordered"] > 0
    if "coin_same" in case.needs:
        assert got["coin_ones"] in (0, got["coin_votes"])


def test_restamped_keeps_the_graph():
    import numpy as np
    from swirld_b200 import traces
    base = traces.adversarial(M=8, N=500, seed=3, p_cross=0.1, p_stale=0.3)
    for times in traces.TIME_KINDS:
        for sigs in traces.SIG_KINDS:
            tr = traces.restamped("adversarial", times, sigs, seed=3, M=8, N=500, p_cross=0.1, p_stale=0.3)
            for k in ("p0", "p1", "creator"):
                assert np.array_equal(getattr(tr, k), getattr(base, k))
            assert tr.t.dtype == np.float64 and tr.sig.dtype == np.uint8 and tr.sig.shape == (500, 64)
            assert np.isfinite(tr.t).all() or (times == "huge" and np.isfinite(tr.t[tr.t != 1e308]).all())
            assert not (tr.t == 0).any() and len({bytes(s) for s in tr.sig}) == tr.N
            if sigs.startswith("prefix"):
                P = int(sigs[6:].split("_")[0])
                lo = 1 if sigs.endswith("_coin") else 0
                assert (tr.sig[:, lo:P] == tr.sig[0, lo:P]).all()
                if lo:
                    assert np.array_equal(tr.sig[:, 0] >> 7, base.sig[:, 0] >> 7)
                    assert ((tr.sig[:, 0] & 0x7F) == (tr.sig[0, 0] & 0x7F)).all()
            else:
                assert (tr.sig[:, 0] >> 7 == int(sigs[-1])).all()
    assert traces.restamped("gossip", "const", "coin1", seed=2, M=4, N=50).t.tolist() == [1234.5] * 50
    t = traces.restamped("gossip", "tiny", "coin0", seed=2, M=4, N=50).t
    assert (t < 2.3e-308).all() and (t > 0).all()
