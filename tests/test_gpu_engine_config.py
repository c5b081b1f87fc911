"""Creating or loading an engine changes nothing that other engines of the process share: a checkpoint restores its
own kernel family without touching SW_FORCE_WIDE, and an engine with few members leaves the kernels' launch limits
where engines with many members need them."""
import hashlib

import pytest

import golden_specs as gs
import oracle as orc
from util import assert_same, load_golden

pytestmark = pytest.mark.gpu


def _divided(M, N, seed, K=500):
    """An engine over a gossip trace with its first call divided."""
    from swirld_b200 import engine, traces
    tr = traces.gossip(M, N, seed)
    e = engine.Engine(M, N)
    e.append_trace(tr)
    e.divide_rounds(0, K)
    return e, tr


def test_load_keeps_the_callers_kernel_choice(monkeypatch, tmp_path):
    """With SW_FORCE_WIDE=1, an engine created after a checkpoint was loaded still runs the any-M kernels: a batch of
    it and the saved engine is one kernel family."""
    from swirld_b200 import engine
    monkeypatch.setenv("SW_FORCE_WIDE", "1")
    e1, _ = _divided(8, 3000, 51)
    e1.save(str(tmp_path / "wide.ckpt"))
    engine.Engine.load(str(tmp_path / "wide.ckpt")).close()
    e2, _ = _divided(8, 3000, 52)
    engine.batch_decide_fame([e1, e2])


def test_forced_wide_checkpoint_loads_wide(monkeypatch, tmp_path):
    """A checkpoint of an SW_FORCE_WIDE=1 engine loads with the any-M kernels when the switch is unset, and goes on to
    the oracle's results."""
    from swirld_b200 import engine, traces
    from swirld_b200.engine import EngineError
    monkeypatch.setenv("SW_FORCE_WIDE", "1")
    e1, tr = _divided(8, 3000, 53)
    ew, _ = _divided(8, 3000, 54)
    e1.save(str(tmp_path / "wide.ckpt"))
    monkeypatch.delenv("SW_FORCE_WIDE")
    el = engine.Engine.load(str(tmp_path / "wide.ckpt"))
    ed, _ = _divided(8, 3000, 55)
    with pytest.raises(EngineError) as ei:
        engine.batch_decide_fame([ed, el])           # not one family with the M <= 64 engine ...
    assert ei.value.code == -8
    ncs = [sorted(engine.batch_decide_fame([ew, el])[1])]      # ... but with the forced-wide one
    # the loaded engine goes on with the rest of the schedule, against the oracle
    K = 500
    for first, cnt in traces.chunks(tr.N, K):
        if first > 0:
            el.divide_rounds(first, cnt)
            ncs.append(sorted(el.decide_fame()))
    got = el.results()
    got["new_c_per_call"] = ncs
    exp = orc.run_oracle(tr, K)
    exp["oracle"].close()
    assert_same(exp, got, keys=["round", "witness_table", "famous", "consensus"], what="loaded forced-wide engine")


def test_small_engine_leaves_a_large_one_working():
    """An M = 4 engine created after an M = 96 one: the M = 96 engine still runs its golden fixture (its can_see scan
    needs more dynamic shared memory than an M = 4 engine would)."""
    from swirld_b200 import engine, traces
    name = "g1_m96_n20000_s3_k3000"
    tr, K, stake = gs.make_trace(name)
    big = engine.Engine(tr.M, tr.N, stake)
    small = engine.Engine(4, 100)
    ncs = []
    for first, cnt in traces.chunks(tr.N, K):
        big.append_trace(tr, first, cnt)
        big.divide_rounds(first, cnt)
        nc = big.decide_fame()
        big.find_order(nc)
        ncs.append(sorted(nc))
    got = big.results()
    got["new_c_per_call"] = ncs
    g = load_golden(name)
    assert_same(g, got, what=name)
    assert bytes(g["can_see_sha256"]) == hashlib.sha256(big.can_see().tobytes()).digest(), name + ": can_see differs"
    small.close()
