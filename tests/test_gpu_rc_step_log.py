"""The cluster round kernel's per-CTA step log (SW_RC_STEPS, sw_rc_step_log, tools/rc_steps.py): an engine with the
log computes what its twin without it computes, logs one record per step and CTA of every cluster launch, and its
sender / tester intervals are made of the phases they span."""
import numpy as np
import pytest

from util import assert_same

pytestmark = pytest.mark.gpu

# swirld_rcluster.cuh, RL_*
WAIT, CTL, BAR1, MASK, BAR2, PUSH, TEST1, MWAIT, TEST2, BAR3, SEND, DEFER, SENDER, TESTER = range(14)


def test_gpu_rc_step_log(monkeypatch):
    from swirld_b200 import engine, traces
    tr = traces.gossip(16, 12000, seed=5)
    monkeypatch.setenv("SW_ROUNDS_AHEAD", "0")                 # one cluster launch per call
    monkeypatch.setenv("SW_RC_STEPS", "4096")
    a = engine.Engine(16, tr.N)
    monkeypatch.delenv("SW_RC_STEPS")
    b = engine.Engine(16, tr.N)
    assert b.rc_step_log().shape == (0, 16, 16)                 # no log unless asked for
    for e in (a, b):
        e.append_trace(tr)
    logs = []
    for first in range(0, tr.N, 4000):
        for e in (a, b):
            e.divide_rounds(first, min(4000, tr.N - first))
            e.decide_fame()
        logs.append(a.rc_step_log())
    assert_same(b.results(), a.results(), what="with the step log")
    L = np.concatenate(logs).astype(np.int64)
    assert L.shape[0] > 3 and L.shape[1:] == (16, 16)
    assert (L[:, :, SENDER] == L[:, :, CTL:PUSH + 1].sum(2)).all()
    assert (L[:, :, TESTER] == L[:, :, TEST2:SEND + 1].sum(2)).all()
    assert (L[:, :, SENDER] > 0).all()                         # every (step, CTA) record was written
