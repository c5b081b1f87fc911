"""Per-CTA step timings of the cluster round kernel (k_rounds_cluster, swirld_rcluster.cuh).

Runs resident steps of a workload (every call of bench.py's schedule: divide_rounds + decide_fame) on an engine
created with SW_RC_STEPS, reads the kernel's step log (Engine.rc_step_log: one record per step and CTA, in cycles of
that CTA's thread 0) and prints, per CTA, the mean and p90 of every phase of a step, and how many steps that CTA was
the critical sender (the largest interval from the arrival of the results to the end of its mask push: the CTA whose
masks the others wait for) and the critical tester (the largest interval from the arrival of the masks to its result
send: the CTA whose results the others wait for).

    python tools/rc_steps.py [c3] [c2] [--steps 2]
"""
import argparse
import os
import sys

os.environ.setdefault("SW_RC_STEPS", "16384")    # (read when the engine is created)
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(R, "py-swirld_b200"))
sys.path.insert(0, R)
import numpy as np  # noqa: E402

import bench  # noqa: E402
from swirld_b200 import engine  # noqa: E402
from swirld_b200.traces import chunks  # noqa: E402

# swirld_rcluster.cuh, RL_*
FIELDS = ["wait", "ctl", "bar1", "mask", "bar2", "push", "test1", "mwait", "test2", "bar3", "send", "defer",
          "sender", "tester"]


def run(name, steps):
    wl = bench.WORKLOADS[name]
    tr = bench.make_trace(wl, 1)
    e = engine.Engine(wl["M"], tr.N)
    e.append_trace(tr)
    logs = []
    for s in range(steps + 1):                   # the first is a warm-up
        e.rewind()
        e.rc_step_log()
        for first, cnt in chunks(tr.N, wl["K"]):
            e.divide_rounds(first, cnt)
            e.decide_fame()
        if s:
            logs.append(e.rc_step_log())
    L = np.concatenate(logs).astype(np.int64)    # [steps, CTA, field]
    S, ncta = L.shape[0], L.shape[1]
    crit_s = np.bincount(L[:, :, FIELDS.index("sender")].argmax(1), minlength=ncta)
    crit_t = np.bincount(L[:, :, FIELDS.index("tester")].argmax(1), minlength=ncta)
    print("%s: M=%d, K=%d, %d steps logged over %d resident step(s); cycles of each CTA's thread 0" % (
        name, wl["M"], wl["K"], S, steps))
    print("cta " + " ".join("%13s" % f for f in FIELDS) + "  crit_sender crit_tester")
    for q in range(ncta):
        cells = ["%6.0f/%6.0f" % (L[:, q, i].mean(), np.percentile(L[:, q, i], 90)) for i in range(len(FIELDS))]
        print("%3d " % q + " ".join(cells) + "  %11d %11d" % (crit_s[q], crit_t[q]))
    allm = [L[:, :, i].mean() for i in range(len(FIELDS))]
    print("all " + " ".join("%13.0f" % v for v in allm))
    step = L[:, :, :FIELDS.index("defer") + 1].sum(2).mean()
    print("per step (mean over CTAs of the sum of the phases): %.0f cycles; critical sender interval (max over CTAs) "
          "mean %.0f, critical tester interval mean %.0f" % (
              step, L[:, :, FIELDS.index("sender")].max(1).mean(), L[:, :, FIELDS.index("tester")].max(1).mean()))
    print("(mean/p90 per cell)")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["c3", "c2"])
    ap.add_argument("--steps", type=int, default=1)
    a = ap.parse_args()
    for w in a.workloads:
        run(w, a.steps)
