"""Generate tests/golden/*.npz by running the UNMODIFIED reference
(py-swirld's swirld.py, imported in place through oracle/ref_harness.py)
on the traces and call schedules of oracle/golden_specs.py.

With a checkout of py-swirld at $SWIRLD_REFERENCE:
    python oracle/make_golden.py [name ...]
    python oracle/make_golden.py --nodes     # golden_specs.NODE_FIXTURES, from a fresh simulation
    python oracle/make_golden.py --views [name ...]   # golden_specs.VIEW_FIXTURES

Each fixture holds, in index space: round[N], witness_table[R,M], famous[N]
(-1 = no entry), consensus[], transactions[], the per-call new_c lists
(flattened), sha256 of the can_see matrix (and the matrix itself when small).
"""
from __future__ import annotations

import hashlib
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
sys.path.insert(0, HERE)

import golden_specs as gs  # noqa: E402
import ref_harness as rh   # noqa: E402


def main(names):
    os.makedirs(gs.GOLDEN_DIR, exist_ok=True)
    for name in names:
        tr, K, stake = gs.make_trace(name)
        t0 = time.time()
        r = rh.run_reference(tr, K, stake)
        cs = rh.can_see_matrix(r["can_see_node"], tr.N, tr.M)
        flat, offs = [], [0]
        for nc in r["new_c_per_call"]:
            flat.extend(nc)
            offs.append(len(flat))
        out = dict(
            round=r["round"], witness_table=r["witness_table"], famous=r["famous"],
            consensus=r["consensus"], transactions=r["transactions"],
            new_c_flat=np.array(flat, dtype=np.int32), new_c_offs=np.array(offs, dtype=np.int32),
            can_see_sha256=np.frombuffer(hashlib.sha256(cs.tobytes()).digest(), dtype=np.uint8),
            trace_sha256=np.frombuffer(hashlib.sha256(
                tr.p0.tobytes() + tr.p1.tobytes() + tr.creator.tobytes() + tr.t.tobytes()
                + tr.sig.tobytes()).digest(), dtype=np.uint8),
            ref_seconds=np.array([r["t_divide_rounds"], r["t_decide_fame"], r["t_find_order"]]),
        )
        if cs.size <= 200000:
            out["can_see"] = cs
        np.savez_compressed(gs.path(name), **out)
        print("%-32s N=%d M=%d K=%d  max_r=%d wit=%d famous=%d/%d cons=%d ordered=%d  "
              "ref dr=%.2fs df=%.2fs fo=%.2fs  (%.1fs, %d KB)" % (
                  name, tr.N, tr.M, K, r["round"].max(), int(r["witness"].sum()),
                  int((r["famous"] >= 0).sum()), int((r["famous"] == 1).sum()),
                  len(r["consensus"]), len(r["transactions"]),
                  r["t_divide_rounds"], r["t_decide_fame"], r["t_find_order"],
                  time.time() - t0, os.path.getsize(gs.path(name)) // 1024), flush=True)


def main_nodes():
    """Each fixture: one node's arrival trace and call schedule (chunk sizes) from a gossip simulation over the
    tests' host with the oracle as the engine, and the reference's replay of that trace and schedule."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import node_sim
    from oracle_engine import OracleEngine
    sim = node_sim.run_sim(4, 400, OracleEngine, capacity=64, seed=5)
    for name, nd in zip(gs.NODE_FIXTURES, sim):
        tr, sizes = node_sim.node_trace(nd)
        r = rh.run_reference(tr, sizes)
        np.savez_compressed(gs.path(name), M=tr.M, p0=tr.p0, p1=tr.p1, creator=tr.creator, t=tr.t, sig=tr.sig,
                            sizes=np.array(sizes, np.int32), round=r["round"], famous=r["famous"],
                            consensus=r["consensus"], transactions=r["transactions"])
        print("%-24s N=%d calls=%d ordered=%d" % (name, tr.N, len(sizes), len(r["transactions"])), flush=True)


def main_views(names):
    """Each fixture: a node view of a generator trace (golden_specs.VIEW_FIXTURES) and the reference's replay of it
    with one call per sync, stored as main_nodes stores its fixtures."""
    for name in names:
        tr, sizes = gs.make_view(name)
        t0 = time.time()
        r = rh.run_reference(tr, sizes)
        np.savez_compressed(gs.path(name), M=tr.M, p0=tr.p0, p1=tr.p1, creator=tr.creator, t=tr.t, sig=tr.sig,
                            sizes=np.array(sizes, np.int32), round=r["round"], famous=r["famous"],
                            consensus=r["consensus"], transactions=r["transactions"])
        print("%-28s N=%d calls=%d ordered=%d  (%.1fs)" % (name, tr.N, len(sizes), len(r["transactions"]),
                                                           time.time() - t0), flush=True)


if __name__ == "__main__":
    if not rh.reference_available():
        sys.exit("set SWIRLD_REFERENCE to a checkout of py-swirld")
    if sys.argv[1:] == ["--nodes"]:
        main_nodes()
    elif sys.argv[1:2] == ["--views"]:
        main_views(sys.argv[2:] or list(gs.VIEW_FIXTURES))
    else:
        main(sys.argv[1:] or list(gs.SPECS))
