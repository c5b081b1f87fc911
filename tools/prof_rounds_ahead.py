"""The round stream of the 64-member path (SW_ROUNDS_AHEAD) in one resident bench step: one step under torch.profiler
(CUDA activities), then the round stream's pieces (k_rb_prep, k_rounds_cluster, the hand-over launch of
k_rounds_batch) with the idle gaps between them, and how many of the fame kernels on the compute stream ran while a
cluster round kernel did.
    python tools/prof_rounds_ahead.py [workload] [out_dir]
Profile in a run of its own: tracing slows the host, so gaps here are upper bounds of the untraced ones."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "py-swirld_b200"))
import bench  # noqa: E402
import torch  # noqa: E402
from swirld_b200 import engine  # noqa: E402
from swirld_b200.traces import chunks  # noqa: E402

wl_name = sys.argv[1] if len(sys.argv) > 1 else "c3"
out_dir = sys.argv[2] if len(sys.argv) > 2 else "."
os.makedirs(out_dir, exist_ok=True)
wl = bench.WORKLOADS[wl_name]
M, N, K = wl["M"], wl["N"], wl["K"]
torch.cuda.set_device(0)
tr = bench.make_trace(wl, bench.rank_seed(0, wl))
eng = engine.Engine(M, N)
sched = list(chunks(N, K))
for first, cnt in sched:
    eng.append_trace(tr, first, cnt)


def step():
    eng.rewind()
    eng.flush_l2()
    eng.sync()
    for first, cnt in sched:
        eng.divide_rounds(first, cnt)
        eng.decide_fame()
    eng.sync()


for _ in range(3):
    step()
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.profiler.profile(activities=acts) as prof:
    step()
path = os.path.join(out_dir, "prof_ahead_%s.pt.trace.json" % wl_name)
prof.export_chrome_trace(path)
clk = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()

with open(path) as f:
    evs = json.load(f)["traceEvents"]
kern = sorted((e for e in evs if e.get("ph") == "X" and e.get("cat") == "kernel"), key=lambda e: e["ts"])
stream = lambda e: e.get("args", {}).get("stream", e.get("tid"))  # noqa: E731
name = lambda e: e["name"].split("(")[0].split("<")[0].replace("void ", "")  # noqa: E731
cluster = [e for e in kern if name(e) == "k_rounds_cluster"]
rs = stream(cluster[0]) if cluster else None
# a piece on the round stream: k_rb_prep .. the k_rounds_batch after it
pieces, cur = [], None
for e in kern:
    if stream(e) != rs:
        continue
    n = name(e)
    if n == "k_rb_prep":
        cur = {"a": e["ts"]}
    elif n == "k_rounds_batch" and cur is not None:
        cur["b"] = e["ts"] + e["dur"]
        pieces.append(cur)
        cur = None
gaps = [pieces[i + 1]["a"] - pieces[i]["b"] for i in range(len(pieces) - 1)]
fame = [e for e in kern if name(e).startswith("k_fame")]
over = sum(1 for f in fame if any(c["ts"] < f["ts"] + f["dur"] and f["ts"] < c["ts"] + c["dur"] for c in cluster))
res = {
    "workload": wl_name, "gpu": clk, "round_stream": rs,
    "compute_streams": sorted({stream(e) for e in kern} - {rs}),
    "pieces": len(pieces),
    "piece_us": [round(p["b"] - p["a"], 1) for p in pieces],
    "gap_between_pieces_us": [round(g, 1) for g in gaps],
    "mean_gap_us": round(sum(gaps) / max(1, len(gaps)), 1),
    "fame_kernels": len(fame), "fame_kernels_beside_a_cluster_kernel": over,
    "step_us": round(kern[-1]["ts"] + kern[-1]["dur"] - kern[0]["ts"], 1) if kern else None,
}
print(json.dumps(res, indent=1))
with open(os.path.join(out_dir, "prof_ahead_%s.json" % wl_name), "w") as f:
    json.dump(res, f, indent=1)
