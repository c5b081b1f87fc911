"""Where the time of one resident bench step goes, chunk by chunk: one step under torch.profiler (CUDA activities),
then per chunk the kernels, copies and their durations, the GPU-idle time, the time from the end of a chunk's last
kernel to the next chunk's first kernel, and the cluster round kernel's cycles in its step loop (sw_debug_counters).
    python tools/prof_chunks.py [workload] [out_dir]
Profile in a run of its own: tracing slows the host, so gaps here are upper bounds of the untraced ones."""
import collections
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
eng.debug_counters(clear=True)
l0 = eng.stats()["kernel_launches"]
acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
with torch.profiler.profile(activities=acts) as prof:
    step()
launches = eng.stats()["kernel_launches"] - l0
dbg = eng.debug_counters(clear=True).tolist()
path = os.path.join(out_dir, "prof_%s.pt.trace.json" % wl_name)
prof.export_chrome_trace(path)
clk = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip()

with open(path) as f:
    evs = json.load(f)["traceEvents"]
gpu = sorted((e for e in evs if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")),
             key=lambda e: e["ts"])
# a chunk ends with its decide_fame's last kernel: the fame kernel that is not followed by another fame kernel
fame = [i for i, e in enumerate(gpu) if "fame" in e["name"]]
ends = [i for j, i in enumerate(fame) if j + 1 == len(fame) or fame[j + 1] != i + 1]
# (rewind's fills, the L2 flush and the first chunk's can_see scan precede chunk 0: chunks 1.. are the steady state)
per = []
for c in range(1, len(ends)):
    seg = gpu[ends[c - 1] + 1: ends[c] + 1]
    busy, cur_a, cur_b = 0.0, None, None
    for e in seg:
        a, b = e["ts"], e["ts"] + e["dur"]
        if cur_b is None or a > cur_b:
            if cur_b is not None:
                busy += cur_b - cur_a
            cur_a, cur_b = a, b
        else:
            cur_b = max(cur_b, b)
    busy += cur_b - cur_a
    prev_end = gpu[ends[c - 1]]["ts"] + gpu[ends[c - 1]]["dur"]
    span = seg[-1]["ts"] + seg[-1]["dur"] - prev_end
    rc = [e for e in seg if "rounds_cluster" in e["name"]]
    per.append({"ops": [(e["name"].split("(")[0].split("<")[0].replace("void ", ""), round(e["dur"], 2)) for e in seg],
                "span_us": span, "busy_us": busy, "idle_us": span - busy,
                "gap_after_prev_chunk_us": next(e["ts"] for e in seg if e["cat"] == "kernel") - prev_end,
                "cluster_us": sum(e["dur"] for e in rc)})
agg = collections.OrderedDict()
for p in per:
    for name, d in p["ops"]:
        agg.setdefault(name, []).append(d)
nch = len(per)
mean = lambda xs: sum(xs) / max(1, len(xs))  # noqa: E731
res = {
    "workload": wl_name, "gpu": clk, "chunks_measured": nch, "kernel_launches_step": launches,
    "ops_per_chunk": {k: {"count": round(len(v) / nch, 2), "mean_us": round(mean(v), 2)} for k, v in agg.items()},
    "mean_chunk_span_us": round(mean([p["span_us"] for p in per]), 1),
    "mean_idle_us": round(mean([p["idle_us"] for p in per]), 1),
    "mean_gap_after_prev_chunk_us": round(mean([p["gap_after_prev_chunk_us"] for p in per]), 1),
    "mean_cluster_kernel_us": round(mean([p["cluster_us"] for p in per]), 1),
    "rc_dbg": {"loop_cycles_lead_cta": sum(dbg[0:6]), "steps": dbg[6], "launches": dbg[7], "handed": dbg[15]},
}
print(json.dumps(res, indent=1))
with open(os.path.join(out_dir, "prof_%s.json" % wl_name), "w") as f:
    json.dump({"summary": res, "chunks": per}, f, indent=1)
