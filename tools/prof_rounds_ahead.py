"""The round stream of the 64-member path (SW_ROUNDS_AHEAD) in one resident bench step: one step under torch.profiler
(CUDA activities), then the round stream's pieces (k_rb_prep, k_rounds_cluster, the hand-over launch of
k_rounds_batch) with each kernel's duration and the gaps inside and between pieces (negative where a piece's prep ran
beside the piece before it), the idle time from one cluster kernel to the next, the can_see scan of the first
call, the step loop's cycles per cluster launch and the hand-overs (sw_debug_counters), and how many of the fame
kernels on the compute stream ran while a cluster round kernel did.
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
# the step loop's cycles and the hand-overs of untraced steps (slots: [0, 6) phase cycles of CTA 0's control warp,
# summed over launches; 7 cluster launches; 15 launches that handed work to k_rounds_batch)
eng.debug_counters()
for _ in range(3):
    step()
dbg = eng.debug_counters()
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
end = lambda e: e["ts"] + e["dur"]  # noqa: E731
cluster = [e for e in kern if name(e) == "k_rounds_cluster"]
rs = stream(cluster[0]) if cluster else None
# a piece: its k_rb_prep (on a stream of its own, or on the round stream), k_rounds_cluster and the k_rounds_batch after
# it on the round stream.  A piece's prep is the last k_rb_prep off the compute stream that ends before its cluster kernel.
comp = {stream(e) for e in kern if name(e).startswith("k_fame")}
preps = [e for e in kern if name(e) == "k_rb_prep" and stream(e) not in comp]
pieces, cur = [], None
for e in kern:
    if stream(e) != rs:
        continue
    n = name(e)
    if n == "k_rounds_cluster":
        before = [p for p in preps if end(p) <= e["ts"]]
        cur = {"prep": before[-1], "cluster": e} if before else None
    elif n == "k_rounds_batch" and cur is not None:
        cur["batch"] = e
        pieces.append(cur)
        cur = None
r1 = lambda x: round(x, 1)  # noqa: E731
steps = int(dbg[6])
launches = max(1, int(dbg[7]))
cyc = float(sum(dbg[:6])) / launches
per_piece = [{
    "prep_us": r1(p["prep"]["dur"]),
    "prep_to_cluster_us": r1(p["cluster"]["ts"] - end(p["prep"])),
    "cluster_us": r1(p["cluster"]["dur"]),
    "cluster_to_batch_us": r1(p["batch"]["ts"] - end(p["cluster"])),
    "batch_us": r1(p["batch"]["dur"]),
    "piece_us": r1(end(p["batch"]) - p["prep"]["ts"]),
} for p in pieces]
gaps = [pieces[i + 1]["prep"]["ts"] - end(pieces[i]["batch"]) for i in range(len(pieces) - 1)]
# between two step loops the round stream does everything but rounds: the end of one cluster kernel to the start of the
# next, plus the next cluster kernel's own time outside its step loop (its duration less the loop's cycles)
c2c = [pieces[i + 1]["cluster"]["ts"] - end(pieces[i]["cluster"]) for i in range(len(pieces) - 1)]
# the can_see scan of the first call: every k_cs_ kernel that ends before the first cluster kernel starts, and all of them
cs = [e for e in kern if name(e).startswith("k_cs_")]
first_c = cluster[0]["ts"] if cluster else float("inf")
cs_before = [e for e in cs if end(e) <= first_c]
span = lambda xs: r1(end(xs[-1]) - xs[0]["ts"]) if xs else 0.0  # noqa: E731
fame = [e for e in kern if name(e).startswith("k_fame")]
over = sum(1 for f in fame if any(c["ts"] < end(f) and f["ts"] < end(c) for c in cluster))
mean = lambda xs: r1(sum(xs) / max(1, len(xs)))  # noqa: E731
res = {
    "workload": wl_name, "gpu": clk, "round_stream": rs,
    "compute_streams": sorted({stream(e) for e in kern} - {rs}),
    "calls": len(sched), "pieces": len(pieces),
    "per_piece": per_piece,
    "gap_between_pieces_us": [r1(g) for g in gaps],
    "mean_gap_us": mean(gaps),
    "cluster_end_to_next_cluster_start_us": [r1(g) for g in c2c],
    "mean_cluster_end_to_next_cluster_start_us": mean(c2c),
    "mean_prep_us": mean([p["prep_us"] for p in per_piece]),
    "mean_batch_us": mean([p["batch_us"] for p in per_piece]),
    "sum_cluster_us": r1(sum(p["cluster"]["dur"] for p in pieces)),
    "first_scan_before_first_cluster_us": span(cs_before),
    "scan_kernels_us_total": r1(sum(e["dur"] for e in cs)),
    "scan_span_us": span(cs),
    "step_loop_steps_per_bench_step": steps / 3.0,
    "cluster_launches_per_bench_step": launches / 3.0,
    "step_loop_cycles_per_launch": round(cyc, 0),
    "step_loop_cycles_per_bench_step": round(cyc * launches / 3.0, 0),
    "hand_overs_per_bench_step": int(dbg[15]) / 3.0,
    "fame_kernels": len(fame), "fame_kernels_beside_a_cluster_kernel": over,
    "step_us": r1(end(kern[-1]) - kern[0]["ts"]) if kern else None,
}
print(json.dumps({k: v for k, v in res.items() if k not in ("per_piece",)}, indent=1))
for i, p in enumerate(per_piece):
    print("piece %2d: %s" % (i, json.dumps(p)))
with open(os.path.join(out_dir, "prof_ahead_%s.json" % wl_name), "w") as f:
    json.dump(res, f, indent=1)
