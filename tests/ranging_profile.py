"""Time of full sensitivity analysis on the LP whose solve bench.py times for wall_to_optimal_s
(random_sparse_lp(3000, 30000, 0.01, 20260923)), optionally also C5 (transportation_lp()).

After the solve: dualRanging with values and primalRanging over all n+m sequences, timed by the host
clock (each call ends in a stream synchronisation) and by CUDA events recorded around it after a device
synchronisation; then the same calls once more under torch.profiler (CUDA activities) for the time per
kernel.  The PRICE pass reads A once per kRangeBatch (16) tableau rows: its algorithmic bytes are set
against the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.
  python tests/ranging_profile.py [out.json] [c5]"""
import json
import os
import re
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, ".")
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import clp_b200
from clp_b200 import generators as G

out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "ranging_profile.json")
with_c5 = len(sys.argv) > 2 and sys.argv[2] == "c5"
BATCH = 16
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t0 = time.perf_counter()
    res = fn()
    wall = time.perf_counter() - t0
    e1.record()
    torch.cuda.synchronize()
    return res, wall * 1e3, e0.elapsed_time(e1)


def measure(name, lp):
    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    t0 = time.perf_counter()
    assert s.dual() == 0
    solve_s = time.perf_counter() - t0
    st = s.statusArray()
    basics = int((st == 1).sum())
    s.dualRanging(np.arange(min(64, lp.n + lp.m)), values=True)  # warm-up: module load, first launches
    s.primalRanging(np.arange(min(64, lp.n + lp.m)))
    dual, dual_wall, dual_ev = timed(lambda: s.dualRanging(values=True))
    primal, primal_wall, primal_ev = timed(lambda: s.primalRanging())
    kernels = {}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.dualRanging(values=True)
        s.primalRanging()
        torch.cuda.synchronize()
    for ev in prof.events():
        found = re.search(r"range_\w+_kernel", ev.name)
        if ev.device_type != torch.autograd.DeviceType.CUDA or not found:
            continue
        k = kernels.setdefault(found.group(0), {"count": 0, "total_us": 0.0})
        k["count"] += 1
        k["total_us"] += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
    price = kernels.get("range_dual_price_kernel")
    batches = (basics + BATCH - 1) // BATCH
    # per pass: A's values, row indices and column starts once, status and dj of the columns, the rho block once
    price_bytes = batches * (12.0 * lp.nnz + 4.0 * (lp.n + 1) + 9.0 * lp.n + 8.0 * BATCH * lp.m + 9.0 * lp.m)
    res = {"lp": name, "m": lp.m, "n": lp.n, "nnz": lp.nnz, "solve_s": solve_s, "iterations": s.numberIterations(),
           "nucleus": s.nucleusSize(), "basic_sequences": basics,
           "dual_ranging_with_values": {"wall_ms": dual_wall, "cuda_event_ms": dual_ev},
           "primal_ranging": {"wall_ms": primal_wall, "cuda_event_ms": primal_ev},
           "price_passes": batches, "price_algorithmic_bytes": price_bytes,
           "kernels": dict(sorted(kernels.items(), key=lambda kv: -kv[1]["total_us"]))}
    if price:
        res["price_kernel_us"] = price["total_us"]
        res["price_share_of_3.35TBps"] = price_bytes / (price["total_us"] * 1e-6) / HBM_BYTES_PER_S
    finite = np.isfinite(dual[0]) & (dual[0] < 1e300)
    res["finite_cost_increases"] = int(finite.sum())
    return res


torch.cuda.init()
result = {"card": card(), "runs": [measure("rand-3000x30000", G.random_sparse_lp(3000, 30000, 0.01, 20260923))]}
if with_c5:
    result["runs"].append(measure("C5-transport", G.transportation_lp()))
os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
with open(out, "w") as f:
    json.dump(result, f, indent=1)
print(json.dumps({"card": result["card"]}))
for r in result["runs"]:
    print(json.dumps({k: v for k, v in r.items() if k != "kernels"}))
    for name, v in r["kernels"].items():
        print(f"  {v['count']:7d} {v['total_us']:12.1f} us  {name}")
