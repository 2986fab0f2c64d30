"""Per-kernel split of the refactorization at the C2 bench basis (k ~ 4.7k).

Two solves from the bench's start basis, each forcing a refactorization every `frequency` iterations:
the first without a profiler gives the CUDA-event ms per refactorization, the second runs under
torch.profiler (CUDA activities) and gives count and total device us per kernel name.  Only the
kernels of the refactorization are kept (factor.cu, the nucleus gather and the cuBLAS DGEMMs).
  python tests/refactor_profile.py [out.json] [frequency] [iterations]"""
import json
import os
import sys
import tempfile

sys.path.insert(0, ".")
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import clp_b200
from clp_b200 import generators as G

out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(tempfile.gettempdir(), "refactor_profile.json")
freq = int(sys.argv[2]) if len(sys.argv) > 2 else 50
iters = int(sys.argv[3]) if len(sys.argv) > 3 else 300

# kernel-name fragments of the refactorization; everything else (the simplex iterations) is dropped
REFACTOR = ("lu_", "trsm", "gemm", "identity", "transpose_kernel", "zero_padding", "gather_nucleus_matrix", "permute_weights")

lp = G.random_sparse_lp(10000, 100000, 0.01, 20260923)
status = np.load(os.path.join("tests", "golden", "c2_status_it12000.npz"))["status"].astype(np.uint8)


def solve():
    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    s.copyinStatus(status)
    for k, v in (("timing", 1), ("factorizationFrequency", freq), ("maximumIterations", iters), ("batch", 16)):
        s.setParameter(k, v)
    s.dual()
    return s


torch.cuda.init()
s = solve()
nr = s.numberRefactorizations()
timed = {"refactorizations": nr, "nucleus": s.nucleusSize(),
         "refactor_ms_each": s.phaseTimes()["refactor"] / max(1, nr), "iterations": s.numberIterations()}

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    s = solve()
    torch.cuda.synchronize()
nr_prof = s.numberRefactorizations()
kernels = {}
spans = []  # (start, end) us of each refactorization kernel on the device timeline
for ev in prof.events():
    if ev.device_type != torch.autograd.DeviceType.CUDA:
        continue
    name = ev.name
    if not any(f in name.lower() for f in REFACTOR) or "transpose_times" in name:
        continue
    spans.append((ev.time_range.start, ev.time_range.end, name))
    k = kernels.setdefault(name, {"count": 0, "total_us": 0.0})
    k["count"] += 1
    k["total_us"] += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
total = sum(v["total_us"] for v in kernels.values())
# device time from the nucleus gather to the last refactorization kernel before the next simplex
# iterations, and how much of it no refactorization kernel runs
spans.sort()
windows, idle_after = [], {}
for st, en, name in spans:
    if "gather_nucleus_matrix" in name or not windows:
        windows.append({"start": st, "end": st, "busy": 0.0, "last": name})
    w = windows[-1]
    if st > w["end"]:
        idle_after[w["last"]] = idle_after.get(w["last"], 0.0) + st - w["end"]
    w["busy"] += max(0.0, en - max(st, w["end"]))
    if en > w["end"]:
        w["end"], w["last"] = en, name
nw = max(1, len(windows))
device_window = {"us_per_refactor": sum(w["end"] - w["start"] for w in windows) / nw,
                 "busy_us_per_refactor": sum(w["busy"] for w in windows) / nw,
                 "idle_us_after_kernel_per_refactor": {k[:60]: v / nw for k, v in
                                                       sorted(idle_after.items(), key=lambda kv: -kv[1])[:8]}}
for v in kernels.values():
    v["us_per_refactor"] = v["total_us"] / max(1, nr_prof)
result = {"gpu": torch.cuda.get_device_name(0), **timed, "profiled_refactorizations": nr_prof,
          "kernel_us_per_refactor": total / max(1, nr_prof), "device_window": device_window,
          "kernels": dict(sorted(kernels.items(), key=lambda kv: -kv[1]["total_us"]))}
os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
with open(out, "w") as f:
    json.dump(result, f, indent=1)
print(json.dumps({k: v for k, v in result.items() if k != "kernels"}))
for name, v in result["kernels"].items():
    print(f"{v['count']:7d} {v['us_per_refactor']:10.1f} us/refactor  {name[:110]}")
