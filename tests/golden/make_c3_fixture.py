"""Start basis of the C3 bench window (BASELINE.json configs[2], m=50k n=500k): the basis the GPU
engine reaches after ITER dual simplex iterations from the all-slack basis -- the analogue of
tests/golden/c2_status_it12000.npz (which the CPU oracle produced; at C3 the oracle would need days).
Needs a GPU:   python tests/golden/make_c3_fixture.py [ITER]   -> tests/golden/c3_status.npz"""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np
import clp_b200
import importlib.util
spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
bench = importlib.util.module_from_spec(spec); spec.loader.exec_module(bench)

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 60000
t = time.time()
fx = os.path.join(ROOT, "tests", "golden", "c3_status.npz")
if os.path.exists(fx):
    os.remove(fx)  # always from the all-slack basis
lp, _, _ = bench.build_workload("c3", 0)
print("generated", lp.name, lp.nnz, round(time.time() - t, 1), "s", flush=True)
s = clp_b200.ClpSimplex(); s.loadLP(lp)
s.setParameter("maximumIterations", iters); s.setParameter("logLevel", 1); s.setParameter("batch", 32)
t = time.time(); st = s.dual(); el = time.time() - t
print("status", st, "iterations", s.numberIterations(), "refactorizations", s.numberRefactorizations(), "nucleus", s.nucleusSize(),
      "seconds", round(el, 1), "it/s", round(s.numberIterations() / max(1e-9, s.secondsInLoop()), 1), flush=True)
np.savez_compressed(fx, status=s.statusArray(), iterations=s.numberIterations())
print("wrote", fx, os.path.getsize(fx), "bytes")
