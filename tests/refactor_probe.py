"""Refactorization time at the C2 bench basis (k ~ 4.7k): CUDA-event ms per refactorization
(gather + LU + inverse + transpose + host symbolic part).
  python tests/refactor_probe.py [frequency] [iterations]"""
import os, sys, json
sys.path.insert(0, ".")
import numpy as np
import clp_b200
from clp_b200 import generators as G

freq = int(sys.argv[1]) if len(sys.argv) > 1 else 50
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 600
lp = G.random_sparse_lp(10000, 100000, 0.01, 20260923)
z = np.load(os.path.join("tests", "golden", "c2_status_it12000.npz"))
s = clp_b200.ClpSimplex(); s.loadLP(lp); s.copyinStatus(z["status"].astype(np.uint8))
for k, v in (("timing", 1), ("factorizationFrequency", freq), ("maximumIterations", iters), ("batch", 16)):
    s.setParameter(k, v)
s.dual()
ph = s.phaseTimes()
nr = s.numberRefactorizations()
print(json.dumps({"refactorizations": nr, "nucleus": s.nucleusSize(),
                  "refactor_ms_each": ph["refactor"] / max(1, nr), "iterations": s.numberIterations()}))
