"""Full-size parity probe (not a pytest test; tests/test_fullsize.py holds the -m gpu versions):
BASELINE.json configs[1] (C2, random 10 000 x 100 000, planted optimum), configs[3] (C4, staircase
m=n=20 000) and configs[4] (C5, degenerate transportation 5 050 x 250 000) solved on the GPU from the
all-slack basis and audited: KKT on the true data (oracle.kkt_violations) and the optimum against
the planted value / HiGHS dual simplex (tests/golden/fullsize_highs.json).
  python tests/fullsize_probe.py [c2] [c5] [c4] [c4s] [key=value ...]"""
import json, os, sys, time
sys.path.insert(0, ".")
import numpy as np
import clp_b200
from clp_b200 import generators as G
from oracle import oracle as O

ref = {}
p = os.path.join("tests", "golden", "fullsize_highs.json")
if os.path.exists(p):
    ref = json.load(open(p))
extra = {a.split("=")[0]: float(a.split("=")[1]) for a in sys.argv[1:] if "=" in a}
which = [a for a in sys.argv[1:] if "=" not in a] or ["c5", "c4"]
cases = {"c2": ("C2 rand-10000x100000", lambda: G.random_sparse_lp(10000, 100000, 0.01, 20260923), [{}]),
         "c5": ("C5 transport-50x5000", lambda: G.transportation_lp(50, 5000, 20260926), [{}, {"perturbation": 50}]),
         "c4": ("C4 staircase-20000", lambda: G.staircase_lp(40, 500, 20260925), [{}]),
         "c4s": ("C4 staircase-20000", lambda: G.staircase_lp(40, 500, 20260925), [{"scaling": 3, "perturbation": 50}])}
out = []
for w in which:
    name, gen, variants = cases[w]
    lp = gen()
    for params in variants:
        params = dict(params, **extra)
        s = clp_b200.ClpSimplex(); s.loadLP(lp)
        s.setParameter("maximumSeconds", 900)
        for k, v in params.items():
            s.setParameter(k, v)
        t = time.time(); st = s.dual(); el = time.time() - t
        kkt = O.kkt_violations(lp, s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution()) if st == 0 else None
        expect = lp.known_objective if lp.known_objective is not None else ref.get(name, {}).get("objective")
        r = {"case": name, "params": params, "m": lp.m, "n": lp.n, "nnz": lp.nnz, "status": st, "objective": s.objectiveValue(),
             "iterations": s.numberIterations(), "refactorizations": s.numberRefactorizations(), "seconds": round(el, 2),
             "seconds_in_loop": round(s.secondsInLoop(), 2),
             "iterations_per_sec": round(s.numberIterations() / max(1e-9, s.secondsInLoop()), 1), "nucleus": s.nucleusSize(),
             "kkt_violations": kkt, "expected_objective": expect,
             "n_basic": int((s.statusArray() == 1).sum())}
        if expect is not None:
            r["rel_diff"] = abs(r["objective"] - expect) / (1 + abs(expect))
        print(json.dumps(r), flush=True)
        out.append(r)
outdir = os.environ.get("CLPB_PROBE_OUT", ".")
os.makedirs(outdir, exist_ok=True)
json.dump(out, open(os.path.join(outdir, "fullsize_probe_%s.json" % "_".join(which)), "w"), indent=1)
