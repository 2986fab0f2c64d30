"""Profiling target (not a test): a short mid-solve window of the C2 workload without graph
replay, so that a kernel profiler (ncu, torch.profiler) sees ordinary kernel launches."""
import os, sys
sys.path.insert(0, ".")
import numpy as np
import clp_b200
from bench import build_workload, default_cycle

name = sys.argv[1] if len(sys.argv) > 1 else "c2"
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 40
lp, status, start = build_workload(name)
s = clp_b200.ClpSimplex(); s.loadLP(lp)
if status is not None:
    s.copyinStatus(status)
s.setParameter("useGraph", 0); s.setParameter("batch", 8)
s.setMaximumIterations(iters); s.setFactorizationFrequency(default_cycle(lp.m))
if len(sys.argv) > 3: s.setParameter('usePriceTma', int(sys.argv[3]))
if len(sys.argv) > 4: s.setLogLevel(int(sys.argv[4]))
st = s.dual()
print("status", st, "iterations", s.numberIterations(), "nucleus", s.nucleusSize(), "objective", s.objectiveValue())
