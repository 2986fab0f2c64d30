"""Inverse of the C2 bench nucleus through clp_b200.denseInvert, saved for a bitwise comparison between
two builds of the refactorization.

The nucleus is built on the host from the bench's start basis: the rows whose slack is nonbasic times
the basic structural columns, unscaled, dense (k ~ 4.7k).  Writes X as .npy when a path is given and prints k, info, the
largest |N X - I| and a SHA-256 of X's bytes.
  python tests/nucleus_inverse.py [out.npy]"""
import hashlib
import json
import os
import sys

sys.path.insert(0, ".")
import numpy as np
import scipy.sparse as sp

import clp_b200
from clp_b200 import generators as G

out = sys.argv[1] if len(sys.argv) > 1 else None
lp = G.random_sparse_lp(10000, 100000, 0.01, 20260923)
status = np.load(os.path.join("tests", "golden", "c2_status_it12000.npz"))["status"]
basic = status == clp_b200.ClpSimplex.basic
cols = np.nonzero(basic[:lp.n])[0]
rows = np.nonzero(~basic[lp.n:])[0]
A = sp.csc_matrix((lp.element, lp.row_index, lp.col_start), shape=(lp.m, lp.n))
N = A[:, cols].toarray()[rows, :]
info, X = clp_b200.denseInvert(N)
res = float(np.abs(N @ X - np.eye(len(rows))).max()) if info == 0 else None
if out:
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    np.save(out, X)
print(json.dumps({"k": len(rows), "info": info, "max_abs_NX_minus_I": res, "max_abs_X": float(np.abs(X).max()),
                  "sha256": hashlib.sha256(np.ascontiguousarray(X).tobytes()).hexdigest()}))
