"""CPU tests of tests/iteration_ref.py, the high-precision reference of one dual simplex iteration: its solves
agree with the oracle's factorization, and on its own it takes the oracle's pivots."""
import os
import re
import tempfile

import numpy as np
import pytest

from clp_b200 import generators as G
from oracle import oracle as O

import iteration_ref as R


def _basis_from_oracle(lp, iters):
    o = O.OracleSimplex(lp)
    o.set_option("maximumIterations", iters)
    o.dual()
    st = o.status()
    return [j for j in range(lp.n + lp.m) if st[j] == 1]


@pytest.mark.parametrize("shape", [(60, 300, 0.1, 40), (300, 2000, 0.03, 250), (1000, 6000, 0.01, 900)])
def test_reference_solves_agree_with_the_oracle(shape):
    m, n, dens, iters = shape
    lp = G.random_sparse_lp(m, n, dens, 5)
    basis = _basis_from_oracle(lp, iters)
    o = O.OracleSimplex(lp)
    rc, pv = o.factorize(basis)
    assert rc == 0
    ref = R.Basis(R.ext_matrix(lp), pv)
    assert ref.cond1() < 1e8
    rng = np.random.default_rng(2)
    for _ in range(3):
        b = rng.standard_normal(lp.m)
        x, xo = ref.ftran(b), o.ftran(b)
        np.testing.assert_allclose(x, xo, rtol=1e-9, atol=1e-9 * (1 + np.abs(xo).max()))
        y, yo = ref.btran(b), o.btran(b)
        np.testing.assert_allclose(y, yo, rtol=1e-9, atol=1e-9 * (1 + np.abs(yo).max()))
        # and the refinement leaves a residual at the level of float64 rounding of the result
        assert np.abs(ref.B @ x - b).max() <= 1e-13 * (1 + np.abs(x).max()) * (1 + abs(ref.B).max())


def test_reference_iteration_takes_the_pivots_of_the_oracle():
    """from the all-slack basis the reference's CHUZR -> BTRAN -> PRICE -> CHUZC -> dual update -> FTRANs ->
    primal / DSE update takes the first 100 pivots of the oracle run with the bucketed ratio test"""
    lp = G.random_sparse_lp(300, 3000, 0.03, 17)
    N = 100
    tf = tempfile.TemporaryFile(mode="w+b")
    old = os.dup(2)
    os.dup2(tf.fileno(), 2)
    try:
        o = O.OracleSimplex(lp)
        for k, v in (("logLevel", 3), ("bucketedRatioTest", 1), ("maximumIterations", N)):
            o.set_option(k, v)
        o.dual()
    finally:
        os.dup2(old, 2)
        os.close(old)
    tf.seek(0)
    pat = re.compile(r"TRACE (\d+) out=(\d+) in=(\d+) sigma=(-?\d+) thetaD=(\S+) thetaP=(\S+)")
    trace = [pat.match(l) for l in tf.read().decode(errors="ignore").splitlines() if l.startswith("TRACE")]
    assert len(trace) == N
    aext = R.ext_matrix(lp)
    amax = max(1.0, float(np.abs(lp.element).max()))
    s = R.dual_feasible_start(lp)
    for it, mt in enumerate(trace):
        res = R.step(aext, s, amax)
        assert res is not None, it
        r, out, q, sigma, theta = res
        assert (out, q, sigma) == (int(mt.group(2)), int(mt.group(3)), int(mt.group(4))), (it, res, mt.group(0))
        tb = float(mt.group(5))
        assert abs(theta - tb) <= 1e-6 * (1e-9 + abs(tb)) + 1e-12, (it, theta, tb)
