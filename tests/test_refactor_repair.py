"""The refactorization's repair of a singular basis (-m gpu): the dense LU reports the nucleus column
without a pivot, Engine::refactor swaps the structural that the row permutation parked there for a slack,
and the solve goes on from the repaired basis."""
import dataclasses

import numpy as np
import pytest

import clp_b200
from clp_b200 import generators as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def test_dual_repairs_basis_with_two_identical_columns():
    base = G.random_sparse_lp(200, 1500, 0.04, 31)
    # column n is a copy of column 0
    s0, s1 = base.col_start[0], base.col_start[1]
    lp = dataclasses.replace(
        base, name="dup-column", n=base.n + 1,
        col_start=np.append(base.col_start, base.col_start[-1] + (s1 - s0)).astype(base.col_start.dtype),
        row_index=np.concatenate([base.row_index, base.row_index[s0:s1]]),
        element=np.concatenate([base.element, base.element[s0:s1]]),
        col_lower=np.append(base.col_lower, base.col_lower[0]),
        col_upper=np.append(base.col_upper, base.col_upper[0]),
        objective=np.append(base.objective, base.objective[0]),
        known_objective=None)
    # both copies basic, with the slacks of two rows of the column nonbasic: a singular 2 x 2 nucleus
    rows = base.row_index[s0:s0 + 2]
    status = np.full(lp.n + lp.m, clp_b200.ClpSimplex.atLowerBound, dtype=np.uint8)
    status[lp.n:] = clp_b200.ClpSimplex.basic
    status[[0, lp.n - 1]] = clp_b200.ClpSimplex.basic
    for r in rows:
        finite_lower = lp.row_lower[r] > -1e29
        status[lp.n + r] = clp_b200.ClpSimplex.atLowerBound if finite_lower else clp_b200.ClpSimplex.atUpperBound
    assert (status == clp_b200.ClpSimplex.basic).sum() == lp.m

    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    s.copyinStatus(status)
    assert s.dual() == 0
    o = O.OracleSimplex(lp)
    assert o.dual() == 0
    ref = o.objective_value
    assert abs(s.objectiveValue() - ref) <= 1e-8 * (1 + abs(ref)), (s.objectiveValue(), ref)
    assert O.kkt_violations(lp, s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution()) == 0
