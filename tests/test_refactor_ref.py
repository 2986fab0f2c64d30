"""CPU tests of tests/refactor_ref.py, the reference of the refactorization and refresh tests: the restated LU is
an LU and takes scipy's pivots where neither a tie nor the key truncation decides, it reports the planted column
of a singular matrix, its bounds hold for a plain float64 inverse, and the restated refresh reproduces the
oracle's duals and primals at an optimal basis."""
import numpy as np
import pytest
import scipy.linalg as sla

from conftest import load_golden
from oracle import oracle as O

import iteration_ref as R
import refactor_ref as F


@pytest.mark.parametrize("k", [1, 2, 31, 32, 33, 100, 257])
def test_restated_lu_agrees_with_scipy(k):
    a = np.random.default_rng(k).standard_normal((k, k))
    piv, L, Um, info = F.lu_pivot_rule(a)
    assert info == 0
    _, ipiv = sla.lu_factor(a)
    np.testing.assert_array_equal(piv, ipiv)
    perm = F.row_order(piv)
    assert sorted(perm) == list(range(k))
    assert np.abs(L @ Um - a[perm]).max() <= F.gamma(k) * (np.abs(L) @ np.abs(Um)).max()
    assert np.abs(np.tril(L, -1)).max(initial=0.0) <= 1.0 + 2.0 ** -30


def test_pivot_rule_ties_and_truncation():
    # equal maxima: the smallest row wins
    a = np.array([[1.0, 2.0, 0.0], [-3.0, 1.0, 1.0], [3.0, 0.0, 1.0]])
    assert F.lu_pivot_rule(a)[0][0] == 1
    # maxima that differ inside the low 20 bits compare equal: still the smallest row, although row 2 is larger
    a[2, 0] = np.nextafter(3.0, 4.0)
    assert F.lu_pivot_rule(a)[0][0] == 1
    a[2, 0] = 3.0 * (1.0 + 2.0 ** -30)
    assert F.lu_pivot_rule(a)[0][0] == 2
    # the threshold is compared on the truncated magnitude
    assert F.truncated(1.0e-11) < 1.0e-11
    assert F.lu_pivot_rule(np.array([[1.0e-11]]))[3] == 1
    assert F.lu_pivot_rule(np.array([[1.01e-11]]))[3] == 0
    assert F.lu_pivot_rule(np.array([[0.99e-11]]))[3] == 1


@pytest.mark.parametrize("k,col", [(1, 0), (40, 0), (40, 31), (40, 32), (70, 69), (70, 45)])
def test_restated_lu_reports_the_planted_singular_column(k, col):
    a = np.random.default_rng(col).standard_normal((k, k))
    a[:, col] = a[:, :col] @ np.random.default_rng(1).standard_normal(col) if col else 0.0
    assert F.lu_pivot_rule(a)[3] == col + 1
    if col + 3 < k:  # a second dependent column later on: the first is the one reported
        a[:, col + 3] = a[:, col + 1] - a[:, col + 2]
        assert F.lu_pivot_rule(a)[3] == col + 1
    assert F.lu_pivot_rule(np.zeros((k, k)))[3] == 1


def test_panel_branches_are_counted():
    piv = np.arange(70)
    piv[0], piv[1], piv[2], piv[3], piv[33] = 5, 40, 40, 41, 69
    assert F.panel_branches(piv) == dict(none=65, inside=1, outside=3, repeat=1)


@pytest.mark.parametrize("k", [5, 64, 200])
def test_bounds_hold_for_a_float64_inverse(k):
    a = np.random.default_rng(k).standard_normal((k, k))
    x_ref, kappa = F.inverse_ref(a)
    assert kappa < 1e8
    x_hat = sla.lu_solve(sla.lu_factor(a), np.eye(k))
    env = F.lu_envelope(a, x_hat)
    w = R.Worst()
    w("residual", np.abs(a @ x_hat - np.eye(k)), F.residual_bound(a, x_hat, env))
    w("forward", np.abs(x_hat - x_ref), F.forward_bound(x_ref, env))
    # and they are not vacuous: an inverse with one element off by 1e-7 relative fails
    x_bad = x_hat.copy()
    i, j = np.unravel_index(np.argmax(np.abs(x_hat)), x_hat.shape)
    x_bad[i, j] *= 1.0 + 1e-7
    assert np.any(np.abs(x_bad - x_ref) > F.forward_bound(x_ref, env))
    assert np.any(np.abs(a @ x_bad - np.eye(k)) > F.residual_bound(a, x_bad, env))


@pytest.mark.parametrize("name", ["UFL-20x60", "transport-20x500"])
def test_refresh_reference_agrees_with_the_oracle_at_the_optimum(name):
    lp = load_golden(name)
    o = O.OracleSimplex(lp)
    assert o.dual() == 0
    st = o.status()
    n, m = lp.n, lp.m
    cost = np.concatenate([lp.objective, np.zeros(m)]).astype(np.float64)
    lo = np.maximum(np.concatenate([lp.col_lower, lp.row_lower]).astype(np.float64), -F.INF)
    up = np.minimum(np.concatenate([lp.col_upper, lp.row_upper]).astype(np.float64), F.INF)
    ref = F.refresh_ref(R.ext_matrix(lp), cost, lo, up, st, np.zeros(n + m, dtype=np.uint8), np.flatnonzero(st == R.BASIC),
                        1.0e10)
    scale = 1.0 + np.abs(ref["dj"]).max()
    np.testing.assert_allclose(ref["dj"][:n], o.reduced_cost(), rtol=0, atol=1e-9 * scale)
    np.testing.assert_allclose(ref["pi"], o.row_price(), rtol=0, atol=1e-9 * scale)
    assert not ref["fake"].any()
    x = np.concatenate([o.column_solution(), o.row_activity()])
    np.testing.assert_allclose(ref["sol"], x, rtol=0, atol=1e-8 * (1.0 + np.abs(x).max()))
