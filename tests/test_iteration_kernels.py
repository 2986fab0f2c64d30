"""GPU tests (-m gpu) of the kernels of one dual simplex iteration at every launch shape they select, against
the high-precision step reference of tests/iteration_ref.py.

Each kernel picks a launch variant or a loop trip count from the problem shape: the FTRAN / BTRAN GEMVs from the
nucleus size k, the eta kernels from the number of etas t, the row pass from n+m per SM, PRICE from m.  A solve
that only checks its final objective cannot see an error the simplex absorbs (an extra refactorization, another
pivot), so here every output of every call is compared with the reference built from the device state before
that call.  Shapes that must select a variant compute their size from the SM count of the card and assert the
variant they land in."""
import math

import numpy as np
import pytest
import torch

import clp_b200
from clp_b200 import generators as G

import iteration_ref as R

pytestmark = pytest.mark.gpu

U = R.U


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def row_pass_entries(nm):
    """entries per thread of the cooperative row pass: row_pass_kernel<E> (rowpass.cu launch_row_pass)"""
    need = -(-nm // (sms() * 1024))
    return next(e for e in (1, 2, 4, 8) if need <= e)


def engine(lp, **params):
    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    for k, v in params.items():
        s.setParameter(k, v)
    return s


def conditioned_lp(m, n, k, seed, off=4, permute_homes=False):
    """An LP whose bases stay well conditioned.  Every column has one dominant entry of magnitude 10..20 on its
    home row and `off` entries U(-1, 1) on other rows, so a basis whose columns have distinct home rows is
    column-diagonally dominant (||B^-1||_1 <= 1).  Structurals 0..k-1 have home rows 0..k-1, the others a random
    home row.  All bounds are finite (columns [0, 1..4], rows a narrow range around a random point), so the
    working bounds are the true bounds.  Returns (lp, status) with structurals 0..k-1 and the slacks of rows
    k..m-1 basic: a basis with a nucleus of exactly k."""
    rng = np.random.default_rng(seed)
    home = np.concatenate([np.arange(k), rng.integers(0, m, size=n - k)]) if m > 1 else np.zeros(n, dtype=np.int64)
    if permute_homes:
        home[:k] = np.random.default_rng([seed, k]).permutation(k)
    rows = np.empty((n, off + 1), dtype=np.int64)
    vals = np.empty((n, off + 1))
    rows[:, 0] = home
    vals[:, 0] = rng.uniform(10.0, 20.0, size=n) * rng.choice([-1.0, 1.0], size=n)
    rows[:, 1:] = (home[:, None] + rng.integers(1, m, size=(n, off))) % m
    vals[:, 1:] = rng.uniform(-1.0, 1.0, size=(n, off))
    import scipy.sparse as sp

    A = sp.csc_matrix((vals.ravel(), (rows.ravel(), np.repeat(np.arange(n), off + 1))), shape=(m, n))
    A.sum_duplicates()
    A.sort_indices()
    x0 = rng.uniform(0.0, 1.0, size=n)
    center = A @ x0 + rng.uniform(-3.0, 3.0, size=m)
    lp = G.LP(f"conditioned-{m}x{n}-k{k}", m, n, A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data,
              np.zeros(n), rng.uniform(1.0, 4.0, size=n), rng.standard_normal(n), center - 0.05, center + 0.05)
    status = np.full(n + m, 3, dtype=np.uint8)
    status[:k] = 1
    status[n + k:] = 1
    return lp, status


def pivoting_lp(m, n, k, seed, off=4):
    """conditioned_lp with the home rows of the k nucleus columns a random permutation of the nucleus rows: the
    basis is as well conditioned, but the dominant entry of a nucleus column is off the diagonal, so the partial
    pivoting of the refactorization interchanges in every panel."""
    return conditioned_lp(m, n, k, seed, off, permute_homes=True)


Worst = R.Worst


def check_solve(worst, name, x, ref, kappa):
    worst(name, np.abs(x - ref).max(initial=0.0), R.solve_bound(ref, kappa))


# ------------------------------------------------------------------ FTRAN / BTRAN entry points
K_SWEEP = [0, 1, 7, 9, 1023, 1024, 1025, 4095, 4096, 4097]
T_SWEEP = [0, 1, 255, 256, 257, 1023, 1024, 1025, 2047, 2048]


@pytest.mark.parametrize("k", K_SWEEP)
def test_ftran_btran_entry_points_at_every_nucleus_and_eta_count(k):
    """updateColumn (gemv_rows_kernel<1,1,8>: a second trip of its j loop for k > 4096), updateTwoColumnsFT
    (<2,2,2>: k > 1024) and updateColumnTranspose (<1,1,8> on N^-T), each after t = 0 ... 2048 product-form
    updates (pfi_apply_warp_kernel: t > 256; pfi_mu_kernel, eta_rowvec_kernel: t > 1024)"""
    m, n = k + 300, k + 2400
    lp, status = conditioned_lp(m, n, k, seed=1000 + k)
    aext = R.ext_matrix(lp)
    s = engine(lp, factorizationFrequency=2048)
    rc, pv = s.factorize(np.flatnonzero(status == 1))
    assert rc == 0
    assert s.nucleusSize() == k
    pv = pv.astype(np.int64)
    rng = np.random.default_rng(k)
    worst = Worst()
    entering, t = iter(range(k, n)), 0
    for target in T_SWEEP:
        while t < target:
            q = next(entering)
            f = s.updateColumn(aext[:, q].toarray().ravel())
            r = int(np.argmax(np.abs(f)))
            assert s.replaceColumn(q, r) == 0
            pv[r] = q
            t += 1
        ref = R.Basis(aext, pv)
        kappa = ref.cond1()
        b, c = rng.standard_normal(m), rng.standard_normal(m)
        xb, xc = ref.ftran(b), ref.ftran(c)
        check_solve(worst, "updateColumn", s.updateColumn(b), xb, kappa)
        nz, y1, y2 = s.updateTwoColumnsFT(b, c)
        check_solve(worst, "updateTwoColumnsFT", y2, xc, kappa)
        if t < 2048:  # the FT column keeps its spike for replaceColumn: no room for one more at t = tmax
            check_solve(worst, "updateTwoColumnsFT", y1, xb, kappa)
        else:
            assert nz < 0
        check_solve(worst, "updateColumnTranspose", s.updateColumnTranspose(c), ref.btran(c), kappa)
        assert s.nucleusSize() == k
    worst.report(f"k={k}")


def test_replace_column_with_more_than_16384_entries():
    """replaceColumn scatters the entering column from the device copy of A: all 20 000 entries of it, not the
    first 16 384, must reach the eta, or every later FTRAN / BTRAN is wrong"""
    m = 20000
    rng = np.random.default_rng(7)
    dense = rng.uniform(-1e-3, 1e-3, size=m)
    dense[100] = 20.0
    start = np.array([0, m, m + 1, m + 2], dtype=np.int32)
    index = np.concatenate([np.arange(m), [5, 6]]).astype(np.int32)
    value = np.concatenate([dense, [1.0, 1.0]])
    lp = G.LP("long-column", m, 3, start, index, value, np.zeros(3), np.ones(3), np.zeros(3), np.full(m, -1.0),
              np.ones(m))
    aext = R.ext_matrix(lp)
    s = engine(lp)
    pv = np.arange(3, 3 + m)
    rc, pvd = s.factorize(pv)
    assert rc == 0 and np.array_equal(pvd, pv)
    f = s.updateColumn(dense)
    r = int(np.argmax(np.abs(f)))
    assert r == 100
    assert s.replaceColumn(0, r) == 0
    pv[r] = 0
    ref = R.Basis(aext, pv)
    kappa = ref.cond1()
    worst = Worst()
    b = rng.standard_normal(m)
    check_solve(worst, "updateColumn", s.updateColumn(b), ref.ftran(b), kappa)
    check_solve(worst, "updateColumnTranspose", s.updateColumnTranspose(b), ref.btran(b), kappa)
    worst.report("long column")


# ------------------------------------------------------------------ checked stepwise iterations
def checked_iteration(s, lp, aext, amax, worst):
    """pivotRow -> updateColumnTransposeAndPrice -> dualColumnDevice -> updateWeights -> updatePrimalSolution,
    every output and the device state after every call against the reference built from the state before it"""
    n, m = lp.n, lp.m
    dv = lambda name: s.deviceVector(name)
    sol, dj, cost = dv("sol"), dv("dj"), dv("cost")
    lower, upper = dv("lower"), dv("upper")
    status = dv("status").astype(np.uint8)
    pv = dv("pivotVariable").astype(np.int64)
    w = s.weights()
    basis = R.Basis(aext, pv)
    kappa = basis.cond1()

    # CHUZR
    r, seq_out, sigma, infeas = s.pivotRow()
    _, accepted = R.chuzr(sol, lower, upper, w, pv)
    assert r in accepted, (r, accepted)
    assert seq_out == pv[r]
    assert (sigma, infeas) == R.pivot_row_scalars(sol, lower, upper, seq_out)

    # BTRAN + PRICE
    _, rho, raw = s.updateColumnTransposeAndPrice()
    e = np.zeros(m)
    e[r] = 1.0
    check_solve(worst, "BTRAN rho", rho, basis.btran(e), kappa)
    exact, gbound = R.price(aext, rho, n)
    nb = (status[:n] != R.BASIC) & (status[:n] != R.FIXED)
    worst("PRICE alphaRow", np.abs(raw - exact)[nb], gbound[nb])
    assert np.all(raw[~nb] == 0.0)

    # CHUZC, dual update, bound flips, the row pass's FTRAN right-hand sides
    q, theta, alpha_q = s.dualColumnDevice()
    alpha = R.finalize_row(raw, rho, status, n)
    np.testing.assert_array_equal(dv("alphaRow"), alpha)
    q_ref, theta_ref = R.chuzc(alpha, dj, status, lower, upper, sigma, infeas)
    assert (q, theta) == (q_ref, theta_ref)
    assert alpha_q == alpha[q]
    du = R.dual_update(alpha, dj, status, lower, upper, sol, cost, sigma, theta, q)
    sol1, dj1, cost1 = dv("sol"), dv("dj"), dv("cost")
    status1 = dv("status").astype(np.uint8)
    keep = np.ones(n + m, dtype=bool)
    keep[du["edge"]] = False
    worst("dual update dj", np.abs(dj1 - du["dj"])[keep], du["dj_bound"][keep])
    worst("cost shift", np.abs(cost1 - du["cost"])[keep], du["dj_bound"][keep])
    flips = np.flatnonzero(status1 != status)
    assert set(flips.tolist()) ^ set(du["flips"].tolist()) <= set(du["edge"].tolist())
    np.testing.assert_array_equal(status1[keep], du["status"][keep])
    np.testing.assert_array_equal(sol1[flips], np.where(status1[flips] == R.AT_UPPER, upper[flips], lower[flips]))
    np.testing.assert_array_equal(np.delete(sol1, flips), np.delete(sol, flips))
    rhs3 = dv("rhs3")
    np.testing.assert_array_equal(rhs3[:m], aext[:, q].toarray().ravel())
    np.testing.assert_array_equal(rhs3[m:2 * m], rho)
    fl, fl_bound = R.flip_column(aext, flips, status1, lower, upper, amax)
    worst("flip column", np.abs(rhs3[2 * m:] - fl), fl_bound)

    # the three FTRANs
    alpha_col, rc = s.updateWeights()
    assert rc == 0
    f3 = dv("rhs3")
    for c, name in enumerate(("FTRAN alpha_q", "FTRAN tau", "FTRAN flip column")):
        check_solve(worst, name, f3[c * m:(c + 1) * m], basis.ftran(rhs3[c * m:(c + 1) * m]), kappa)
    assert alpha_col == f3[r]

    # primal update, DSE recurrence, housekeeping
    s.updatePrimalSolution()
    ac, tau, ffl = f3[:m], f3[m:2 * m], f3[2 * m:]
    theta_p = R.primal_step(sol1, lower, upper, seq_out, sigma, ac, ffl, len(flips), r)
    bound_out = lower[seq_out] if sigma < 0 else upper[seq_out]
    sol_ref, sb = R.primal_update(sol1, pv, ac, ffl, len(flips), theta_p, r, q, seq_out, bound_out)
    worst("primal update", np.abs(dv("sol") - sol_ref), sb)
    w_ref, wb = R.dse_update(w, ac, tau, r, math.fsum(rho * rho), m)
    worst("DSE weights", np.abs(s.weights() - w_ref), wb)
    st_ref = status1.copy()
    st_ref[q] = R.BASIC
    st_ref[seq_out] = R.FIXED if lower[seq_out] == upper[seq_out] else (R.AT_LOWER if sigma < 0 else R.AT_UPPER)
    np.testing.assert_array_equal(dv("status").astype(np.uint8), st_ref)
    pv_ref = pv.copy()
    pv_ref[r] = q
    np.testing.assert_array_equal(dv("pivotVariable").astype(np.int64), pv_ref)
    dj2 = dv("dj")
    assert dj2[q] == 0.0 and dj2[seq_out] == -sigma * theta
    return len(flips)


def _stepwise_cases():
    # (id, m, n, k, off, etas before the checked iterations, row pass E or None)
    return [
        ("E1", 300, 3000, 100, 4, 0, 1),
        ("E2", 300, "1.5S", 100, 2, 0, 2),
        ("E4", 300, "3S", 100, 2, 0, 4),
        ("E8", 300, "4.4S", 100, 2, 0, 8),
        ("k1030", 1500, 5000, 1030, 4, 0, None),
        ("k4100", 4400, 9000, 4100, 4, 0, None),
        ("t257", 1500, 6000, 300, 4, 257, None),
        ("t1025", 3000, 9000, 600, 4, 1025, None),
    ]


@pytest.mark.parametrize("case", _stepwise_cases(), ids=lambda c: c[0])
def test_checked_stepwise_iterations(case):
    name, m, n, k, off, t0, E = case
    if isinstance(n, str):  # n+m just inside the row pass variant, from this card's SM count
        n = int(float(n[:-1]) * sms() * 1024) - m
    if E is not None:
        assert row_pass_entries(n + m) == E
    lp, status = conditioned_lp(m, n, k, seed=20261016)
    aext = R.ext_matrix(lp)
    amax = max(1.0, float(np.abs(lp.element).max()))
    s = engine(lp, factorizationFrequency=2048)
    s.copyinStatus(status)
    assert s.startup() == 0
    assert s.nucleusSize() == k
    if t0:
        assert s.iterate(t0) == t0
        assert s.nucleusSize() == k
    worst = Worst()
    nflips = sum(checked_iteration(s, lp, aext, amax, worst) for _ in range(3))
    worst.report(f"{name} flips={nflips}")
