"""GPU tests (-m gpu) of the plug-in level of the boundary: the ClpDualRowPivot / ClpFactorization /
ClpMatrixBase calls of one iteration taken one at a time, the packed-vector forms, the FT entry
points and the replaceColumn return codes -- plus direct parity tests of the two hot kernels the
fused iteration runs (price_ldg_kernel and the cooperative row_pass_kernel) against the oracle."""
import numpy as np
import pytest

import clp_b200
from clp_b200 import generators as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def engine(lp, **params):
    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    for k, v in params.items():
        s.setParameter(k, v)
    return s


def test_stepwise_plugin_calls_take_the_pivots_of_the_fused_iteration():
    """pivotRow -> updateColumnTranspose+transposeTimes -> dualColumn -> updateWeights ->
    updatePrimalSolution, called one by one, walk exactly the path Clpb_iterate walks"""
    lp = G.random_sparse_lp(300, 3000, 0.03, 17)
    N = 120
    a = engine(lp, factorizationFrequency=200)
    assert a.startup() == 0
    assert a.iterate(N) == N
    b = engine(lp, factorizationFrequency=200)
    assert b.startup() == 0
    b.saveWeights(5)
    for it in range(N):
        r, seq_out, direction, infeas = b.pivotRow()
        assert r >= 0 and infeas > 0 and direction in (-1, 1)
        nz, rho, row = b.updateColumnTransposeAndPrice()
        assert nz >= 1
        q, theta, alpha_row = b.dualColumnDevice()
        assert q >= 0 and theta >= 0
        alpha_col, rc = b.updateWeights()
        assert rc == 0
        assert abs(alpha_col - alpha_row) <= 1e-7 * (1 + abs(alpha_col))
        assert b.unrollWeights() == 0
        t, change = b.updatePrimalSolution()
        assert t == it + 1 and change >= 0
    for name in ("sol", "dj", "status", "pivotVariable"):
        np.testing.assert_array_equal(a.deviceVector(name), b.deviceVector(name))
    np.testing.assert_array_equal(a.weights(), b.weights())


def _price_variant(m):
    """the price_ldg_kernel instance launch_price (price.cu) selects: rho in shared memory with two 640-thread
    CTAs per SM (<= 112 KiB), with one 1024-thread CTA (<= 224 KiB), or read through L1/L2"""
    b = 8 * m
    return "640x2,smem" if b <= 112 * 1024 else "1024x1,smem" if b <= 224 * 1024 else "640x2,ldg"


@pytest.mark.parametrize("shape", [(400, 6000, 0.02, 3, "640x2,smem"), (1200, 9000, 0.01, 4, "640x2,smem"),
                                   (14337, 4000, 0.01, 5, "1024x1,smem"), (28673, 4000, 0.01, 6, "640x2,ldg"),
                                   (40000, 4000, 0.01, 7, "640x2,ldg")])
def test_price_kernel_row_against_oracle(shape):
    """the tableau row the HOT price kernel (price_ldg_kernel) writes for the BTRAN'd rho, dense and
    sparse rho: alphaRow_j = rho^T a_j for every nonbasic column (1e-12, DESIGN.md section 6).  The three
    launch variants, and (m >= 14 337 at 1 % density) columns longer than the 128 entries of the first pass"""
    m, n, dens, seed, variant = shape
    assert _price_variant(m) == variant
    lp = G.random_sparse_lp(m, n, dens, seed)
    if m > 10000:
        assert np.diff(lp.col_start).mean() > 128
    A = lp.to_scipy()
    s = engine(lp, factorizationFrequency=400)
    assert s.startup() == 0
    for burst in (0, 5, 150):  # all-slack basis (rho = -e_r: sparse), then denser and denser rho
        if burst:
            assert s.iterate(burst) == burst
        r, *_ = s.pivotRow()
        assert r >= 0
        nz, rho, row = s.updateColumnTransposeAndPrice()
        stat = s.deviceVector("status")[:n]
        nonbasic = (stat != 1) & (stat != 5)
        ref = A.T @ rho
        scale = 1.0 + np.abs(A).T @ np.abs(rho)
        assert np.all(np.abs(row - ref)[nonbasic] <= 1e-12 * scale[nonbasic])
        o = O.OracleSimplex(lp)
        np.testing.assert_allclose(row[nonbasic], o.transpose_times(1.0, rho)[nonbasic], rtol=1e-11, atol=1e-12)
        # finish the iteration so that the next burst starts from a consistent state
        q, *_ = s.dualColumnDevice()
        assert q >= 0
        s.updateWeights()
        s.updatePrimalSolution()


def _row_case(rng, nm, kind):
    """adversarial tableau rows for the ratio test: (alphaRow, dj, range, status)"""
    alpha = np.where(rng.uniform(size=nm) < 0.7, rng.standard_normal(nm), 0.0)
    stat = rng.choice(np.array([2, 3], dtype=np.uint8), size=nm)
    dj = np.abs(rng.standard_normal(nm)) * 0.1
    rangeb = np.ones(nm)
    if kind == "ties":            # > 4096 candidates with ratio exactly 0: the short list overflows
        dj[: nm // 2] = 0.0
    elif kind == "boxed-small":   # small ranges: hundreds of break points are passed before the slope is used up
        rangeb[:] = 2e-2
    elif kind == "free":          # free columns: zero-ratio candidates that cannot be flipped
        stat[:25] = 0
        dj[:25] = 0.0
    elif kind == "wide":          # ratios spread over many octaves: the Harris bound leaves the listed window
        dj *= np.exp(rng.uniform(-20, 5, size=nm))
    elif kind == "flip-wide":     # thousands of passed break points with ranges over 12 decades: the flips and
        rangeb = 10.0 ** rng.uniform(-6, 6, size=nm)   # the fixed-point flip column (DESIGN.md section 4)
        alpha = np.where(alpha != 0.0, np.sign(alpha) * rng.uniform(0.5, 1.0, size=nm) / rangeb, 0.0)
        dj = rng.uniform(0.0, 1.0, size=nm) * np.abs(alpha)   # ratios U(0, 1), independent of the range;
        dj[nm - 64:] *= 1e-3                                   # the slacks' come first: slack flips too
    dj = np.where(stat == 2, -dj, dj)
    return alpha, dj, rangeb, stat


@pytest.mark.parametrize("kind", ["plain", "ties", "boxed-small", "free", "wide", "flip-wide"])
@pytest.mark.parametrize("n", [20000, 400000, "E2", "E8"])   # 1 and 4 entries per thread of the cooperative kernel;
def test_dual_column_on_adversarial_rows_against_reference_rule(kind, n):   # 2 and 8 on this card
    """Clpb_dualColumn, i.e. the cooperative row_pass_kernel of the fused iteration, on adversarial rows, against
    the oracle's restatement of the reference's SORTED-PASS dualColumn (ClpSimplexDual.cpp:4331-4658):
    never beyond its break point and within the histogram resolution + Harris slack of it; and identical
    to the bucketed restatement.  The dual update, the bound flips and the flip column the same kernel
    writes against tests/iteration_ref.py."""
    import zlib

    import torch

    import iteration_ref as R

    m = 64
    if isinstance(n, str):  # n+m in the row_pass_kernel<2> / <8> range of this card
        S = torch.cuda.get_device_properties(0).multi_processor_count * 1024
        E = int(n[1:])
        n = int((E - 0.5) * S) - m
        assert -(-(n + m) // S) == E
    rng = np.random.default_rng(zlib.crc32(f"{kind}-{n}".encode()))
    nm = n + m
    alpha, dj, rangeb, stat = _row_case(rng, nm, kind)
    # a model that only provides sizes and bounds 0 <= x <= range (one entry per column)
    start = np.arange(n + 1, dtype=np.int32)
    rows = (np.arange(n) % m).astype(np.int32)
    ub = rangeb.copy()
    ub[stat == 0] = 1e30
    lp = G.LP("rowpass", m, n, start, rows, np.ones(n), np.where(stat[:n] == 0, -1e30, 0.0), ub[:n].copy(),
              np.zeros(n), np.zeros(m), ub[n:].copy())
    s = engine(lp)
    # flip-wide: every candidate uses up |alpha| * range ~ 1 of the slope, so thousands pass before 3 000 is
    # used up, and |alpha| (theta - ratio) exceeds the dual tolerance up to ranges of 1e6
    infeas, sigma = (3.0e3 if kind == "flip-wide" else 3.0), 1
    q, theta = s.dualColumn(alpha, dj, stat, sigma, infeas)
    idx = np.nonzero((alpha != 0) & (np.abs(alpha) > 1e-12))[0]
    rng_arg = np.where(stat == 0, 1e30, rangeb)
    args = (sigma * alpha[idx], dj[idx], rng_arg[idx], stat[idx], infeas)
    kb, theta_b, _ = O.dual_column(*args, bucketed=True)
    k, theta_c, _ = O.dual_column(*args)
    assert (q >= 0) == (kb >= 0) == (k >= 0)
    if q < 0:
        return
    assert q == idx[kb], (q, idx[kb], theta, theta_b)
    assert theta == theta_b
    slack = 2e-6 / max(1e-7, abs(alpha[q]))
    assert theta >= theta_c * (1 - 1e-3) - slack
    if kind not in ("boxed-small", "flip-wide"):
        assert theta <= theta_c * (1 + 1e-9) + slack
    elif kind == "boxed-small":
        # (flip-wide passes thousands of break points too; there the bucketed restatement itself passes up to
        # ~1e-4 relative more slope than the infeasibility, so only its identity with the kernel is checked)
        # the reference gives up after MAXTRY = 100 passes (ClpSimplexDual.cpp:4400) and stops short of the
        # point where the slope is used up; the histogram rule has no pass limit.  What must hold is that
        # the step is still a valid long step: the break points passed do not overshoot the infeasibility
        ab_all = sigma * alpha
        cand = ((stat == 3) & (ab_all > 1e-12)) | ((stat == 2) & (ab_all < -1e-12))
        ratio = np.abs(dj[cand]) / np.abs(alpha[cand])
        passed = (np.abs(alpha[cand]) * rangeb[cand])[ratio < theta * (1 - 2.0 ** -14)].sum()
        assert passed <= infeas * (1 + 1e-9)
    ab = sigma * alpha[q]
    assert (stat[q] == 3 and ab > 0) or (stat[q] == 2 and ab < 0) or stat[q] == 0
    assert abs(alpha[q]) >= 1e-7
    # the dual update, the bound flips and the flip column (rhs3[2m:]) the same kernel wrote
    lower, upper = s.deviceVector("lower"), s.deviceVector("upper")
    fin = R.finalize_row(alpha[:n], -alpha[n:], stat, n)
    np.testing.assert_array_equal(s.deviceVector("alphaRow"), fin)
    du = R.dual_update(fin, dj, stat, lower, upper, np.zeros(nm), np.zeros(nm), sigma, theta, q)
    status1, dj1, sol1 = s.deviceVector("status").astype(np.uint8), s.deviceVector("dj"), s.deviceVector("sol")
    keep = np.ones(nm, dtype=bool)
    keep[du["edge"]] = False
    assert np.all(np.abs(dj1 - du["dj"])[keep] <= du["dj_bound"][keep])
    flips = np.flatnonzero(status1 != stat)
    assert set(flips.tolist()) ^ set(du["flips"].tolist()) <= set(du["edge"].tolist())
    np.testing.assert_array_equal(status1[keep], du["status"][keep])
    np.testing.assert_array_equal(sol1[flips], np.where(status1[flips] == R.AT_UPPER, upper[flips], lower[flips]))
    fl, fl_bound = R.flip_column(R.ext_matrix(lp), flips, status1, lower, upper, 1.0)
    assert np.all(np.abs(s.deviceVector("rhs3")[2 * m:] - fl) <= fl_bound)
    if kind == "flip-wide":
        assert len(flips) >= 1000 and (flips >= n).any()


def test_packed_forms_match_dense():
    lp = G.random_sparse_lp(200, 1500, 0.05, 21)
    s = engine(lp, factorizationFrequency=100)
    assert s.startup() == 0
    assert s.iterate(40) == 40
    rng = np.random.default_rng(5)
    idx = np.sort(rng.choice(lp.m, size=7, replace=False)).astype(np.int32)
    val = rng.standard_normal(7)
    dense = np.zeros(lp.m); dense[idx] = val
    ref = s.updateColumn(dense)
    i2, v2 = s.updateColumnPacked(idx, val)
    keep = np.abs(ref) > 1e-13
    np.testing.assert_array_equal(i2, np.nonzero(keep)[0])
    np.testing.assert_array_equal(v2, ref[keep])
    reft = s.updateColumnTranspose(dense)
    i3, v3 = s.updateColumnTransposePacked(idx, val)
    np.testing.assert_array_equal(v3, reft[np.abs(reft) > 1e-13])
    z = s.transposeTimes(-1.0, dense)
    iz, vz = s.transposeTimesPacked(-1.0, idx, val)
    np.testing.assert_array_equal(iz, np.nonzero(np.abs(z) > 1e-13)[0])
    np.testing.assert_array_equal(vz, z[np.abs(z) > 1e-13])


def test_ft_entry_points_and_replace_column_codes():
    lp = G.random_sparse_lp(120, 900, 0.06, 8)
    o = O.OracleSimplex(lp)
    o.set_option("maximumIterations", 60)
    o.dual()
    st = o.status()
    basis = [j for j in range(lp.n + lp.m) if st[j] == 1]
    s = engine(lp, factorizationFrequency=8)
    pv = s.factorize(basis)
    A = lp.to_scipy().tocsc()
    nonbasic = [j for j in range(lp.n) if st[j] != 1]
    col = np.asarray(A[:, nonbasic[0]].todense()).ravel()
    other = np.random.default_rng(2).standard_normal(lp.m)
    nz, ft = s.updateColumnFT(col)
    ref = s.updateColumn(col)
    np.testing.assert_array_equal(ft, np.where(np.abs(ref) < 1e-13, 0.0, ref))
    assert nz == int((ft != 0).sum())
    nz2, a, b = s.updateTwoColumnsFT(col, other)
    np.testing.assert_array_equal(a, ft)
    np.testing.assert_array_equal(b, s.updateColumn(other))
    # replaceColumn: a good pivot with a matching check value -> 0; a check value 1e-7 off -> 1
    # ("probably ok") or 2 depending on the reference's tolerance ladder; a zero pivot -> 2; then the
    # update buffer fills up -> 5 (maximum pivots)
    r = int(np.argmax(np.abs(ft)))
    assert s.replaceColumnChecked(nonbasic[0], r, ft[r]) == 0
    done = 1
    for j in nonbasic[1:]:
        colj = np.asarray(A[:, j].todense()).ravel()
        f = s.updateColumn(colj)
        rj = int(np.argmax(np.abs(f)))
        zero_rows = np.nonzero(np.abs(f) < 1e-14)[0]
        if done == 1 and len(zero_rows):
            assert s.replaceColumnChecked(j, int(zero_rows[0]), 0.0) == 2     # singular: nothing changed
            assert s.replaceColumnChecked(j, rj, f[rj] * (1 + 1e-3)) == 2     # pivot disagrees with the row
        rc = s.replaceColumnChecked(j, rj, f[rj])
        if done >= 8:
            assert rc == 5
            break
        assert rc == 0
        done += 1
    assert done == 8


@pytest.mark.parametrize("name", ["UFL-20x60", "TSP-MTZ-40", "staircase-480"])
def test_dantzig_row_pivot_reaches_the_same_optimum(name):
    """ClpDualRowDantzig (largest infeasibility) instead of dual steepest edge: another path, same optimum"""
    import os
    from conftest import load_golden

    lp = load_golden(name)
    s = engine(lp, dualRowPivot=1)
    assert s.dual() == 0
    assert abs(s.objectiveValue() - lp.known_objective) <= 1e-6 * (1 + abs(lp.known_objective))
    assert O.kkt_violations(lp, s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution()) == 0
    w = s.weights()
    assert np.all(w == 1.0)          # the steepest-edge weights are left alone in this mode


def test_hot_start_after_bound_changes_matches_a_cold_solve():
    """branching-style re-solves: tighten column bounds, fastDual() keeps the device-resident factors
    (no upload, no refactorization at the start) and must end at the optimum a cold solve of the modified
    LP finds (cross-checked with the CPU oracle)"""
    lp = G.random_sparse_lp(400, 4000, 0.02, 77)
    s = engine(lp)
    assert s.dual() == 0
    x = s.primalColumnSolution()
    frac = np.nonzero((x > 0.05) & (x < 0.95))[0]
    assert len(frac) >= 6
    up = lp.col_upper.copy(); lo = lp.col_lower.copy()
    total_hot = 0
    for round_, j in enumerate(frac[:6]):
        if round_ % 2 == 0:
            up[j] = 0.0          # "down branch"
            s.chgColumnUpper(up)
        else:
            lo[j] = 1.0          # "up branch"
            s.chgColumnLower(lo)
        st = s.fastDual()
        assert s.lastSolveWasHot()
        total_hot += s.numberIterations()
        mod = G.LP(lp.name, lp.m, lp.n, lp.col_start, lp.row_index, lp.element, lo.copy(), up.copy(),
                   lp.objective, lp.row_lower, lp.row_upper)
        o = O.OracleSimplex(mod)
        ost = o.dual()
        assert st == ost
        if st == 0:
            assert abs(s.objectiveValue() - o.objective_value) <= 1e-8 * (1 + abs(o.objective_value))
            assert O.kkt_violations(mod, s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution()) == 0
    cold = engine(mod)
    assert cold.dual() == st
    # the hot re-solves together need far fewer iterations than one cold solve of the last LP
    assert total_hot < cold.numberIterations()
