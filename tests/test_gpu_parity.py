"""GPU parity tests (-m gpu): the CUDA path, called through the C ABI, against the CPU oracle
on the same seeded inputs and against the committed golden fixtures."""
import json
import os

import numpy as np
import pytest

from conftest import ROOT, load_golden

import clp_b200
from clp_b200 import generators as G
from oracle import oracle as O

pytestmark = pytest.mark.gpu

MANIFEST = json.load(open(os.path.join(ROOT, "tests", "golden", "manifest.json")))
ALL = sorted(MANIFEST)


def engine(lp, **params):
    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    for k, v in params.items():
        s.setParameter(k, v)
    return s


def kkt(lp, s):
    return O.kkt_violations(lp, s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution())


# ------------------------------------------------------------------ matrix interface
def test_transpose_times_and_times():
    lp = G.random_sparse_lp(400, 5000, 0.02, 11)
    rng = np.random.default_rng(1)
    s, o = engine(lp), O.OracleSimplex(lp)
    pi = rng.standard_normal(lp.m)
    z_gpu, z_cpu = s.transposeTimes(-1.0, pi), o.transpose_times(-1.0, pi)
    np.testing.assert_allclose(z_gpu, z_cpu, rtol=1e-12, atol=1e-12)
    x = rng.standard_normal(lp.n)
    y_gpu, y_cpu = s.times(1.0, x), o.times(1.0, x)
    np.testing.assert_allclose(y_gpu, y_cpu, rtol=1e-11, atol=1e-11)


# ------------------------------------------------------------------ factorization interface
def _basis_from_oracle(lp, iters):
    o = O.OracleSimplex(lp)
    o.set_option("maximumIterations", iters)
    o.dual()
    st = o.status()
    return [j for j in range(lp.n + lp.m) if st[j] == 1]


@pytest.mark.parametrize("shape", [(60, 300, 0.1, 40), (300, 2000, 0.03, 250), (1000, 6000, 0.01, 900)])
def test_factorize_ftran_btran(shape):
    m, n, dens, iters = shape
    lp = G.random_sparse_lp(m, n, dens, 5)
    basis = _basis_from_oracle(lp, iters)
    assert len(basis) == lp.m
    s, o = engine(lp), O.OracleSimplex(lp)
    rc_g, pv_g = s.factorize(basis)
    rc_c, pv_c = o.factorize(basis)
    assert rc_g == 0 and rc_c == 0
    assert sorted(pv_g) == sorted(pv_c) == sorted(basis)
    # slack of row i must pivot on row i in both
    for p, seq in enumerate(pv_g):
        if seq >= lp.n:
            assert seq - lp.n == p
    rng = np.random.default_rng(2)
    for _ in range(3):
        b = rng.standard_normal(lp.m)
        xg, xc = s.updateColumn(b), o.ftran(b)
        byvar_g = {int(v): xg[p] for p, v in enumerate(pv_g)}
        byvar_c = {int(v): xc[p] for p, v in enumerate(pv_c)}
        dg = np.array([byvar_g[v] for v in basis]); dc = np.array([byvar_c[v] for v in basis])
        np.testing.assert_allclose(dg, dc, rtol=1e-8, atol=1e-8 * (1 + np.abs(dc).max()))
        cvar = rng.standard_normal(lp.n + lp.m)
        yg = s.updateColumnTranspose(np.array([cvar[v] for v in pv_g]))
        yc = o.btran(np.array([cvar[v] for v in pv_c]))
        np.testing.assert_allclose(yg, yc, rtol=1e-8, atol=1e-8 * (1 + np.abs(yc).max()))


def test_replace_column_sequence():
    """rank-one basis updates (product form on the GPU, Forrest-Tomlin in the oracle) give the
    same FTRAN/BTRAN results, and the same as a fresh factorization of the final basis."""
    lp = G.random_sparse_lp(200, 1500, 0.04, 9)
    basis = _basis_from_oracle(lp, 120)
    s, o = engine(lp, factorizationFrequency=100), O.OracleSimplex(lp)
    rc, pv_g = s.factorize(basis); assert rc == 0
    rc, pv_c = o.factorize(basis); assert rc == 0
    pv_g, pv_c = list(pv_g), list(pv_c)
    rng = np.random.default_rng(3)
    nonbasic = [j for j in range(lp.n) if j not in set(basis)]
    rng.shuffle(nonbasic)
    done = 0
    for q in nonbasic[:60]:
        col = np.zeros(lp.m)
        sl = slice(lp.col_start[q], lp.col_start[q + 1])
        col[lp.row_index[sl]] = lp.element[sl]
        a = o.ftran(col)
        r_c = int(np.argmax(np.abs(a)))
        if abs(a[r_c]) < 1e-3:
            continue
        leaving = pv_c[r_c]
        r_g = pv_g.index(leaving)
        assert o.replace_column(q, r_c) in (0, 1)
        assert s.replaceColumn(q, r_g) == 0
        pv_c[r_c] = q; pv_g[r_g] = q
        done += 1
        if done % 10 == 0:
            b = rng.standard_normal(lp.m)
            xg, xc = s.updateColumn(b), o.ftran(b)
            dg = {v: xg[p] for p, v in enumerate(pv_g)}; dc = {v: xc[p] for p, v in enumerate(pv_c)}
            for v in dg:
                assert abs(dg[v] - dc[v]) <= 1e-7 * (1 + abs(dc[v])), (done, v, dg[v], dc[v])
            cvar = rng.standard_normal(lp.n + lp.m)
            yg = s.updateColumnTranspose(np.array([cvar[v] for v in pv_g]))
            yc = o.btran(np.array([cvar[v] for v in pv_c]))
            np.testing.assert_allclose(yg, yc, rtol=1e-7, atol=1e-7 * (1 + np.abs(yc).max()))
    assert done >= 30


def test_unit_test_3x5_primals():
    """src/unitTest.cpp:1415-1482 : factorize basis {c0,c1,c4}, getSolution -> colsol"""
    lp = load_golden("unitTest-3x5")
    s = engine(lp)
    st = np.full(lp.n + lp.m, 3, dtype=np.uint8)
    st[[0, 1, 4]] = 1
    s.copyinStatus(st)
    assert s.startup() == 0
    sol = s.deviceVector("sol")
    np.testing.assert_allclose(sol[:5], [20.0 / 7.0, 3.0, 0.0, 0.0, 23.0 / 7.0], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("k", [1, 5, 31, 33, 100, 257, 700, 1500])
def test_dense_invert(k):
    """the dense LU + inverse of the refactorization (cooperative multi-CTA panel, TRSM, DGEMM)"""
    rng = np.random.default_rng(k)
    a = rng.standard_normal((k, k)) + np.diag(rng.uniform(0.5, 1.5, size=k) * np.sqrt(k) * rng.choice([-1, 1], size=k))
    # make partial pivoting matter: shuffle rows
    a = a[rng.permutation(k)]
    info, x = clp_b200.denseInvert(a)
    assert info == 0
    ref = np.linalg.inv(a)
    np.testing.assert_allclose(x, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())
    res = np.abs(a @ x - np.eye(k)).max()
    assert res < 1e-10 * k


def test_dense_invert_singular():
    rng = np.random.default_rng(0)
    a = rng.standard_normal((64, 64))
    a[:, 40] = a[:, 3] * 2.0 - a[:, 7]
    info, _ = clp_b200.denseInvert(a)
    assert info > 0


# ------------------------------------------------------------------ ratio test
def test_dual_column_against_oracle():
    lp = G.random_sparse_lp(200, 3000, 0.03, 21)
    rng = np.random.default_rng(4)
    s = engine(lp)
    nm = lp.n + lp.m
    for trial in range(6):
        alpha = np.where(rng.uniform(size=nm) < 0.6, rng.standard_normal(nm), 0.0)
        stat = rng.choice([2, 3], size=nm).astype(np.uint8)
        stat[rng.choice(nm, size=lp.m, replace=False)] = 1
        dj = np.abs(rng.standard_normal(nm)) * 0.1 * rng.choice([0.0, 1.0], size=nm, p=[0.1, 0.9])
        dj = np.where(stat == 2, -dj, dj)
        infeas = float(rng.uniform(0.5, 20.0))
        sigma = int(rng.choice([-1, 1]))
        q, theta = s.dualColumn(alpha, dj, stat, sigma, infeas)
        lo = np.concatenate([lp.col_lower, lp.row_lower]); up = np.concatenate([lp.col_upper, lp.row_upper])
        idx = np.nonzero((alpha != 0) & (stat != 1) & (np.abs(alpha) > 1e-12))[0]
        args = (sigma * alpha[idx], dj[idx], (up - lo)[idx], stat[idx], infeas)
        # (1) identical to the oracle's restatement of the two-level histogram rule
        kb, theta_b, _ = O.dual_column(*args, bucketed=True)
        assert q == idx[kb], (q, idx[kb])
        assert theta == theta_b
        # (2) against the sorted-pass BFRT of the reference: never beyond its break point, and
        # within the histogram resolution (2^-16 relative) + Harris slack of it
        k, theta_c, _ = O.dual_column(*args)
        assert q >= 0 and k >= 0
        assert theta <= theta_c * (1 + 1e-9) + 2e-6 / max(1e-7, abs(alpha[q]))
        assert theta >= theta_c * (1 - 1e-3) - 2e-6 / max(1e-7, abs(alpha[q]))
        ab = sigma * alpha[q]
        assert (stat[q] == 3 and ab > 0) or (stat[q] == 2 and ab < 0)
        assert abs(alpha[q]) >= 1e-7


def test_pivot_sequence_follows_oracle():
    """the first iterations take exactly the pivots of the CPU restatement run with the same
    (histogram) ratio test: same leaving and entering variables, same step lengths"""
    import os, re, tempfile

    lp = G.random_sparse_lp(1500, 15000, 0.01, 99)
    N = 250

    def run(kind):
        tf = tempfile.TemporaryFile(mode="w+b")
        old = os.dup(2); os.dup2(tf.fileno(), 2)
        try:
            if kind == "gpu":
                s = engine(lp, logLevel=3, maximumIterations=N)
                s.dual()
            else:
                o = O.OracleSimplex(lp)
                for k, v in (("logLevel", 3), ("bucketedRatioTest", 1), ("maximumIterations", N)):
                    o.set_option(k, v)
                o.dual()
        finally:
            os.dup2(old, 2); os.close(old)
        tf.seek(0)
        return [l for l in tf.read().decode(errors="ignore").splitlines() if l.startswith("TRACE")]

    pat = re.compile(r"TRACE (\d+) out=(\d+) in=(\d+) sigma=(-?\d+) thetaD=(\S+) thetaP=(\S+)")
    g, c = run("gpu"), run("cpu")
    assert len(g) == N and len(c) == N
    for a, b in zip(g, c):
        ma, mb = pat.match(a), pat.match(b)
        assert ma.group(2, 3, 4) == mb.group(2, 3, 4), (a, b)
        ta, tb = float(ma.group(5)), float(mb.group(5))
        assert abs(ta - tb) <= 1e-6 * (1e-9 + abs(tb)) + 1e-12, (a, b)


# ------------------------------------------------------------------ DSE weights
def test_dse_weights_after_iterations():
    lp = G.random_sparse_lp(150, 1200, 0.05, 13)
    s = engine(lp, factorizationFrequency=100)
    assert s.startup() == 0
    done = s.iterate(60)
    assert done == 60
    w = s.weights()
    # brute force ||B^-T e_p||^2 through the engine's own BTRAN (etas included)
    for p in np.random.default_rng(0).choice(lp.m, size=25, replace=False):
        e = np.zeros(lp.m); e[p] = 1.0
        rho = s.updateColumnTranspose(e)
        true = float(rho @ rho)
        assert abs(w[p] - true) <= 1e-6 * (1 + true), (p, w[p], true)


# ------------------------------------------------------------------ full solves
@pytest.mark.parametrize("name", ALL)
def test_golden_fixture_solves(name):
    lp = load_golden(name)
    s = engine(lp)
    st = s.dual()
    assert st == lp.expect_status, (name, st)
    if st == 0:
        tol = 1e-4 if MANIFEST[name]["objective_source"] == "reference" else 1e-8
        assert abs(s.objectiveValue() - lp.known_objective) <= tol * (1 + abs(lp.known_objective))
        # identical to the CPU oracle to the reference's CoinRelFltEq(1e-8)
        ref = MANIFEST[name]["oracle_objective"]
        assert abs(s.objectiveValue() - ref) <= 1e-8 * (1 + abs(ref))
        assert kkt(lp, s) == 0
        stat = s.statusArray()
        assert int((stat == 1).sum()) == lp.m


@pytest.mark.parametrize("shape", [(300, 3000, 0.02, 7), (1000, 10000, 0.01, 20260923)])
def test_planted_random_lp(shape):
    m, n, dens, seed = shape
    lp = G.random_sparse_lp(m, n, dens, seed)
    s = engine(lp)
    assert s.dual() == 0
    assert abs(s.objectiveValue() - lp.known_objective) <= 1e-8 * (1 + abs(lp.known_objective))
    assert kkt(lp, s) == 0
    o = O.OracleSimplex(lp)
    assert o.dual() == 0
    assert abs(s.objectiveValue() - o.objective_value) <= 1e-8 * (1 + abs(o.objective_value))


@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("name", ["TSP-MTZ-40", "UFL-30x100", "modified_afiro", "staircase-480", "SetCover-50x200",
                                  "NQueens-20", "hello"])
def test_scaled_solve_matches_unscaled(name, mode):
    """ClpModel::scaling(mode): the scaled problem is solved on the device, the answer comes back
    in the caller's units: same optimum (CoinRelFltEq 1e-8 of the reference's tests), KKT audit
    on the UNSCALED data."""
    lp = load_golden(name)
    s = engine(lp)
    s.scaling(mode)
    assert s.dual() == 0
    assert abs(s.objectiveValue() - lp.known_objective) <= 1e-7 * (1 + abs(lp.known_objective))
    ref = MANIFEST[name]["oracle_objective"]
    assert abs(s.objectiveValue() - ref) <= 1e-7 * (1 + abs(ref))
    assert kkt(lp, s) == 0
    assert int((s.statusArray() == 1).sum()) == lp.m


def test_scaled_planted_random_lp():
    lp = G.random_sparse_lp(500, 5000, 0.01, 77)
    lp.element = lp.element * np.repeat(10.0 ** np.random.default_rng(5).uniform(-3, 3, size=lp.n), np.diff(lp.col_start))
    o = O.OracleSimplex(lp)
    assert o.dual() == 0
    for mode in (0, 3):
        s = engine(lp)
        s.scaling(mode)
        assert s.dual() == 0, mode
        assert abs(s.objectiveValue() - o.objective_value) <= 1e-7 * (1 + abs(o.objective_value))
        assert kkt(lp, s) == 0


@pytest.mark.parametrize("name", ["transport-10x200", "transport-20x500", "NQueens-50", "SetPart-40x200",
                                  "UFL-30x100", "staircase-480", "Infeasible-50"])
def test_perturbed_solve_reaches_the_true_optimum(name):
    """ClpSimplex::setPerturbation(50): costs are perturbed before the first iteration
    (ClpSimplexDual::perturb), removed at the first optimal basis, and the dual simplex finishes on
    the true costs: same status, same optimum, KKT on the true data."""
    lp = load_golden(name)
    s = engine(lp)
    s.setPerturbation(50)
    st = s.dual()
    assert st == lp.expect_status
    if st == 0:
        tol = 1e-4 if MANIFEST[name]["objective_source"] == "reference" else 1e-8
        assert abs(s.objectiveValue() - lp.known_objective) <= tol * (1 + abs(lp.known_objective))
        ref = MANIFEST[name]["oracle_objective"]
        assert abs(s.objectiveValue() - ref) <= 1e-8 * (1 + abs(ref))
        assert kkt(lp, s) == 0
        assert int((s.statusArray() == 1).sum()) == lp.m


@pytest.mark.parametrize("name", ["TSP-MTZ-40", "SetCover-100x500", "transport-20x500"])
def test_graph_replay_matches_direct_launches(name):
    """The captured iteration graph against direct kernel launches: the same kernels with the same
    arguments, so the solves must be identical (iterations and objective bit for bit)."""
    lp = load_golden(name)
    res = []
    for params in ({}, {"useGraph": 0}):
        s = engine(lp, **params)
        assert s.dual() == 0, params
        res.append((s.numberIterations(), s.objectiveValue()))
    assert res[0] == res[1], res


def test_long_row_multi_entry_row_pass_with_and_without_graph():
    """n+m above 132*1024 (one 1024-thread CTA per SM of an H100): every thread of the cooperative row kernel owns two entries of the
    tableau row (row_pass_kernel<2>); same optimum as the planted solution, with and without graph
    replay."""
    lp = G.random_sparse_lp(500, 170000, 0.02, 31)
    s = engine(lp)
    assert s.dual() == 0
    assert abs(s.objectiveValue() - lp.known_objective) <= 1e-8 * (1 + abs(lp.known_objective))
    assert kkt(lp, s) == 0
    s2 = engine(lp, useGraph=0)
    assert s2.dual() == 0
    assert abs(s2.objectiveValue() - s.objectiveValue()) <= 1e-9 * (1 + abs(s.objectiveValue()))


def test_batch_size_does_not_change_result():
    lp = load_golden("TSP-MTZ-20")
    objs = []
    for b in (1, 7, 32):
        s = engine(lp, batch=b)
        assert s.dual() == 0
        objs.append((s.objectiveValue(), s.numberIterations()))
    assert objs[0] == objs[1] == objs[2]


def test_warm_start_from_optimal_status():
    lp = load_golden("UFL-10x30")
    s = engine(lp)
    assert s.dual() == 0
    st = s.statusArray()
    s2 = engine(lp)
    s2.copyinStatus(st)
    assert s2.dual() == 0
    assert s2.numberIterations() <= 2
    assert abs(s2.objectiveValue() - s.objectiveValue()) <= 1e-9 * (1 + abs(s.objectiveValue()))
