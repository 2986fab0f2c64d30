"""GPU tests (-m gpu) of everything Engine::refresh() runs once per update cycle, against the high-precision
reference of tests/refactor_ref.py: the dense LU and inverse of the nucleus (factor.cu) at the edges of every
launch shape and every branch of its pivot bookkeeping, Engine::refactor with a nucleus that really
interchanges, the repair of singular bases, and the refresh kernels of update.cu.

A wrong refactorization or refresh rarely changes the optimum a solve reaches: refresh() answers the drift with
a back-track and shorter cycles, a wrong dual feasible bound costs pivots.  So every output is compared per call,
and every check reports "worst error, bound, fraction of it" (pytest -s)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import clp_b200
from clp_b200 import generators as G

import iteration_ref as R
import refactor_ref as F
from test_iteration_kernels import conditioned_lp, engine, pivoting_lp, sms

pytestmark = pytest.mark.gpu

U = R.U
NB = F.NB
CLUSTER_ROWS = 16 * 640          # kPanelCluster x kPanelMaxRowsPerCta: taller panels run lu_panel_coop_kernel


# ------------------------------------------------------------------ matrix families (all seeded)
def gaussian(k, seed=0):
    return np.random.default_rng([k, seed]).standard_normal((k, k))


def planted(k, piv, seed=0):
    """A matrix whose LU takes exactly the interchanges j <-> piv[j]: a dominant diagonal (1..2, random sign)
    plus noise of 1e-3, with the interchanges undone from the last to the first."""
    rng = np.random.default_rng([k, seed, 1])
    a = 1.0e-3 * rng.standard_normal((k, k))
    a[np.arange(k), np.arange(k)] = rng.uniform(1.0, 2.0, size=k) * rng.choice([-1.0, 1.0], size=k)
    for j in range(k - 1, -1, -1):
        if piv[j] != j:
            a[[j, piv[j]]] = a[[piv[j], j]]
    return a


def pivot_sequence(k, kind, seed=0):
    rng = np.random.default_rng([k, seed, 2])
    piv = np.arange(k)
    for j0 in range(0, k, NB):
        j1 = min(j0 + NB, k)
        below = k - j1
        for j in range(j0, j1):
            if kind == "inside":
                piv[j] = rng.integers(j, j1)
            elif kind == "outside" and below >= j1 - j0:
                piv[j] = j1 + (j - j0) * (below // (j1 - j0))       # distinct rows below the panel
            elif kind == "repeat" and below >= 1:
                piv[j] = j1 + ((j - j0) // 2) % min(below, 5)       # every chosen outside row more than once
    return piv


def tied(k, seed=0):
    """integer-valued columns whose largest magnitude, 8, occurs on two rows (ties go to the smallest row)"""
    rng = np.random.default_rng([k, seed, 3])
    a = rng.integers(-2, 3, size=(k, k)).astype(np.float64)
    a[rng.permutation(k), np.arange(k)] = 8.0
    a[rng.permutation(k), np.arange(k)] = -8.0
    return a


def low_bits(k, seed=0):
    """the two largest entries of every column differ only inside the 20 bits the pivot keys drop"""
    rng = np.random.default_rng([k, seed, 4])
    a = rng.uniform(-1.0, 1.0, size=(k, k))
    perm = rng.permutation(k)
    for j in range(k):
        big = 4.0 + rng.random()
        a[perm[j], j] = big
        a[perm[(j + 1) % k], j] = -big * (1.0 + 2.0 ** -40) if k > 1 else big
    return a


def row_scaled(k, seed=0):
    rng = np.random.default_rng([k, seed, 5])
    return gaussian(k, seed) * (10.0 ** rng.uniform(-8.0, 8.0, size=k))[:, None]


def nucleus_like(k, seed=0):
    """about 1 % dense plus a permuted diagonal: whole CTAs see only zeros in a column"""
    rng = np.random.default_rng([k, seed, 6])
    a = sp.random(k, k, density=0.01, random_state=rng, data_rvs=lambda s: rng.uniform(-1.0, 1.0, size=s)).toarray()
    a[rng.permutation(k), np.arange(k)] += rng.uniform(2.0, 4.0, size=k) * rng.choice([-1.0, 1.0], size=k)
    return a


# ------------------------------------------------------------------ checks
def check_inverse(worst, a, tag, expect_piv=None):
    """denseInvert(a) against the bounds of refactor_ref: elementwise residual and forward error in full up to
    k = 2049 / 513, residuals from both sides on 64 dense columns above"""
    k = a.shape[0]
    info, x = clp_b200.denseInvert(a)
    piv, L, Um, info_ref = F.lu_pivot_rule(a)
    assert info == info_ref == 0, (tag, info, info_ref)
    if expect_piv is not None:
        np.testing.assert_array_equal(piv, expect_piv)
    assert np.isfinite(x).all(), tag
    perm = F.row_order(piv)
    aL, aU = np.abs(L), np.abs(Um)

    def env_of(y):      # P^T |L^| |U^| y
        e = np.empty_like(y)
        e[perm] = aL @ (aU @ y)
        return e

    if k <= 2049:
        env = env_of(np.abs(x))
        worst("A X - I", np.abs(a @ x - np.eye(k)), F.residual_bound(a, x, env))
        if k <= 513:
            x_ref, _ = F.inverse_ref(a)
            worst("X - inverse", np.abs(x - x_ref), F.forward_bound(x_ref, env))
    else:
        z = np.random.default_rng(k).standard_normal((k, 64))
        az, ax = np.abs(z), np.abs(x)
        g = F.gamma(3 * k)
        # |A X^ Z - Z| <= |A X^ - I| |Z|, and the host's own two float64 products
        worst("A (X Z) - Z", np.abs(a @ (x @ z) - z),
              g * env_of(ax @ az) + 2 * F.gamma(k) * (np.abs(a) @ (ax @ az)) + U * az)
        # X^ A - I = A^-1 (A X^ - I) A, with |A^-1| <= |X^| + |X^ - A^-1| (the second term is of second order)
        worst("X (A Z) - Z", np.abs(x @ (a @ z) - z),
              1.01 * g * (ax @ env_of(ax @ (np.abs(a) @ az))) + 2 * F.gamma(k) * (ax @ (np.abs(a) @ az)) + U * az)
    return piv


K_SWEEP = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 287, 288, 289, 511, 513,
           1000, 2049, 4100]


def test_k_sweep_covers_the_switches():
    """288 is the first size whose first trailing update (k - 32 square) reaches the 256^2 of gemm_sub's switch"""
    assert (287 - NB) ** 2 < 256 * 256 <= (288 - NB) ** 2
    assert {15, 16, 17} <= set(K_SWEEP)          # CTAs of the 16-CTA cluster that own no row
    assert {127, 128, 129} <= set(K_SWEEP)       # OB = 128 outer blocks of the substitutions
    assert any(k % 8 for k in K_SWEEP)           # ld padding


@pytest.mark.parametrize("k", K_SWEEP)
def test_dense_invert_gaussian(k):
    """real pivoting and growth, no planted diagonal"""
    worst = R.Worst()
    piv = check_inverse(worst, gaussian(k), f"gaussian {k}")
    if k > 2 * NB:
        br = F.panel_branches(piv)
        assert br["inside"] > 0 and br["outside"] > 0, br
    worst.report(f"gaussian k={k}")


@pytest.mark.parametrize("k", [33, 65, 129, 289, 1000])
@pytest.mark.parametrize("kind", ["identity", "inside", "outside", "repeat", "reversed"])
def test_dense_invert_planted_pivot_sequence(kind, k):
    """one family per branch of compose_panel_perm; the restated LU confirms the branch is the one taken"""
    worst = R.Worst()
    if kind == "reversed":
        a = planted(k, np.arange(k))[::-1].copy()
        piv = check_inverse(worst, a, f"{kind} {k}")
        np.testing.assert_array_equal(piv[:k // 2], k - 1 - np.arange(k // 2))
    else:
        want = pivot_sequence(k, kind)
        piv = check_inverse(worst, planted(k, want), f"{kind} {k}", expect_piv=want)
    br = F.panel_branches(piv)
    if kind == "identity":
        assert br == dict(none=k, inside=0, outside=0, repeat=0)
    elif kind == "inside":
        assert br["inside"] > 0 and br["outside"] == br["repeat"] == 0, br
    elif kind == "outside" and k >= 2 * NB:     # at k = 33 one row lies below the first panel
        assert br["outside"] >= NB and br["repeat"] == br["inside"] == 0, br
    elif kind == "repeat":
        assert br["repeat"] >= NB // 2 and br["outside"] > 0, br
    worst.report(f"{kind} k={k}")


@pytest.mark.parametrize("k", [9, 64, 257])
@pytest.mark.parametrize("family", [tied, low_bits, row_scaled, nucleus_like], ids=lambda f: f.__name__)
def test_dense_invert_pivot_rule_edges(family, k):
    worst = R.Worst()
    a = family(k)
    if family is low_bits and k > 1:   # the larger entry sits in the larger row for some column: the key ties
        col = np.abs(a)
        top2 = np.sort(col, axis=0)[-2:]
        assert np.mean(F.truncated(top2[0]) == F.truncated(top2[1])) > 0.9 and np.all(top2[0] != top2[1])
    check_inverse(worst, a, f"{family.__name__} {k}")
    worst.report(f"{family.__name__} k={k}")


@pytest.mark.parametrize("k", [513, 2049])
def test_dense_invert_nucleus_like(k):
    worst = R.Worst()
    a = nucleus_like(k)
    # with 16 CTAs of ceil(k/16) consecutive rows, some CTA sees only zeros in some column of the first panel
    rc = -(-k // 16)
    assert any(not a[c * rc:(c + 1) * rc, j].any() for c in range(16) for j in range(NB))
    check_inverse(worst, a, f"nucleus-like {k}")
    worst.report(f"nucleus-like k={k}")


def _dependent(k, cols, seed=0):
    a = gaussian(k, seed)
    for c in cols:
        a[:, c] = a[:, :c] @ np.random.default_rng(c).uniform(-1.0, 1.0, size=c) if c else 0.0
    return a


SINGULAR = {
    "zero matrix": lambda: np.zeros((40, 40)),
    "zero 1x1": lambda: np.zeros((1, 1)),
    "column 0": lambda: _dependent(70, [0]),
    "column 31": lambda: _dependent(70, [31]),
    "column 32": lambda: _dependent(70, [32]),
    "last partial panel": lambda: _dependent(70, [66]),
    "column k-1": lambda: _dependent(70, [69]),
    "two columns": lambda: _dependent(300, [140, 200]),
    "beyond OB": lambda: _dependent(300, [299]),
    "pivot 0.99e-11": lambda: np.diag([1.0, 2.0, 0.99e-11, 3.0]),
    "pivot 1.0e-11 (truncated below the threshold)": lambda: np.diag([1.0, 2.0, 1.0e-11, 3.0]),
}


def test_dense_invert_singular():
    """an error code, nothing else: the first column without an acceptable pivot, as the restated rule finds it"""
    for name, make in SINGULAR.items():
        a = make()
        info, _ = clp_b200.denseInvert(a)
        info_ref = F.lu_pivot_rule(a)[3]
        assert info_ref > 0, name
        assert info == info_ref, (name, info, info_ref)


def test_dense_invert_accepts_a_pivot_just_above_the_threshold():
    worst = R.Worst()
    check_inverse(worst, np.diag([1.0, 2.0, 1.01e-11, 3.0]), "pivot 1.01e-11")


# ------------------------------------------------------------------ cooperative panel and the hand-over
def coop_geometry(k):
    """(panels that run lu_panel_coop_kernel, its grid G and rows per CTA R for the first panel)"""
    coop = [j0 for j0 in range(0, k, NB) if k - j0 > CLUSTER_ROWS]
    g = min(-(-k // 32), sms())
    return coop, g, -(-k // g)


def probe_residuals(worst, a, x, tag):
    """columns of unit 1-norm: |R z| <= max |R|, so 1e-10 k bounds what the unit columns of the earlier
    test_dense_invert bounded, for every column of the residual at once and from both sides"""
    k = a.shape[0]
    z = np.random.default_rng(k).standard_normal((k, 64))
    z /= np.abs(z).sum(axis=0)
    scale = max(1.0, np.abs(x).max())
    worst("A (X Z) - Z", np.abs(a @ (x @ z) - z).max(), 1e-10 * k * scale)
    worst("X (A Z) - Z", np.abs(x @ (a @ z) - z).max(), 1e-10 * k * scale)


@pytest.mark.parametrize("k,family", [(10271, "gaussian"), (10400, "repeat")])
def test_dense_invert_cooperative_panel_and_hand_over(k, family):
    coop, g, r = coop_geometry(k)
    assert coop == ([0] if k == 10271 else [0, 32, 64, 96, 128]) and g == sms() and r <= 640
    assert (k % 8 != 0) == (k == 10271)     # ld padding on the odd size
    if family == "gaussian":
        a = gaussian(k)
    else:
        want = pivot_sequence(k, "repeat")
        a = planted(k, want)
    info, x = clp_b200.denseInvert(a)
    assert info == 0
    worst = R.Worst()
    probe_residuals(worst, a, x, family)
    worst.report(f"cooperative {family} k={k}")


def test_dense_invert_singular_around_the_hand_over():
    """column 20 lies in the one cooperative panel of k = 10 271, column 40 in the first cluster panel after it"""
    k = 10271
    assert coop_geometry(k)[0] == [0]
    a = gaussian(k, 1)
    keep = a[:, 40].copy()
    a[:, 40] = 2.0 * a[:, 3] - a[:, 7]
    assert clp_b200.denseInvert(a)[0] == 41
    a[:, 20] = 2.0 * a[:, 3] - a[:, 7]          # two dependent columns: the first is reported
    assert clp_b200.denseInvert(a)[0] == 21
    a[:, 40] = keep
    assert clp_b200.denseInvert(a)[0] == 21


# ------------------------------------------------------------------ Engine::refactor with a pivoting nucleus
def canonical(pv, basic, n):
    pv = np.asarray(pv, dtype=np.int64)
    assert sorted(pv.tolist()) == sorted(int(j) for j in basic)
    sl = pv >= n
    np.testing.assert_array_equal(pv[sl] - n, np.flatnonzero(sl))


def check_ftran_btran(worst, s, aext, pv, seed, tag=""):
    ref = R.Basis(aext, pv)
    kappa = ref.cond1()
    rng = np.random.default_rng(seed)
    b = rng.standard_normal(aext.shape[0])
    worst(tag + "updateColumn", np.abs(s.updateColumn(b) - ref.ftran(b)).max(), R.solve_bound(ref.ftran(b), kappa))
    worst(tag + "updateColumnTranspose", np.abs(s.updateColumnTranspose(b) - ref.btran(b)).max(),
          R.solve_bound(ref.btran(b), kappa))
    return kappa


@pytest.mark.parametrize("m,n,k", [(300, 900, 0), (333, 900, 33), (557, 1200, 257), (1500, 3000, 1030),
                                   (4400, 6000, 4100), (261, 800, 261), (1003, 2000, 997)])
def test_refactor_with_a_pivoting_nucleus(m, n, k):
    lp, status = pivoting_lp(m, n, k, seed=77 + k)
    aext = R.ext_matrix(lp)
    if NB < k <= 1100:      # the nucleus really interchanges: the LU of N^T pivots off the diagonal
        nt = lp.to_scipy()[:k, :k].toarray().T
        assert F.panel_branches(F.lu_pivot_rule(nt)[0])["none"] < k // 2
    s = engine(lp, factorizationFrequency=2048)
    basic = np.flatnonzero(status == 1)
    rc, pv = s.factorize(basic)
    assert rc == 0 and s.nucleusSize() == k
    canonical(pv, basic, lp.n)
    pv = pv.astype(np.int64)
    worst = R.Worst()
    check_ftran_btran(worst, s, aext, pv, k)
    entering = iter(range(k, lp.n))
    for _ in range(40):
        q = next(entering)
        f = s.updateColumn(aext[:, q].toarray().ravel())
        r = int(np.argmax(np.abs(f)))
        assert s.replaceColumn(q, r) == 0
        pv[r] = q
    check_ftran_btran(worst, s, aext, pv, k + 1, "after 40 updates: ")
    worst.report(f"pivoting nucleus m={m} k={k}")


def test_duplicate_entries_of_a_column_are_added_in_the_nucleus():
    """loadProblem keeps two entries of a column on the same row apart; PRICE, times and S1 add them, and so
    must the dense nucleus gather"""
    lp, status = pivoting_lp(60, 200, 40, seed=5)
    cs, ri, el = lp.col_start.copy(), lp.row_index, lp.element
    j = 7
    e = cs[j] + int(np.argmax(np.abs(el[cs[j]:cs[j + 1]])))    # a second entry on the home row of basic column 7
    ri2 = np.insert(ri, e, ri[e])
    el2 = np.insert(el, e, 1.0)
    cs[j + 1:] += 1
    lp2 = G.LP("dup-entry", lp.m, lp.n, cs, ri2.astype(np.int32), el2, lp.col_lower, lp.col_upper, lp.objective,
               lp.row_lower, lp.row_upper)
    assert ri2[e] == ri2[e + 1] < 40
    aext = R.ext_matrix(lp2)
    aext.sum_duplicates()
    s = engine(lp2)
    rc, pv = s.factorize(np.flatnonzero(status == 1))
    assert rc == 0
    worst = R.Worst()
    check_ftran_btran(worst, s, aext, pv.astype(np.int64), 3)
    worst.report("duplicate entry")


# ------------------------------------------------------------------ repair of singular bases
def singular_lp(k, kind, deficiency, seed):
    """pivoting_lp whose basis has `deficiency` planted dependent structurals among the k nucleus columns.
    Returns (lp, status, planted sets): each set is the structurals of one dependency, of which exactly one must
    leave."""
    m, n = k + 40, k + 300
    lp, status = pivoting_lp(m, n, k, seed)
    a = lp.to_scipy().tolil()
    rng = np.random.default_rng(seed)
    victims = rng.choice(np.arange(3, k), size=deficiency, replace=False)
    sets = []
    for t, v in enumerate(victims):
        if kind == "duplicate":
            src = [int(t % 3)]
            a[:, v] = a[:, src[0]]
        elif kind == "combination":
            src = [0, 1, 2]
            a[:, v] = 2.0 * a[:, 0] - a[:, 1] + 0.5 * a[:, 2]
        else:   # every entry on a row whose slack is basic: a zero nucleus column
            src = []
            a[:, v] = 0.0
            a[k + t, v] = 3.0
        sets.append(set(src) | {int(v)})
    a = a.tocsc()
    a.sort_indices()
    lp = G.LP(f"singular-{kind}-{k}", m, n, a.indptr.astype(np.int32), a.indices.astype(np.int32), a.data,
              lp.col_lower, lp.col_upper, lp.objective, lp.row_lower, lp.row_upper)
    return lp, status, sets


def check_repair(lp, status, sets, pv, worst, s):
    """structurals left and as many slacks came in, at least one per planted dependency; the basis that remains
    is one the reference can factorize, and FTRAN / BTRAN on it are as accurate as its condition allows"""
    n = lp.n
    basic = set(np.flatnonzero(status == 1).tolist())
    now = set(int(j) for j in pv)
    dropped, entered = basic - now, now - basic
    assert len(dropped) == len(entered) >= len(sets), (dropped, entered)
    assert all(j < n for j in dropped) and all(j >= n for j in entered)
    assert len(dropped & set().union(*sets)) >= len(sets), (dropped, sets)
    assert s.nucleusSize() == len(now & basic & set(range(n)))
    canonical(pv, now, n)
    ref = R.Basis(R.ext_matrix(lp), np.asarray(pv, dtype=np.int64))
    kappa = ref.cond1()
    assert np.isfinite(kappa) and kappa < 1.0e12, kappa
    b = np.random.default_rng(11).standard_normal(lp.m)
    for name, got, want in (("updateColumn", s.updateColumn(b), ref.ftran(b)),
                            ("updateColumnTranspose", s.updateColumnTranspose(b), ref.btran(b))):
        worst(name, np.abs(got - want).max(), 64.0 * U * kappa * (1.0 + np.abs(want).max()))
    return dropped, entered, kappa


def _repair_cases():
    for k, deficiency in [(20, 1), (50, 3), (200, 5), (1030, 1)]:
        for kind in ["duplicate", "combination", "zero column"]:
            marks = ()
            if (kind, k) == ("combination", 50):
                marks = pytest.mark.xfail(strict=True, reason="structural 30, outside the planted span, leaves first; "
                                          "in the nucleus that remains the identical columns 34 and 37 are both "
                                          "basic, yet rounding carried through a pivot of 1e-8 leaves 7e-11 on the "
                                          "last diagonal, above the absolute threshold of 1e-11: kappa_1 = 7e17 is "
                                          "accepted (DESIGN.md section 6)")
            yield pytest.param(kind, k, deficiency, marks=marks, id=f"{kind}-{k}-{deficiency}")


@pytest.mark.parametrize("kind,k,deficiency", list(_repair_cases()))
def test_repair_of_a_singular_basis(kind, k, deficiency):
    lp, status, sets = singular_lp(k, kind, deficiency, seed=k + deficiency)
    basic = np.flatnonzero(status == 1)
    worst = R.Worst()
    # through factorize
    s = engine(lp)
    rc, pv = s.factorize(basic)
    assert rc == 0
    check_repair(lp, status, sets, pv, worst, s)
    # through copyinStatus + startup
    s = engine(lp)
    s.copyinStatus(status)
    assert s.startup() == 0
    pv = s.deviceVector("pivotVariable").astype(np.int64)
    dropped, entered, _ = check_repair(lp, status, sets, pv, worst, s)
    st, sol = s.deviceVector("status"), s.deviceVector("sol")
    lo, up = s.deviceVector("lower"), s.deviceVector("upper")
    for j in dropped:
        assert st[j] in (R.AT_LOWER, R.AT_UPPER, R.FIXED)
        assert sol[j] == (up[j] if st[j] == R.AT_UPPER else lo[j]) and abs(sol[j]) < 1e29
    # a slack that comes in starts at the weight of a fresh basis
    w = s.weights()
    assert all(w[int(np.flatnonzero(pv == j)[0])] == 1.0 for j in entered)
    worst.report(f"repair {kind} k={k} d={deficiency}")


@pytest.mark.xfail(strict=True, reason="Engine::refactor drops the structural the row permutation parked on the "
                   "failing LU column; when the LU of the sparse nucleus fails before its last column that one "
                   "need not belong to the dependency, so more structurals leave than the rank deficiency and "
                   "the basis that remains can be badly conditioned (DESIGN.md section 6)")
@pytest.mark.parametrize("kind", ["duplicate", "combination", "zero column"])
@pytest.mark.parametrize("k,deficiency", [(20, 1), (50, 3)])
def test_repair_drops_exactly_the_dependent_structurals(kind, k, deficiency):
    lp, status, sets = singular_lp(k, kind, deficiency, seed=k + deficiency)
    s = engine(lp)
    rc, pv = s.factorize(np.flatnonzero(status == 1))
    assert rc == 0
    dropped, _, kappa = check_repair(lp, status, sets, pv, R.Worst(), s)
    assert len(dropped) == deficiency and dropped <= set().union(*sets) and kappa < 1.0e4


# ------------------------------------------------------------------ the refresh
def all_bounds_lp(m, n, k, seed):
    """conditioned_lp with every bound type on columns (free, lower only, upper only, boxed, fixed) and rows (free,
    >=, <=, ranged, equality), costs of both signs, and 40 extra columns of cost 0 that touch only rows whose
    slack is basic: their reduced cost is exactly 0, the neutral band of make_dual_feasible"""
    lp, status = conditioned_lp(m, n, k, seed)
    rng = np.random.default_rng(seed + 1)
    extra = 40
    a = sp.hstack([lp.to_scipy(), sp.csc_matrix((np.ones(extra), (k + rng.integers(0, m - k, size=extra),
                                                                   np.arange(extra))), shape=(m, extra))]).tocsc()
    a.sort_indices()
    nn = n + extra
    cl = np.concatenate([lp.col_lower, np.zeros(extra)])
    cu = np.concatenate([lp.col_upper, np.ones(extra)])
    obj = np.concatenate([lp.objective, np.zeros(extra)])
    tj = np.arange(nn) % 5
    cl[tj == 0] = -1e31
    cu[tj == 0] = 1e31
    cu[tj == 1] = 1e31
    cl[tj == 2] = -1e31
    cu[tj == 4] = cl[tj == 4]
    rl, ru = lp.row_lower.copy(), lp.row_upper.copy()
    ti = np.arange(m) % 5
    rl[ti == 0] = -1e31
    ru[ti == 0] = 1e31
    ru[ti == 1] = 1e31
    rl[ti == 2] = -1e31
    ru[ti == 4] = rl[ti == 4]
    st = np.concatenate([status[:n], np.full(extra, 3, dtype=np.uint8), status[n:]])
    st[n:nn][np.arange(extra) % 2 == 0] = 2      # half of the neutral columns start at their upper bound
    lp2 = G.LP(f"all-bounds-{m}x{nn}", m, nn, a.indptr.astype(np.int32), a.indices.astype(np.int32), a.data, cl, cu,
               obj, rl, ru)
    return lp2, st


def true_bounds(lp):
    lo = np.concatenate([lp.col_lower, lp.row_lower]).astype(np.float64)
    up = np.concatenate([lp.col_upper, lp.row_upper]).astype(np.float64)
    return np.where(lo < -1e29, -F.INF, lo), np.where(up > 1e29, F.INF, up)


def device_state(s):
    dv = s.deviceVector
    return dict(sol=dv("sol"), dj=dv("dj"), cost=dv("cost"), lower=dv("lower"), upper=dv("upper"),
                status=dv("status").astype(np.uint8), fake=dv("fake").astype(np.uint8),
                pv=dv("pivotVariable").astype(np.int64), weights=s.weights())


def check_refresh(worst, lp, aext, before, after, dual_bound):
    """the state a refresh left (after) against refresh_ref on the state it started from (before)"""
    n = lp.n
    lo, up = true_bounds(lp)
    ref = F.refresh_ref(aext, after["cost"], lo, up, before["status"], before["fake"], after["pv"], dual_bound)
    basic = before["status"] == R.BASIC
    np.testing.assert_array_equal(after["status"] == R.BASIC, basic)
    assert np.all(after["dj"][basic] == 0.0)
    worst("dj", np.abs(after["dj"] - ref["dj"]), ref["dj_bound"])
    sure = ~ref["edge"]
    for name in ("status", "lower", "upper", "fake"):
        np.testing.assert_array_equal(after[name][sure], ref[name][sure], err_msg=name)
    nb = sure & ~basic
    np.testing.assert_array_equal(after["sol"][nb], ref["sol"][nb])
    assert ref["edge"].sum() <= 2
    if not ref["edge"].any():   # every nonbasic value is the reference's: so must the basic ones be
        scale = 1.0 + np.abs(ref["sol"]).max()
        worst("basic sol", np.abs(after["sol"] - ref["sol"])[basic], np.full(int(basic.sum()), 64.0 * U * ref["kappa"] * scale))
    return ref


@pytest.mark.parametrize("dual_bound", [1.0e3, 1.0e10])
def test_refresh_after_startup_and_after_iterations(dual_bound):
    m, n, k = 400, 2000, 150
    lp, status = all_bounds_lp(m, n, k, seed=99)
    aext = R.ext_matrix(lp)
    s = engine(lp, factorizationFrequency=2048, dualBound=dual_bound)
    s.copyinStatus(status)
    # the state resetStateForRun hands to the first refresh: statuses as given (fixed where the bounds meet,
    # a one-sided variable on its finite bound, a free one free), no fake bounds
    lo, up = true_bounds(lp)
    st0 = status.copy()
    nbm = st0 != R.BASIC
    st0[nbm & (lo == up)] = R.FIXED
    st0[nbm & (lo > -F.INF) & (up >= F.INF)] = R.AT_LOWER
    st0[nbm & (lo <= -F.INF) & (up < F.INF)] = R.AT_UPPER
    st0[nbm & (lo <= -F.INF) & (up >= F.INF)] = R.FREE
    assert s.startup() == 0
    assert s.nucleusSize() == k
    worst = R.Worst()
    after = device_state(s)
    before = dict(status=st0, fake=np.zeros(lp.n + m, dtype=np.uint8))
    ref = check_refresh(worst, lp, aext, before, after, dual_bound)
    took = {b: int((ref["branch"] == b).sum()) for b in set(ref["branch"].tolist())}
    for b in ("fixed", "to lower", "to fake lower", "to upper", "to fake upper", "neutral stays at upper",
              "neutral to lower", "neutral free"):
        assert took.get(b, 0) > 0, (b, took)
    print(f"[dualBound={dual_bound:g}] branches after startup: {took}")

    for t in (1, 300):
        done = s.iterate(t)
        assert done > 0
        before = device_state(s)
        assert s.refresh() == 0
        after = device_state(s)
        canonical(after["pv"], before["pv"], lp.n)
        # the weights follow their variables, bit for bit
        pos = {int(j): p for p, j in enumerate(before["pv"])}
        src = np.array([pos[int(j)] for j in after["pv"]])
        if t == 300:
            assert np.any(src != np.arange(m))      # positions really moved
        np.testing.assert_array_equal(after["weights"], before["weights"][src])
        # the etas are gone: FTRAN is bit for bit the one of a fresh factorization of the same basis
        s2 = engine(lp, factorizationFrequency=2048)
        rc, pv2 = s2.factorize(after["pv"])
        assert rc == 0
        np.testing.assert_array_equal(pv2, after["pv"])
        b = np.random.default_rng(t).standard_normal(m)
        np.testing.assert_array_equal(s.updateColumn(b), s2.updateColumn(b))
        assert s.deviceVector("primalDrift")[0] == F.primal_drift(after["sol"], before["sol"], after["pv"])
        check_refresh(worst, lp, aext, before, after, dual_bound)
    worst.report(f"refresh dualBound={dual_bound:g}")


def test_refresh_of_a_tall_problem():
    """m above 4 x 256 x SMs: primal_drift_kernel's grid-stride loop and every (m + 255) / 256 launch take more
    than one trip"""
    m = 4 * 256 * sms() + 1500
    n, k = 3000, 60
    lp, status = all_bounds_lp(m, n, k, seed=5)
    aext = R.ext_matrix(lp)
    s = engine(lp, factorizationFrequency=2048)
    s.copyinStatus(status)
    assert s.startup() == 0
    assert s.iterate(20) > 0
    before = device_state(s)
    assert s.refresh() == 0
    after = device_state(s)
    canonical(after["pv"], before["pv"], lp.n)
    drift = F.primal_drift(after["sol"], before["sol"], after["pv"])
    assert s.deviceVector("primalDrift")[0] == drift
    worst = R.Worst()
    check_refresh(worst, lp, aext, before, after, 1.0e10)
    worst.report(f"tall m={m}")
