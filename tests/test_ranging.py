"""Sensitivity analysis: ClpSimplex::dualRanging / primalRanging (ClpSimplexOther.cpp:50-374, :770-1001).

CPU tests check the numpy restatement (tests/ranging_ref.py) on a textbook LP and by re-solving perturbed
LPs with the oracle.  GPU tests compare the device ranging with the restatement on the GPU's own final
basis, and check batching, preconditions and that ranging leaves the solver state alone."""
import numpy as np
import pytest

from conftest import load_golden
from ranging_ref import BASIC, AT_LOWER, AT_UPPER, DBL_MAX, DUAL_NONE, FIXED, PRIMAL_NONE, Ranging

from clp_b200 import generators as G
from oracle import oracle as O


def wyndor():
    # min -3 x1 - 5 x2  s.t.  x1 <= 4, 2 x2 <= 12, 3 x1 + 2 x2 <= 18, x >= 0
    return G.LP("wyndor", 3, 2, np.array([0, 2, 4], np.int32), np.array([0, 2, 1, 2], np.int32),
                np.array([1.0, 3.0, 2.0, 2.0]), np.zeros(2), np.full(2, 1e30), np.array([-3.0, -5.0]),
                np.full(3, -1e30), np.array([4.0, 12.0, 18.0]))


def oracle_status(lp):
    o = O.OracleSimplex(lp)
    assert o.dual() == 0
    return o.status()


def test_wyndor_ranges():
    lp = wyndor()
    r = Ranging(lp, oracle_status(lp))
    ci, si, cd, sd, vi, vd = r.dual_ranging([0, 1])
    np.testing.assert_allclose(ci, [3.0, 3.0], atol=1e-5)
    assert abs(cd[0] - 4.5) < 1e-5
    assert cd[1] == DBL_MAX and sd[1] == -1
    pvi, psi, pvd, psd = r.primal_ranging([3, 4])
    np.testing.assert_allclose(pvi, [6.0, 6.0], atol=1e-5)
    np.testing.assert_allclose(pvd, [6.0, 6.0], atol=1e-5)
    assert list(psi) == [0, 2] and list(psd) == [2, 0]


def _small_planted():
    return G.random_sparse_lp(40, 120, 0.15, 3)


def _resolve(lp, status):
    o = O.OracleSimplex(lp)
    o.set_status(status)
    assert o.dual() == 0
    return o.iterations, o.status()


def _with_cost(lp, j, c):
    obj = lp.objective.copy()
    obj[j] = c
    return G.LP(lp.name, lp.m, lp.n, lp.col_start, lp.row_index, lp.element, lp.col_lower, lp.col_upper, obj,
                lp.row_lower, lp.row_upper)


def _with_fixed(lp, j, v):
    cl, cu = lp.col_lower.copy(), lp.col_upper.copy()
    cl[j] = cu[j] = v
    return G.LP(lp.name, lp.m, lp.n, lp.col_start, lp.row_index, lp.element, cl, cu, lp.objective,
                lp.row_lower, lp.row_upper)


def _cost_samples(r, st, n, rng, count=6):
    cols = np.arange(n)
    ci, si, cd, sd, _, _ = r.dual_ranging(cols, values=False)
    out = []
    for j in rng.permutation(n):
        for rng_, seq, sign in ((ci[j], si[j], 1.0), (cd[j], sd[j], -1.0)):
            if seq >= 0 and 1e-3 < rng_ < 1e20:
                out.append((int(j), sign * rng_))
    return out[:count]


def test_cost_ranges_bound_the_basis_cpu():
    """Moving a cost by 0.99 x its range keeps the optimal basis (0 iterations, same status); 1.01 x
    does not."""
    lp = _small_planted()
    st = oracle_status(lp)
    r = Ranging(lp, st)
    samples = _cost_samples(r, st, lp.n, np.random.default_rng(0))
    assert len(samples) >= 4
    for j, delta in samples:
        it, st2 = _resolve(_with_cost(lp, j, lp.objective[j] + 0.99 * delta), st)
        assert it == 0 and (st2 == st).all(), (j, delta)
        it, st2 = _resolve(_with_cost(lp, j, lp.objective[j] + 1.01 * delta), st)
        assert (st2 != st).any(), (j, delta)  # a basis change or, for a nonbasic column, a bound flip


def _value_samples(r, st, n, count=6):
    nb = [j for j in range(n) if st[j] in (AT_LOWER, AT_UPPER)]
    vi, si, vd, sd = r.primal_ranging(nb)
    out = []
    for q, j in enumerate(nb):
        for v, seq, sign in ((vi[q], si[q], 1.0), (vd[q], sd[q], -1.0)):
            if seq >= 0 and 1e-3 < v < 1e20:
                out.append((j, sign * v, int(seq)))
    return out[:count]


def _infeasible(r, seq, tol=1e-9):
    x = r.x[seq]
    return x < r.lo[seq] - tol * (1 + abs(r.lo[seq])) or x > r.up[seq] + tol * (1 + abs(r.up[seq]))


def test_value_ranges_bound_primal_feasibility_cpu():
    """Fixing a nonbasic column at 0.99 x its primal range keeps the basis primal feasible (0
    iterations); at 1.01 x the blocking basic variable the ranging named is infeasible."""
    lp = _small_planted()
    st = oracle_status(lp)
    r = Ranging(lp, st)
    samples = _value_samples(r, st, lp.n)
    assert len(samples) >= 4
    for j, delta, seq in samples:
        x0 = r.x[j]
        st_fixed = st.copy()
        st_fixed[j] = FIXED
        lp1 = _with_fixed(lp, j, x0 + 0.99 * delta)
        it, _ = _resolve(lp1, st_fixed)
        assert it == 0, (j, delta)
        lp2 = _with_fixed(lp, j, x0 + 1.01 * delta)
        assert _infeasible(Ranging(lp2, st_fixed), seq), (j, delta, seq)
        it, _ = _resolve(lp2, st_fixed)
        assert it > 0, (j, delta)


# ------------------------------------------------------------------------------------------- GPU
def _engine(lp, **params):
    import clp_b200

    s = clp_b200.ClpSimplex()
    s.loadLP(lp)
    for k, v in params.items():
        s.setParameter(k, v)
    return s


def _close(a, b):
    if a == DBL_MAX or b == DBL_MAX or a == -DBL_MAX or b == -DBL_MAX:
        return a == b
    return abs(a - b) <= 1e-8 * (1 + abs(b))


def _check_dual(r, which, got, ref, values=True):
    ci, si, cd, sd = got[:4]
    rci, rsi, rcd, rsd = ref[:4]
    bad = []
    for i, j in enumerate(which):
        for side, (c, s, rc, rs) in enumerate(((ci[i], si[i], rci[i], rsi[i]), (cd[i], sd[i], rcd[i], rsd[i]))):
            if s != rs:
                # accepted only as a tie: the restatement's ratio for the device's sequence is the minimum
                ratios = r.dual_ratios(j)[side] if r.st[j] == BASIC else None
                if ratios is None or s < 0 or rs < 0 or not (ratios[s] < DUAL_NONE and
                                                              ratios[s] - ratios[rs] <= 1e-9 * (1 + abs(ratios[rs]))):
                    bad.append((j, side, s, rs, c, rc))
                continue
            if not _close(c, rc):
                bad.append((j, side, "cost", c, rc))
            elif values and not _close(got[4 + side][i], ref[4 + side][i]):
                bad.append((j, side, "value", got[4 + side][i], ref[4 + side][i]))
    assert not bad, bad[:10]


def _check_primal(r, which, got, ref):
    bad = []
    for i, j in enumerate(which):
        for side in (0, 1):
            v, s, rv, rs = got[2 * side][i], got[2 * side + 1][i], ref[2 * side][i], ref[2 * side + 1][i]
            if s != rs:
                th = r.primal_ratios(j)[side] if r.st[j] != BASIC else None
                ok = th is not None and s >= 0 and rs >= 0 and r.pos[s] >= 0
                if ok:
                    ts, tr = th[r.pos[s]], th[r.pos[rs]]
                    ok = ts < PRIMAL_NONE and ts - tr <= 1e-9 * (1 + abs(tr))
                if not ok:
                    bad.append((j, side, s, rs, v, rv))
            elif not _close(v, rv):
                bad.append((j, side, "value", v, rv))
    assert not bad, bad[:10]


def _agree(lp, **params):
    s = _engine(lp, **params)
    scaling = params.pop("scaling", 0)
    assert s.dual() == 0
    st = s.statusArray()
    rs = cs = None
    if scaling:
        rc, rs, cs = s.scaleFactors()
        if rc != 0:
            rs = cs = None
    r = Ranging(lp, st, row_scale=rs, col_scale=cs)
    which = np.arange(lp.n + lp.m)
    _check_dual(r, which, s.dualRanging(values=True), r.dual_ranging(which))
    _check_primal(r, which, s.primalRanging(), r.primal_ranging(which))


AGREE = ["afiro", "modified_afiro", "UFL-30x100", "TSP-MTZ-40", "transport-10x200", "staircase-480"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", AGREE)
def test_device_ranging_matches_restatement(name):
    _agree(load_golden(name))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(300, 3000, 0.02, 7), (1000, 6000, 0.01, 5)])
def test_device_ranging_matches_restatement_planted(shape):
    _agree(G.random_sparse_lp(*shape))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["UFL-30x100", "staircase-480"])
def test_device_ranging_scaled_in_user_units(name):
    _agree(load_golden(name), scaling=2)


@pytest.mark.gpu
def test_device_cost_and_value_ranges_bound_the_basis():
    lp = _small_planted()
    s = _engine(lp)
    assert s.dual() == 0
    st = s.statusArray()
    ci, si, cd, sd = s.dualRanging(np.arange(lp.n))
    samples = [(j, sign * v) for j in range(lp.n) for v, q, sign in ((ci[j], si[j], 1.0), (cd[j], sd[j], -1.0))
               if q >= 0 and 1e-3 < v < 1e20][:6]
    assert len(samples) >= 4
    for j, delta in samples:
        for f, keeps in ((0.99, True), (1.01, False)):
            t = _engine(_with_cost(lp, j, lp.objective[j] + f * delta))
            t.copyinStatus(st)
            assert t.dual() == 0
            changed = (t.statusArray() != st).any()
            assert (t.numberIterations() == 0 and not changed) if keeps else changed, (j, f)
    nb = np.array([j for j in range(lp.n) if st[j] in (AT_LOWER, AT_UPPER)])
    vi, si, vd, sd = s.primalRanging(nb)
    x = s.primalColumnSolution()
    samples = [(int(j), sign * v, int(q)) for j, a, qa, b, qb in zip(nb, vi, si, vd, sd)
               for v, q, sign in ((a, qa, 1.0), (b, qb, -1.0)) if q >= 0 and 1e-3 < v < 1e20][:6]
    assert len(samples) >= 4
    for j, delta, seq in samples:
        stf = st.copy()
        stf[j] = FIXED
        t = _engine(_with_fixed(lp, j, x[j] + 0.99 * delta))
        t.copyinStatus(stf)
        assert t.dual() == 0 and t.numberIterations() == 0, (j, delta)
        assert _infeasible(Ranging(_with_fixed(lp, j, x[j] + 1.01 * delta), stf), seq), (j, delta, seq)


@pytest.mark.gpu
def test_batching_order_duplicates_and_negatives():
    lp = G.random_sparse_lp(300, 3000, 0.02, 7)
    s = _engine(lp)
    assert s.dual() == 0
    st = s.statusArray()
    full = s.dualRanging(values=True)
    pfull = s.primalRanging()
    rng = np.random.default_rng(4)
    basics = np.flatnonzero(st == BASIC)
    nonbasics = np.flatnonzero(st != BASIC)
    which = np.concatenate([rng.choice(basics, 15), rng.choice(nonbasics, 15), [-1, -5], basics[:3], nonbasics[:2]])
    rng.shuffle(which)
    assert len(which) == 37 and len(set(which.tolist())) < 37
    got = s.dualRanging(which, values=True)
    for i, j in enumerate(which):
        if j < 0:
            assert (got[0][i], got[1][i], got[2][i], got[3][i]) == (0.0, -1, 0.0, -1)
        else:
            for a, b in zip(got, full):
                assert a[i] == b[j], (i, j)
    pw = which[which >= 0]
    pgot = s.primalRanging(pw)
    for i, j in enumerate(pw):
        for a, b in zip(pgot, pfull):
            assert a[i] == b[j], (i, j)


@pytest.mark.gpu
def test_larger_case_sampled():
    lp = G.random_sparse_lp(3000, 30000, 0.01, 20260923)
    s = _engine(lp)
    assert s.dual() == 0
    r = Ranging(lp, s.statusArray())
    which = np.sort(np.random.default_rng(1).choice(lp.n + lp.m, 200, replace=False))
    _check_dual(r, which, s.dualRanging(which, values=True), r.dual_ranging(which))
    _check_primal(r, which, s.primalRanging(which), r.primal_ranging(which))


def _raw(s, which):
    k = len(which)
    w = np.ascontiguousarray(which, np.int32)
    bufs = [np.full(k, 7.0), np.full(k, 7, np.int32), np.full(k, 7.0), np.full(k, 7, np.int32), np.full(k, 7.0),
            np.full(k, 7.0)]
    from clp_b200.simplex import _dp, _ip

    rc = s._L.Clpb_dualRanging(s._h, k, _ip(w), _dp(bufs[0]), _ip(bufs[1]), _dp(bufs[2]), _ip(bufs[3]),
                               _dp(bufs[4]), _dp(bufs[5]))
    rcp = s._L.Clpb_primalRanging(s._h, k, _ip(w), _dp(bufs[0]), _ip(bufs[1]), _dp(bufs[2]), _ip(bufs[3]))
    untouched = all((b == 7).all() for b in bufs)
    return rc, rcp, untouched


@pytest.mark.gpu
def test_preconditions():
    lp = load_golden("afiro")
    which = np.arange(lp.n + lp.m)
    s = _engine(lp)
    assert _raw(s, which) == (1, 1, True)  # never solved
    assert s.dual() == 0
    assert _raw(s, which)[:2] == (0, 0)
    assert _raw(s, [0, lp.n + lp.m]) == (-1, -1, True)
    st = s.statusArray()
    s.chgColumnLower(lp.col_lower)
    assert _raw(s, which) == (1, 1, True)
    assert s.dual() == 0
    s.copyinStatus(st)
    assert _raw(s, which) == (1, 1, True)
    inf = load_golden("Infeasible-10")
    t = _engine(inf)
    assert t.dual() == 1
    assert _raw(t, np.arange(inf.n + inf.m)) == (1, 1, True)


@pytest.mark.gpu
def test_ranging_has_no_side_effects():
    lp = G.random_sparse_lp(300, 3000, 0.02, 7)
    s = _engine(lp)
    assert s.dual() == 0
    assert s.fastDual() == 0 and s.numberIterations() == 0
    before = [s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution(), s.dualRowSolution(),
              s.statusArray()]
    a = s.dualRanging(values=True) + s.primalRanging()
    b = s.dualRanging(values=True) + s.primalRanging()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert s.fastDual() == 0 and s.numberIterations() == 0
    after = [s.primalColumnSolution(), s.primalRowSolution(), s.dualColumnSolution(), s.dualRowSolution(),
             s.statusArray()]
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
