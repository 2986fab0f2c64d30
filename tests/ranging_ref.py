"""Numpy restatement of ClpSimplex::dualRanging / primalRanging (ClpSimplexOther.cpp:50-374, :770-1001)
on a dense factorization of the basis a status array describes.  Used by tests/test_ranging.py and
tests/ranging_profile.py as the reference the device results are compared with.

It follows the same rules as the engine (DESIGN.md "Ranging"): alpha_j = -rho^T a_j over [A | -I], the
smallest ratio wins and ties go to the smallest sequence, infinite bounds never block, unbounded sides are
DBL_MAX with sequence -1, and scaled solves are ranged on the scaled problem and unscaled at the end.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

DBL_MAX = np.finfo(np.float64).max
INF = 1.0e30
FREE, BASIC, AT_UPPER, AT_LOWER, SUPERBASIC, FIXED = range(6)
DUAL_NONE, PRIMAL_NONE = 1.0e31, 1.0e30


def _best(ratio, seqs, none):
    """Smallest ratio below `none`, ties to the smallest sequence: (ratio, sequence) or (none, -1)."""
    ok = ratio < none
    if not ok.any():
        return none, -1
    r, s = ratio[ok], seqs[ok]
    i = np.lexsort((s, r))[0]
    return float(r[i]), int(s[i])


class Ranging:
    def __init__(self, lp, status, dual_tol=1e-7, row_scale=None, col_scale=None):
        m, n = lp.m, lp.n
        self.m, self.n, self.tol = m, n, dual_tol
        A = lp.to_scipy().tocsc().astype(np.float64)
        lo = np.concatenate([lp.col_lower, lp.row_lower]).astype(np.float64)
        up = np.concatenate([lp.col_upper, lp.row_upper]).astype(np.float64)
        lo[lo <= -INF] = -INF
        up[up >= INF] = INF
        cost = np.concatenate([lp.objective, np.zeros(m)]).astype(np.float64)
        self.rs = np.ones(m) if row_scale is None else np.asarray(row_scale, np.float64)
        self.cs = np.ones(n) if col_scale is None else np.asarray(col_scale, np.float64)
        if row_scale is not None:  # the engine's working problem (rim_prep.cpp prepareWorkingProblem)
            A = (sp.diags(self.rs) @ A @ sp.diags(self.cs)).tocsc()
            f = np.concatenate([1.0 / self.cs, self.rs])
            fin = np.abs(lo) < INF
            lo[fin] *= f[fin]
            fin = np.abs(up) < INF
            up[fin] *= f[fin]
            cost[:n] *= self.cs
        self.lo, self.up = lo, up
        self.Aext = sp.hstack([A, -sp.identity(m, format="csc")]).tocsc()
        self.st = np.asarray(status, np.uint8).copy()
        self.basic = np.flatnonzero(self.st == BASIC)
        assert len(self.basic) == m, "status must have m basic variables"
        self.pos = np.full(n + m, -1)
        self.pos[self.basic] = np.arange(m)
        self.lu = sla.lu_factor(self.Aext[:, self.basic].toarray())
        nb = np.flatnonzero(self.st != BASIC)
        xn = np.zeros(n + m)
        xn[self.st == AT_LOWER] = lo[self.st == AT_LOWER]
        xn[self.st == FIXED] = lo[self.st == FIXED]
        xn[self.st == AT_UPPER] = up[self.st == AT_UPPER]
        x = xn.copy()
        x[self.basic] = sla.lu_solve(self.lu, -(self.Aext[:, nb] @ xn[nb]))
        self.x = x
        pi = sla.lu_solve(self.lu, cost[self.basic], trans=1)
        dj = cost - self.Aext.T @ pi
        dj[self.basic] = 0.0
        self.dj = dj

    # ---- scale factors (ClpSimplexOther.cpp:215-227 costs, :824-840 values)
    def cost_scale(self, j):
        return 1.0 / self.cs[j] if j < self.n else self.rs[j - self.n]

    def value_scale(self, j):
        return self.cs[j] if j < self.n else 1.0 / self.rs[j - self.n]

    def user_value(self, j):
        return self.x[j] * self.value_scale(j)

    def _unscale_value(self, v, j):
        if v >= 1.0e29:
            return DBL_MAX
        if v <= -1.0e29:
            return -DBL_MAX
        return v * self.value_scale(j)

    # ---- the two ratio tests
    def dual_ratios(self, j):
        """checkDualRatios for the tableau row of basic j: (up ratios, down ratios) over all n+m
        sequences, DUAL_NONE where a sequence is not a candidate (working units)."""
        e = np.zeros(self.m)
        e[self.pos[j]] = 1.0
        rho = sla.lu_solve(self.lu, e, trans=1)
        alpha = -(self.Aext.T @ rho)
        st, dj, tol = self.st, self.dj, self.tol
        cand = (np.abs(alpha) >= 1e-9) & (st != BASIC) & (st != FIXED)
        ru = np.full(self.n + self.m, DUAL_NONE)
        rd = np.full(self.n + self.m, DUAL_NONE)
        with np.errstate(divide="ignore", invalid="ignore"):
            free = cand & ((st == FREE) | (st == SUPERBASIC))
            ru[free] = rd[free] = 0.0
            u = cand & (st == AT_UPPER)
            ru[u & (alpha > 0)] = ((tol - dj) / alpha)[u & (alpha > 0)]
            rd[u & (alpha < 0)] = (-(tol - dj) / alpha)[u & (alpha < 0)]
            lw = cand & (st == AT_LOWER)
            ru[lw & (alpha < 0)] = (-(tol + dj) / alpha)[lw & (alpha < 0)]
            rd[lw & (alpha > 0)] = ((tol + dj) / alpha)[lw & (alpha > 0)]
        return ru, rd

    def ftran(self, j):
        return sla.lu_solve(self.lu, self.Aext[:, [j]].toarray().ravel())

    def primal_ratios(self, j, other=-1):
        """checkPrimalRatios for the FTRAN'd column of j, both directions: (theta up, theta down) per
        basic sequence (PRIMAL_NONE where not a candidate) and the column's entry at `other`."""
        col = self.ftran(j)
        seqs = self.basic
        xb, lo, up = self.x[seqs], self.lo[seqs], self.up[seqs]
        out = []
        for way in (1.0, -1.0):
            a = col * way
            th = np.full(self.m, PRIMAL_NONE)
            with np.errstate(divide="ignore", invalid="ignore"):
                dn = (np.abs(a) > 1e-7) & (a > 0) & (np.abs(lo) < INF) & (seqs != other)
                th[dn] = np.maximum(0.0, (xb - lo)[dn] / a[dn])
                upm = (np.abs(a) > 1e-7) & (a < 0) & (np.abs(up) < INF) & (seqs != other)
                th[upm] = np.maximum(0.0, (xb - up)[upm] / a[upm])
            out.append(th)
        alpha_other = float(col[self.pos[other]]) if other >= 0 and self.pos[other] >= 0 else 0.0
        return out[0], out[1], alpha_other

    def primal_ranging1(self, which_in, which_other):
        """primalRanging1 (:848-953): value of which_other once which_in enters (user units)."""
        way = 1 if self.st[which_in] == AT_LOWER else -1
        tu, td, ao = self.primal_ratios(which_in, which_other)
        theta, _ = _best(tu if way > 0 else td, self.basic, PRIMAL_NONE)
        ao *= way
        v = self.x[which_other]
        if which_in != which_other:
            v = v - theta * ao if theta < PRIMAL_NONE else (-1e30 if ao > 0 else 1e30)
        else:
            v += theta * way
        return self._unscale_value(v, which_other)

    # ---- the two entry points
    def dual_ranging(self, which, values=True):
        k = len(which)
        ci, cd = np.zeros(k), np.zeros(k)
        si, sd = np.full(k, -1), np.full(k, -1)
        vi, vd = np.zeros(k), np.zeros(k)
        seqs = np.arange(self.n + self.m)
        at_bound = lambda s: s >= 0 and self.st[s] in (AT_LOWER, AT_UPPER)
        for i, j in enumerate(which):
            j = int(j)
            if j < 0:
                ci[i], si[i], cd[i], sd[i] = 0.0, -1, 0.0, -1
                vi[i] = vd[i] = np.nan
                continue
            up = down = DBL_MAX
            sup = sdown = -1
            vi[i] = vd[i] = self.user_value(j)
            s = self.st[j]
            if s == BASIC:
                ru, rd = self.dual_ratios(j)
                r, q = _best(ru, seqs, DUAL_NONE)
                if q >= 0:
                    up, sup = r, q
                    if values and at_bound(q):
                        vi[i] = self.primal_ranging1(q, j)
                r, q = _best(rd, seqs, DUAL_NONE)
                if q >= 0:
                    down, sdown = r, q
                    if values and at_bound(q):
                        vd[i] = self.primal_ranging1(q, j)
            elif s in (FREE, SUPERBASIC):
                up = down = 0.0
                sup = sdown = j
            elif s == AT_UPPER:
                up, sup = max(0.0, -self.dj[j]), j
                if values:
                    vi[i] = self.primal_ranging1(j, j)
            elif s == AT_LOWER:
                down, sdown = max(0.0, self.dj[j]), j
                if values:
                    vd[i] = self.primal_ranging1(j, j)
            f = self.cost_scale(j)
            ci[i] = up * f if up < 1e30 else up
            cd[i] = down * f if down < 1e30 else down
            si[i], sd[i] = sup, sdown
        return ci, si, cd, sd, vi, vd

    def primal_ranging(self, which):
        k = len(which)
        vi, vd = np.zeros(k), np.zeros(k)
        si, sd = np.full(k, -1), np.full(k, -1)
        for i, j in enumerate(which):
            j = int(j)
            up = down = DBL_MAX
            sup = sdown = -1
            if self.st[j] in (BASIC, FREE, SUPERBASIC):  # kept as the reference has it (:792-793)
                down = max(0.0, self.up[j] - self.x[j])
                up = max(0.0, self.x[j] - self.lo[j])
                sup = sdown = j
            else:
                tu, td, _ = self.primal_ratios(j)
                r, q = _best(tu, self.basic, PRIMAL_NONE)
                if q >= 0:
                    up, sup = r, q
                r, q = _best(td, self.basic, PRIMAL_NONE)
                if q >= 0:
                    down, sdown = r, q
            f = self.value_scale(j)
            vi[i] = up * f if up < 1e30 else DBL_MAX
            vd[i] = down * f if down < 1e30 else DBL_MAX
            si[i], sd[i] = sup, sdown
        return vi, si, vd, sd
