"""High-precision restatement of what Engine::refresh() computes every update cycle: the dense LU of the basis
nucleus with the pivot rule of factor.cu, the explicit inverse, and the refresh kernels of update.cu (duals, the
dual feasible bound of every nonbasic variable with its fake bounds, primals, drift).

Used by tests/test_refactor_kernels.py as the reference of every check there.  numpy / scipy only; it does not
import the engine.  Solves go through iteration_ref.Basis (float64 LU refined twice with extended-precision
residuals).

Bounds.  With P A = L U computed in floating point (L^, U^) and A x = b solved by substitution, Higham, Accuracy
and Stability of Numerical Algorithms (2nd ed.), Theorem 9.4, gives (A + dA) x^ = b with |dA| <= gamma_3k P^T |L^| |U^|,
gamma_n = n u / (1 - n u), hence elementwise

    |A X^ - I|  <=  gamma_3k  P^T |L^| |U^| |X^|                                    (residual_bound)

and, because X - X^ = A^-1 (I - A X^),

    |X^ - X|    <=  gamma_3k  |A^-1| P^T |L^| |U^| |X^|                             (forward_bound)

which is the elementwise form of the kappa_1 bound iteration_ref.solve_bound states for one solve.  The device
uses FMAs and another summation order than lu_pivot_rule; to first order in u that changes neither bound.  The
host evaluates A X^ - I in float64, which by itself costs up to gamma_k |A| |X^|; residual_bound adds that term.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp

import iteration_ref as R
from iteration_ref import AT_LOWER, AT_UPPER, BASIC, FIXED, FREE, U

NB = 32                     # panel width of factor.cu
SINGULAR_TOL = 1.0e-11      # Engine::refactor / Clpb_denseInvert
KEY_MASK = ~np.int64(0xFFFFF)
INF = 1.0e30                # kInf (engine.cuh)


def gamma(n):
    return n * U / (1.0 - n * U)


def truncated(a):
    """|a| with the low 20 bits of the double cleared: the magnitude the pivot keys compare"""
    return (np.abs(np.asarray(a, dtype=np.float64)).view(np.int64) & KEY_MASK).view(np.float64)


def lu_pivot_rule(a, tol=SINGULAR_TOL):
    """LU of a with the pivot rule of lu_panel_cluster_kernel / lu_panel_coop_kernel: in column j the row i >= j
    with the largest truncated |a_ij|, ties to the smallest i; the column is singular when that truncated
    magnitude is below tol (a column that is zero on and below the diagonal included), and is then left as it
    is: no interchange, no elimination.  Right-looking in panels of NB columns like the kernels, so the trailing
    matrix sees the same operations.  Returns (piv, L, U, info): piv[j] the row exchanged with row j, L unit lower
    and U upper triangular with L U = a[perm(piv)] where nothing was singular, info = 1 + the first singular
    column or 0."""
    w = np.array(a, dtype=np.float64, order="F")
    k = w.shape[0]
    piv = np.arange(k)
    info = 0
    for j0 in range(0, k, NB):
        j1 = min(j0 + NB, k)
        for j in range(j0, j1):
            key = truncated(w[j:, j])
            p = j + int(np.argmax(key))          # argmax returns the first of equal maxima
            if not key[p - j] >= tol:
                info = info or j + 1
                continue
            piv[j] = p
            if p != j:
                w[[j, p], :] = w[[p, j], :]
            w[j + 1:, j] *= 1.0 / w[j, j]
            w[j + 1:, j + 1:j1] -= np.outer(w[j + 1:, j], w[j, j + 1:j1])
        if j1 < k:
            l11 = np.tril(w[j0:j1, j0:j1], -1) + np.eye(j1 - j0)
            w[j0:j1, j1:] = sla.solve_triangular(l11, w[j0:j1, j1:], lower=True, unit_diagonal=True)
            w[j1:, j1:] -= w[j1:, j0:j1] @ w[j0:j1, j1:]
    return piv, np.tril(w, -1) + np.eye(k), np.triu(w), info


def row_order(piv):
    """perm with a[perm] = L U: the interchanges j <-> piv[j] applied in order to 0 .. k-1"""
    perm = np.arange(len(piv))
    for j, p in enumerate(piv):
        if p != j:
            perm[[j, p]] = perm[[p, j]]
    return perm


def panel_branches(piv):
    """How often each branch of compose_panel_perm is taken: 'none' (pivot on the diagonal), 'inside' (row of the
    same panel), 'outside' (a row below the panel not yet touched in this panel), 'repeat' (a row below the panel
    that an earlier column of the same panel already exchanged)."""
    count = dict(none=0, inside=0, outside=0, repeat=0)
    for j0 in range(0, len(piv), NB):
        seen = set()
        j1 = min(j0 + NB, len(piv))
        for j in range(j0, j1):
            p = int(piv[j])
            if p == j:
                count["none"] += 1
            elif p < j1:
                count["inside"] += 1
            elif p in seen:
                count["repeat"] += 1
            else:
                seen.add(p)
                count["outside"] += 1
    return count


def inverse_ref(a):
    """(a^-1 refined to extended-precision residuals, kappa_1(a))"""
    k = a.shape[0]
    basis = R.Basis(sp.csc_matrix(np.asarray(a, dtype=np.float64)), np.arange(k))
    return basis.ftran(np.eye(k)), basis.cond1()


def lu_envelope(a, x_hat, tol=SINGULAR_TOL):
    """P^T |L^| |U^| |X^| of the restated LU"""
    piv, L, Um, info = lu_pivot_rule(a, tol)
    assert info == 0, info
    env = np.empty_like(x_hat)
    env[row_order(piv)] = np.abs(L) @ (np.abs(Um) @ np.abs(x_hat))
    return env


def residual_bound(a, x_hat, env):
    k = a.shape[0]
    return gamma(3 * k) * env + gamma(k) * (np.abs(a) @ np.abs(x_hat)) + U


def forward_bound(x_ref, env):
    """the reference itself is accurate to a few u per element after refinement"""
    return gamma(3 * x_ref.shape[0]) * (np.abs(x_ref) @ env) + 8.0 * U * np.abs(x_ref)


# ---------------------------------------------------------------- the refresh
def make_dual_feasible(dj, status, fake, lower_true, upper_true, dual_bound, tol=R.DUAL_TOL):
    """make_dual_feasible_kernel branch by branch.  Returns (status, lower, upper, fake, x, branch): the working
    bounds, the fake flags (1 fake lower, 2 fake upper), the value x of every nonbasic variable (NaN for basic
    ones) and the name of the branch each variable took."""
    nm = len(dj)
    st = np.array(status, dtype=np.uint8)
    lo, up = np.array(lower_true, dtype=np.float64), np.array(upper_true, dtype=np.float64)
    f = np.zeros(nm, dtype=np.uint8)
    x = np.full(nm, np.nan)
    branch = np.empty(nm, dtype=object)
    for j in range(nm):
        if st[j] == BASIC:
            branch[j] = "basic"
        elif lo[j] == up[j]:
            st[j], x[j], branch[j] = FIXED, lo[j], "fixed"
        elif dj[j] > tol:
            branch[j] = "to lower"
            if lo[j] <= -INF:
                lo[j] = (up[j] if up[j] < INF else 0.0) - dual_bound
                f[j], branch[j] = 1, "to fake lower"
            st[j], x[j] = AT_LOWER, lo[j]
        elif dj[j] < -tol:
            branch[j] = "to upper"
            if up[j] >= INF:
                up[j] = (lo[j] if lo[j] > -INF else 0.0) + dual_bound
                f[j], branch[j] = 2, "to fake upper"
            st[j], x[j] = AT_UPPER, up[j]
        elif status[j] == AT_UPPER and up[j] < INF and not (fake[j] & 2):
            x[j], branch[j] = up[j], "neutral stays at upper"
        elif lo[j] > -INF:
            st[j], x[j], branch[j] = AT_LOWER, lo[j], "neutral to lower"
        elif up[j] < INF:
            st[j], x[j], branch[j] = AT_UPPER, up[j], "neutral to upper"
        else:
            st[j], x[j], branch[j] = FREE, 0.0, "neutral free"
    return st, lo, up, f, x, branch


def refresh_ref(aext, cost, lower_true, upper_true, status, fake, pivot_variable, dual_bound, tol=R.DUAL_TOL):
    """What Engine::refresh leaves on the device for the basis pivot_variable: pi = B^-T c_B, d = c - [A | -I]^T pi
    (so c + pi on the rows; 0 on basic variables), make_dual_feasible on d, x_B = B^-1 (-N x_N).  dj_bound is the
    a-priori bound of the device's float64 d: a dot product of nnz_j terms plus the error of pi carried through
    it; `edge` marks the nonbasic variables whose |d| is within that bound of tol, where the branch may differ."""
    pv = np.asarray(pivot_variable, dtype=np.int64)
    basis = R.Basis(aext, pv)
    kappa = basis.cond1()
    pi = basis.btran(cost[pv])
    at = aext.T.tocsr()
    dj = (cost.astype(np.longdouble) - at.astype(np.longdouble) @ pi.astype(np.longdouble)).astype(np.float64)
    nnz = np.diff(at.indptr).astype(np.float64)
    absa = abs(at)
    pi_err = 64.0 * U * kappa * (1.0 + np.abs(pi).max(initial=0.0))   # solve_bound's 1e-10 at kappa = 1e4
    dj_bound = gamma(nnz + 2) * (np.abs(cost) + absa @ np.abs(pi)) + (absa @ np.ones(len(pi))) * pi_err
    basic = np.asarray(status) == BASIC
    dj[basic] = 0.0
    st, lo, up, f, x, branch = make_dual_feasible(dj, status, fake, lower_true, upper_true, dual_bound, tol)
    edge = ~basic & (np.abs(np.abs(dj) - tol) <= dj_bound) & (np.asarray(lower_true) != np.asarray(upper_true))
    sol = np.where(basic, 0.0, x)
    rhs = -(aext.astype(np.longdouble) @ sol.astype(np.longdouble)).astype(np.float64)
    xb = basis.ftran(rhs)
    sol[pv] = xb
    return dict(pi=pi, dj=dj, dj_bound=dj_bound, status=st, lower=lo, upper=up, fake=f, sol=sol, branch=branch,
                edge=edge, kappa=kappa, basis=basis)


def primal_drift(sol, sol_old, pivot_variable):
    """primal_drift_kernel: max_p |x - x_old| / (1 + |x|) over the basic variables"""
    pv = np.asarray(pivot_variable, dtype=np.int64)
    return float(np.max(np.abs(sol[pv] - sol_old[pv]) / (1.0 + np.abs(sol[pv])), initial=0.0))
