"""High-precision restatement of one dual simplex iteration of the engine (CHUZR, BTRAN, PRICE, CHUZC, dual
update with bound flips, the three FTRANs, primal update and the DSE recurrence) on a device state.

Used by tests/test_iteration_kernels.py as the reference each kernel of one iteration is compared with.  It is
built from numpy / scipy only and does not import the engine.  The rules are the ones of the kernels
(update.cu, rowpass.cu, kernels_common.cuh); the ratio test itself is the oracle's bucketed restatement
(``oracle.dual_column(..., bucketed=True)``), not a second copy of it.

Solves with B and B^T use a float64 LU (dense for small or dense bases, SuperLU otherwise) followed by two steps
of iterative refinement whose residuals are computed in extended precision, so the reference is accurate to
about u * cond(B) where the kernels are accurate to a multiple of that.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg as sla
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from oracle import oracle as O

# the refinement residuals need a wider type than float64 (x87 80-bit on x86-64 Linux)
assert np.finfo(np.longdouble).eps < 1e-18, "iteration_ref needs an extended-precision np.longdouble"

FREE, BASIC, AT_UPPER, AT_LOWER, SUPERBASIC, FIXED = range(6)
U = np.finfo(np.float64).eps / 2          # unit roundoff of float64
DEVEX_TRY_NORM = 1.0e-4                   # kDevexTryNorm (engine.cuh)
PRIMAL_TOL = DUAL_TOL = ACCEPTABLE = 1.0e-7
ZERO_TOL = 1.0e-13                         # the row pass's zero tolerance on alpha


def ext_matrix(lp):
    """[A | -I] in CSC: column j < n is a structural, column n + i the slack of row i"""
    return sp.hstack([lp.to_scipy().tocsc(), -sp.identity(lp.m, format="csc")]).tocsc().astype(np.float64)


class Basis:
    """Solves with B = [A | -I][:, pivotVariable] and B^T, refined to extended precision."""

    def __init__(self, aext, pivot_variable):
        self.B = aext[:, np.asarray(pivot_variable, dtype=np.int64)].tocsc()
        self.m = self.B.shape[0]
        self.BL = self.B.astype(np.longdouble)
        self.BTL = self.B.T.tocsc().astype(np.longdouble)
        if self.m <= 3000 or self.B.nnz > 0.05 * self.m * self.m:
            lu = sla.lu_factor(self.B.toarray())
            self._solve = lambda b, trans: sla.lu_solve(lu, b, trans=1 if trans else 0)
        else:
            lu = spla.splu(self.B, permc_spec="COLAMD")
            self._solve = lambda b, trans: lu.solve(b, trans="T" if trans else "N")

    def _refined(self, b, trans):
        b = np.asarray(b, dtype=np.float64)
        M = self.BTL if trans else self.BL
        x = self._solve(b, trans).astype(np.longdouble)
        for _ in range(2):
            r = b.astype(np.longdouble) - M @ x
            x = x + self._solve(r.astype(np.float64), trans).astype(np.longdouble)
        return x.astype(np.float64)

    def ftran(self, b):
        """B^-1 b"""
        return self._refined(b, False)

    def btran(self, b):
        """B^-T b"""
        return self._refined(b, True)

    def cond1(self):
        """kappa_1(B) = ||B||_1 ||B^-1||_1 with ||B^-1||_1 from onenormest"""
        m = self.m
        inv = spla.LinearOperator((m, m), matvec=lambda v: self._solve(np.ravel(v), False),
                                  rmatvec=lambda v: self._solve(np.ravel(v), True), dtype=np.float64)
        return float(spla.norm(self.B, 1) * spla.onenormest(inv))


def solve_bound(x, kappa):
    """error bound of a device FTRAN / BTRAN result x on a basis with kappa_1(B) <= 1e4"""
    assert kappa <= 1.0e4, kappa
    return 1.0e-10 * (1.0 + np.abs(x).max(initial=0.0))


class Worst:
    """largest observed error / bound of every check (printed at the end of a test: pytest -s)"""

    def __init__(self):
        self.r = {}

    def __call__(self, name, err, bound):
        err, bound = np.asarray(err, dtype=np.float64).ravel(), np.asarray(bound, dtype=np.float64).ravel()
        assert err.shape == bound.shape
        bad = np.flatnonzero(~(err <= bound))
        assert bad.size == 0, (name, bad[:8], err[bad[:8]], bound[bad[:8]])
        if err.size:
            i = int(np.argmax(err / np.maximum(bound, 1e-300)))
            if err[i] / max(bound[i], 1e-300) >= self.r.get(name, (0.0,))[0]:
                self.r[name] = (float(err[i] / max(bound[i], 1e-300)), float(err[i]), float(bound[i]))

    def report(self, tag):
        for k, (ratio, e, b) in sorted(self.r.items()):
            print(f"[{tag}] {k}: worst error {e:.3g} (bound {b:.3g}, {ratio:.3g} of it)")


# ---------------------------------------------------------------- CHUZR
def chuzr(sol, lower, upper, weights, pivot_variable, tol=PRIMAL_TOL):
    """Dual steepest edge row choice of chuzr_key.  Returns (row, accepted rows): row is the packed-key argmax
    (largest score with its low 20 bits masked, ties to the smallest position); the key masks 20 bits of the
    score, so any row whose score is within 2^-32 relative of the largest one is an acceptable choice."""
    seq = np.asarray(pivot_variable, dtype=np.int64)
    x, lo, up = sol[seq], lower[seq], upper[seq]
    inf = np.where(x < lo - tol, lo - x, np.where(x > up + tol, x - up, 0.0))
    score = np.where(inf > 0.0, inf * inf / weights, 0.0)
    if not (score > 0.0).any():
        return -1, np.zeros(0, dtype=np.int64)
    masked = score.view(np.int64) & ~np.int64(0xFFFFF)
    row = int(np.flatnonzero(masked == masked.max())[0])
    accepted = np.flatnonzero(score >= score.max() * (1.0 - 2.0 ** -32))
    return row, accepted


def pivot_row_scalars(sol, lower, upper, seq_out):
    """(sigma, infeasibility) of the leaving variable (chuzr_finish_body)"""
    v = sol[seq_out]
    if v < lower[seq_out]:
        return -1, lower[seq_out] - v
    return 1, v - upper[seq_out]


# ---------------------------------------------------------------- BTRAN / PRICE
def price(aext, rho, n):
    """alpha_j = a_j^T rho over the structurals, in extended precision, and the a-priori bound
    gamma_{nnz_j} (|A|^T |rho|)_j of a float64 dot product of length nnz_j"""
    A = aext[:, :n].tocsc()
    exact = (A.T.astype(np.longdouble) @ np.asarray(rho, dtype=np.longdouble)).astype(np.float64)
    nnz = np.diff(A.indptr).astype(np.float64)
    gamma = nnz * U / (1.0 - nnz * U)
    return exact, gamma * (abs(A).T @ np.abs(rho))


def finalize_row(raw, rho, status, n):
    """the row pass's P0: basic / fixed entries 0, slack part -rho, zero tolerance"""
    al = np.concatenate([np.asarray(raw, dtype=np.float64), -np.asarray(rho, dtype=np.float64)])
    al[(status == BASIC) | (status == FIXED)] = 0.0
    al[np.abs(al) < ZERO_TOL] = 0.0
    return al


# ---------------------------------------------------------------- CHUZC, dual update, flips
def chuzc(alpha, dj, status, lower, upper, sigma, infeas):
    """(q, theta_d) of the bucketed ratio test on the finalised row; q = -1 when there is no candidate"""
    idx = np.flatnonzero((alpha != 0.0) & (np.abs(alpha) > 1e-12) & (status != BASIC) & (status != FIXED))
    rng = np.where(status[idx] == FREE, 1.0e30, upper[idx] - lower[idx])
    kb, theta, _ = O.dual_column(sigma * alpha[idx], dj[idx], rng, status[idx], infeas, DUAL_TOL, ACCEPTABLE,
                                 bucketed=True)
    return (int(idx[kb]) if kb >= 0 else -1), theta


def dual_update(alpha, dj, status, lower, upper, sol, cost, sigma, theta, q, tol=DUAL_TOL):
    """rowpass.cu P6.  d_j -= theta * sigma * alpha_j; a boxed variable whose new d_j has the wrong sign flips to
    its other bound, any other wrong-signed (or free / superbasic nonzero) one shifts its cost.  Returns the new
    (dj, status, sol, cost), the flipped and the cost-shifted sequences, the per-entry bound 2u(|d|+|theta alpha|)
    of the new d_j (one FMA or two roundings), and the entries whose new d_j is that close to +-tol, where the
    flip / shift decision may go either way."""
    dj, status, sol, cost = dj.copy(), status.copy(), sol.copy(), cost.copy()
    sel = (alpha != 0.0) & (status != BASIC) & (status != FIXED)
    sel[q] = False
    j = np.flatnonzero(sel)
    ta = theta * (sigma * alpha[j])
    dnew = dj[j] - ta
    err = 2.0 * U * (np.abs(dj[j]) + np.abs(ta))
    s = status[j]
    at_lo, at_up = s == AT_LOWER, s == AT_UPPER
    wrong = (at_lo & (dnew < -tol)) | (at_up & (dnew > tol))
    loose = (s == FREE) | (s == SUPERBASIC)
    edge = ((at_lo | loose) & (np.abs(dnew + tol) <= 2 * err)) | ((at_up | loose) & (np.abs(dnew - tol) <= 2 * err))
    boxed = (upper[j] - lower[j]) < 1.0e29
    flip = wrong & boxed
    shift = (wrong & ~boxed) | (loose & (np.abs(dnew) > tol))
    jf = j[flip]
    up_now = status[jf] == AT_LOWER
    status[jf] = np.where(up_now, AT_UPPER, AT_LOWER)
    sol[jf] = np.where(up_now, upper[jf], lower[jf])
    cost[j[shift]] -= dnew[shift]
    dnew[shift] = 0.0
    dj[j] = dnew
    bound = np.zeros_like(dj)
    bound[j] = err
    return dict(dj=dj, status=status, sol=sol, cost=cost, flips=jf, shifts=j[shift], dj_bound=bound,
                edge=j[edge])


def flip_column(aext, flips, status_after, lower, upper, amax):
    """-sum_j a_j delta_j over the flipped variables (delta_j = +range to the upper bound, -range to the lower),
    each row summed exactly (math.fsum), and the bound of the row pass's int64 fixed-point sum (DESIGN.md
    section 4): with Ex from frexp(amax * max range) and Q = 62 - bits(nf) fractional bits every term is rounded
    once to float64 and once to the grid 2^(Ex - Q), the sum is exact, the conversion back rounds once."""
    m = aext.shape[0]
    terms = [[] for _ in range(m)]
    nf = len(flips)
    if nf == 0:
        return np.zeros(m), np.zeros(m)
    rngs = upper[flips] - lower[flips]
    _, ex = math.frexp(float(amax * rngs.max()))
    grid = 2.0 ** (ex - (62 - nf.bit_length()))
    A = aext.tocsc()
    bound = np.zeros(m)
    for j, rg in zip(flips.tolist(), rngs.tolist()):
        delta = rg if status_after[j] == AT_UPPER else -rg
        for e in range(A.indptr[j], A.indptr[j + 1]):
            i, c = int(A.indices[e]), -delta * float(A.data[e])
            terms[i].append(c)
            bound[i] += U * abs(c) + 0.5 * grid
    exact = np.array([math.fsum(t) for t in terms])
    return exact, bound + 2.0 * U * np.abs(exact)


# ---------------------------------------------------------------- after the FTRANs
def primal_step(sol, lower, upper, seq_out, sigma, alpha_col, flip_ftran, nflips, r):
    """theta_p = (x_out [+ flip update] - bound) / alpha_r (pivot_scalars_body)"""
    v = sol[seq_out]
    if nflips > 0:
        v += flip_ftran[r]
    bound = lower[seq_out] if sigma < 0 else upper[seq_out]
    return (v - bound) / alpha_col[r]


def primal_update(sol, pivot_variable, alpha_col, flip_ftran, nflips, theta_p, r, q, seq_out, bound_out):
    """x_B -= theta_p alpha_q (+ the FTRAN'd flip column), the entering variable moves by theta_p, the leaving
    one sits on its bound.  Returns the new sol and the per-basic bound of two roundings."""
    out = sol.copy()
    seq = np.asarray(pivot_variable, dtype=np.int64)
    x = sol[seq] + (flip_ftran if nflips > 0 else 0.0)
    ta = theta_p * alpha_col
    err = 2.0 * U * (np.abs(sol[seq]) + np.abs(flip_ftran if nflips > 0 else 0.0) + np.abs(ta))
    out[seq] = x - ta
    out[q] = sol[q] + theta_p
    out[seq_out] = bound_out
    bound = np.zeros_like(sol)
    bound[seq] = err
    bound[q] = bound[seq_out] = 0.0
    return out, bound


def dse_update(weights, alpha_col, tau, r, rho_norm2, m):
    """the DSE recurrence w_p += (a_p/a_r) ((a_p/a_r) ||rho||^2 - 2 tau_p), clipped at DEVEX_TRY_NORM, and
    w_r = ||rho||^2 / a_r^2; bound for float64 evaluation and an ||rho||^2 summed in another order"""
    w = weights.copy()
    ar = alpha_col[r]
    ratio = alpha_col / ar
    upd = ratio * (ratio * rho_norm2 - 2.0 * tau)
    nz = alpha_col != 0.0
    w[nz] = weights[nz] + upd[nz]
    err = np.where(nz, 8 * U * (np.abs(weights) + ratio * ratio * rho_norm2 + 2 * np.abs(ratio * tau))
                   + ratio * ratio * m * U * rho_norm2, 0.0)
    w[r] = rho_norm2 / (ar * ar)
    err[r] = (m + 4) * U * w[r]
    return np.maximum(w, DEVEX_TRY_NORM), err


# ---------------------------------------------------------------- one whole iteration (the reference on its own)
def dual_feasible_start(lp):
    """all-slack basis with every nonbasic structural at the bound its cost asks for (make_dual_feasible_kernel
    for finite column bounds: no fake bounds), DSE weights 1"""
    m, n = lp.m, lp.n
    lower = np.maximum(np.concatenate([lp.col_lower, lp.row_lower]).astype(np.float64), -1.0e30)
    upper = np.minimum(np.concatenate([lp.col_upper, lp.row_upper]).astype(np.float64), 1.0e30)
    assert np.all(np.abs(lower[:n]) < 1e30) and np.all(np.abs(upper[:n]) < 1e30), "finite column bounds only"
    cost = np.concatenate([lp.objective, np.zeros(m)]).astype(np.float64)
    dj = cost.copy()
    dj[n:] = 0.0
    status = np.full(n + m, AT_LOWER, dtype=np.uint8)
    status[n:] = BASIC
    status[:n] = np.where(lp.col_lower == lp.col_upper, FIXED, np.where(dj[:n] < -DUAL_TOL, AT_UPPER, AT_LOWER))
    sol = np.where(status == AT_UPPER, upper, lower)
    sol[n:] = lp.to_scipy() @ sol[:n]
    return dict(sol=sol, dj=dj, status=status, lower=lower, upper=upper, cost=cost,
                pv=np.arange(n, n + m), weights=np.ones(m))


def step(aext, s, amax):
    """one iteration of the reference on state s (modified in place).  Returns (row, seqOut, seqIn, sigma,
    theta_d) or None when no row is primal infeasible."""
    n = aext.shape[1] - aext.shape[0]
    r, _ = chuzr(s["sol"], s["lower"], s["upper"], s["weights"], s["pv"])
    if r < 0:
        return None
    out = int(s["pv"][r])
    sigma, infeas = pivot_row_scalars(s["sol"], s["lower"], s["upper"], out)
    basis = Basis(aext, s["pv"])
    e = np.zeros(aext.shape[0])
    e[r] = 1.0
    rho = basis.btran(e)
    raw, _ = price(aext, rho, n)
    alpha = finalize_row(raw, rho, s["status"], n)
    q, theta = chuzc(alpha, s["dj"], s["status"], s["lower"], s["upper"], sigma, infeas)
    assert q >= 0
    theta = max(s["dj"][q] / (sigma * alpha[q]), 0.0)
    du = dual_update(alpha, s["dj"], s["status"], s["lower"], s["upper"], s["sol"], s["cost"], sigma, theta, q)
    fl, _ = flip_column(aext, du["flips"], du["status"], s["lower"], s["upper"], amax)
    aq = aext[:, q].toarray().ravel()
    alpha_col, tau, ffl = basis.ftran(aq), basis.ftran(rho), basis.ftran(fl)
    nf = len(du["flips"])
    theta_p = primal_step(du["sol"], s["lower"], s["upper"], out, sigma, alpha_col, ffl, nf, r)
    bound = s["lower"][out] if sigma < 0 else s["upper"][out]
    sol, _ = primal_update(du["sol"], s["pv"], alpha_col, ffl, nf, theta_p, r, q, out, bound)
    w, _ = dse_update(s["weights"], alpha_col, tau, r, math.fsum(rho * rho), aext.shape[0])
    dj = du["dj"]
    dj[q] = 0.0
    dj[out] = -sigma * theta
    status = du["status"]
    status[q] = BASIC
    status[out] = FIXED if s["lower"][out] == s["upper"][out] else (AT_LOWER if sigma < 0 else AT_UPPER)
    s.update(sol=sol, dj=dj, status=status, cost=du["cost"], weights=w)
    s["pv"] = s["pv"].copy()
    s["pv"][r] = q
    return r, out, q, sigma, theta
