"""Exact reference of the spline kernels (omg_eval_batch, omg_shift_free_batch, omg_sample_batch,
omg_shift_batch), built on the standard library's fractions (and decimal for one linear solve).
Every float input is converted exactly (Fraction(float)), so the only rounding left in a comparison
is the kernel's.

* basis: Cox-de Boor with the interval convention of BSplineBasis.eval_basis (reference
  spline.py:131-136): the leading clamped intervals (i < p + 1 and k[i] == k[0]) are closed, every
  other interval is (k_i, k_i+1], zero-length spans are skipped.
* derivative_coeffs / evaluate: de Boor X.16 with a zero coefficient on a zero-length span.
* shift_free: the free-T re-expression of shift_spline, with the collocation points the host
  chooses (BSplineBasis._collocation: the first arg-max on the 501-point grid), the collocation
  matrices exact and the system solved in 120-digit arithmetic (an exact rational solve of a
  48 x 48 system of degree 8 takes some 25 s; _solve(exact=True) is kept to check the two agree).
* bound: the per-entry error bound k u sum_i |w_i| |q_i| / scale^d, u = 2^-53, from the exact
  terms, where |q| is the coefficient magnitude carried through the difference quotients (so the
  cancellation of a derivative is charged to the bound, not hidden in it).
"""
import decimal
from fractions import Fraction as F

import numpy as np

U = 2.0 ** -53
DROP = F(1e-10)           # _DROP_TOL of basics/spline.py, the float 1e-10 exactly


def fr(v):
    return F(float(v))


def basis(knots, p, x):
    """Exact values of the len(knots) - p - 1 basis functions of degree p at the float x."""
    k = [fr(v) for v in knots] if not isinstance(knots[0], F) else knots
    x = fr(x)
    n_int = len(k) - 1
    lvl = []
    for i in range(n_int):
        lo = x >= k[i] if (i < p + 1 and k[0] == k[i]) else x > k[i]
        lvl.append(F(1) if lo and x <= k[i + 1] else F(0))
    for d in range(1, p + 1):
        nxt = []
        for i in range(n_int - d):
            acc = F(0)
            if lvl[i]:
                den = k[i + d] - k[i]
                if den:
                    acc += (x - k[i]) * lvl[i] / den
            if lvl[i + 1]:
                den = k[i + d + 1] - k[i + 1]
                if den:
                    acc += (k[i + d + 1] - x) * lvl[i + 1] / den
            nxt.append(acc)
        lvl = nxt
    return lvl


def derivative_coeffs(knots, p, c, n_der, magnitude=False):
    """Rows d < n_der of the d-th derivative's L - d coefficients (de Boor X.16): q_d[j] =
    (p - d + 1) (q_d-1[j + 1] - q_d-1[j]) / (k[j + p + 1] - k[j + d]), 0 on a zero-length span.
    magnitude=True carries |q| instead: (p - d + 1) (|q_d-1[j + 1]| + |q_d-1[j]|) / |den|."""
    k = [fr(v) for v in knots]
    q = [[abs(fr(v)) if magnitude else fr(v) for v in c]]
    L = len(c)
    for d in range(1, n_der):
        row = []
        for j in range(L - d):
            den = k[j + p + 1] - k[j + d]
            if not den:
                row.append(F(0))
            elif magnitude:
                row.append((p - d + 1) * (q[-1][j + 1] + q[-1][j]) / abs(den))
            else:
                row.append((p - d + 1) * (q[-1][j + 1] - q[-1][j]) / den)
        q.append(row)
    return q


def evaluate(knots, p, c, x, n_der, scale, k_bound=None):
    """Exact d-th derivatives (d < n_der) of the spline with coefficients c at the float x, each
    divided by scale^d; with k_bound also the error bound k_bound u sum_i |w_i| |q_i| / scale^d of
    each.  Returns (values, bounds) as lists of Fractions / floats."""
    L = len(c)
    q = derivative_coeffs(knots, p, c, n_der)
    qa = derivative_coeffs(knots, p, c, n_der, magnitude=True) if k_bound else None
    s = fr(scale)
    vals, bnds = [], []
    for d in range(n_der):
        w = basis(list(knots)[d:len(knots) - d], p - d, x)
        assert len(w) == L - d
        sd = s ** d
        vals.append(sum((wi * qi for wi, qi in zip(w, q[d]) if wi), F(0)) / sd)
        if k_bound:
            bnds.append(float(k_bound * U * sum((wi * qi for wi, qi in zip(w, qa[d]) if wi), F(0)) / sd))
    return vals, bnds


def dot(a, b):
    """Exact dot product of two float vectors and its error bound 4 len u sum |a_i b_i|."""
    terms = [fr(x) * fr(y) for x, y in zip(a, b)]
    return sum(terms, F(0)), float(4 * len(terms) * U * sum(abs(t) for t in terms))


def _solve(A, R, exact=False):
    """X with A X = R (Gaussian elimination on rows, skipping zero entries: A is the banded
    collocation matrix).  A and R are exact; the elimination runs in 120-digit decimal arithmetic
    (relative rounding 1e-120, some 100 orders below any bound here), or with exact=True in
    Fractions, which costs some 25 s at p = 8, L = 48 against milliseconds.  Returns Fractions."""
    n, m = len(A), len(R[0])
    if exact:
        cv, ctx = (lambda f: f), None
    else:
        ctx = decimal.Context(prec=120)
        cv = (lambda f: ctx.divide(decimal.Decimal(f.numerator), decimal.Decimal(f.denominator)))
    with decimal.localcontext(ctx or decimal.getcontext()):
        zero = cv(F(0))
        A = [[cv(v) if v else zero for v in r] for r in A]
        R = [[cv(v) if v else zero for v in r] for r in R]
        for j in range(n):
            piv = next(i for i in range(j, n) if A[i][j])
            if piv != j:
                A[j], A[piv], R[j], R[piv] = A[piv], A[j], R[piv], R[j]
            nzA = [c for c in range(j + 1, n) if A[j][c]]
            nzR = [c for c in range(m) if R[j][c]]
            for i in range(j + 1, n):
                if not A[i][j]:
                    continue
                f = A[i][j] / A[j][j]
                A[i][j] = zero
                for c in nzA:
                    A[i][c] -= f * A[j][c]
                for c in nzR:
                    R[i][c] -= f * R[j][c]
        X = [[zero] * m for _ in range(n)]
        for i in range(n - 1, -1, -1):
            nz = [c for c in range(i + 1, n) if A[i][c]]
            for col in range(m):
                s = R[i][col]
                for c in nz:
                    s -= A[i][c] * X[c][col]
                X[i][col] = s / A[i][i]
    return [[F(v) for v in r] for r in X]


_SHIFT_CACHE = {}


def shift_matrix(knots, p, tau, exact=False):
    """M of shift_spline(., tau, BSplineBasis(knots, p)): knots2 from the same float
    linspace the host builds, the host's collocation points (the first arg-max of each new basis
    function on linspace(tau, end, 501)), bm M = old_basis(points) with bm and old_basis exact and
    solved as _solve solves it, entries with |M| < 1e-10 dropped as BSplineBasis.transform drops
    them.  Cached per (knots, p, tau)."""
    from omg_tools_b200.basics.spline import BSplineBasis
    knots = np.asarray(knots, dtype=float)
    key = (knots.tobytes(), int(p), float(tau), exact)
    M = _SHIFT_CACHE.get(key)
    if M is not None:
        return M
    L = len(knots) - p - 1
    knots2 = np.r_[tau * np.ones(p), np.linspace(tau, knots[-1], L - p + 1), knots[-1] * np.ones(p)]
    b2 = BSplineBasis(knots2, p)
    m, _ = b2._collocation()
    pts = b2._x[m]
    k1, k2 = [fr(v) for v in knots], [fr(v) for v in knots2]
    bm = [basis(k2, p, x) for x in pts]
    R = [basis(k1, p, x) for x in pts]
    M = _solve(bm, R, exact)
    M = [[v if abs(v) >= DROP else F(0) for v in row] for row in M]
    _SHIFT_CACHE[key] = M
    return M


def shift_free(knots, p, c, tau, k_bound):
    """(M c exactly, its error bound k_bound u sum_k |M_ik| |c_k|) for the coefficients c [L, nc]."""
    M = shift_matrix(knots, p, tau)
    c = np.asarray(c, dtype=float)
    cf = [[fr(v) for v in row] for row in c]
    L, nc = c.shape
    val = np.empty((L, nc), dtype=object)
    bnd = np.empty((L, nc))
    for i in range(L):
        nz = [k for k in range(L) if M[i][k]]
        for j in range(nc):
            val[i, j] = sum((M[i][k] * cf[k][j] for k in nz), F(0))
            bnd[i, j] = float(k_bound * U * sum((abs(M[i][k] * cf[k][j]) for k in nz), F(0)))
    return val, bnd
