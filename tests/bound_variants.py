"""Constraint-row type variants of a scenario's NLP (no GPU needed).

Every scenario of the suite lowers to equality rows and upper-only inequality rows.  The
solver kernels branch on the row type (lower bound, upper bound, equality), so the variants
here rebuild a scenario's NLP from its own rows -- construct_constraints() and lower(), as
scenarios.py does -- with the same rows under other bound kinds:

  * ``mirror``: selected inequality rows g <= u rewritten as -g >= -u (the row polynomial
    negated, the bounds swapped and negated).  Negation is exact in floating point and the
    interior-point method is symmetric under it, so the mirrored NLP has the original's
    iterates bit for bit, with lam_g negated on the mirrored rows.
  * ``band``: per-instance lower bounds below a known solution, turning upper-only rows into
    two-sided rows that contain it.
  * ``free_rows`` / ``mixed_types``: per-instance bound arrays in which a row is free,
    lower-only, upper-only or two-sided depending on the instance.
"""
import numpy as np

from omg_tools_b200.basics.lowering import lower
from omg_tools_b200.basics.optilayer import translate_solver_options
from omg_tools_b200.basics.poly import Poly

from oracle.nlp_eval import TableEval


def _neg(row):
    if isinstance(row, Poly):
        return -row
    return -np.asarray(row, dtype=float).reshape(-1)[0]


def rows_of(pr):
    """The scenario's constraint rows and bounds, as lowered into pr.father.tables."""
    rows, lb, ub = pr.father.construct_constraints()
    return list(rows), np.array(lb, dtype=float), np.array(ub, dtype=float)


def relower(pr, rows, lb, ub):
    f = pr.father
    return lower(f._var_ids, f._par_ids, rows, f.construct_objective(), lb, ub, f.order_hint())


def mirror_rows(tb, sel):
    """Indices of the rows to mirror: 'alternate' = every other inequality row, 'all' = every
    inequality row (then no row keeps an upper bound only)."""
    ineq = np.nonzero(tb.lbg != tb.ubg)[0]
    if sel == 'alternate':
        return ineq[::2]
    if sel == 'all':
        return ineq
    raise ValueError(sel)


def mirror(pr, sel):
    """(tables, idx): the scenario's NLP with the rows ``idx`` (see mirror_rows) rewritten as
    -g(x) in [-ubg, -lbg]."""
    rows, lb, ub = rows_of(pr)
    assert np.array_equal(lb, pr.father.tables.lbg) and np.array_equal(ub, pr.father.tables.ubg)
    idx = mirror_rows(pr.father.tables, sel)
    for i in idx:
        rows[i] = _neg(rows[i])
    lb2, ub2 = lb.copy(), ub.copy()
    lb2[idx], ub2[idx] = -ub[idx], -lb[idx]
    tb = relower(pr, rows, lb2, ub2)
    assert tb.n == pr.father.tables.n and tb.m == pr.father.tables.m
    return tb, idx


def constraint_values(tb, X, P):
    """g(x, p) per instance (unscaled), [B, m]."""
    ev = TableEval(tb)
    return np.array([ev.g(x, ev.tape(p)) for x, p in zip(X, P)])


def band(tb, X_ref, P, w, instances=None):
    """Per-instance [B, m] bounds: on every inequality row of the listed instances (default:
    all) the lower bound min(g(x_ref), ubg) - w, so that the rows become two-sided bands that
    contain x_ref; the other instances keep the lowered bounds."""
    B = X_ref.shape[0]
    LB, UB = np.repeat(tb.lbg[None], B, 0), np.repeat(tb.ubg[None], B, 0)
    ineq = tb.lbg != tb.ubg
    assert np.isinf(tb.lbg[ineq]).all(), 'band() expects upper-only inequality rows'
    g = constraint_values(tb, X_ref, P)
    for b in (range(B) if instances is None else instances):
        LB[b, ineq] = np.minimum(g[b, ineq], tb.ubg[ineq]) - w
    return LB, UB


def slack_rows(tb, g, margin):
    """Mask of the upper-only rows whose bound is more than ``margin`` away from g: rows that
    do not hold the solution g = g(x_ref), so that dropping or replacing their upper bound keeps
    x_ref a solution."""
    ineq = tb.lbg != tb.ubg
    return ineq & (tb.ubg - g > margin)


def free_rows(tb, X_ref, P, instances, margin=0.5):
    """Per-instance [B, m] bounds: in the listed instances every other row with a slack above
    ``margin`` at x_ref (slack_rows) is free (-inf, +inf); the other rows and instances keep
    the lowered bounds.  Returns (LB, UB, mask of the free entries)."""
    B = X_ref.shape[0]
    LB, UB = np.repeat(tb.lbg[None], B, 0), np.repeat(tb.ubg[None], B, 0)
    g = constraint_values(tb, X_ref, P)
    free = np.zeros((B, tb.m), dtype=bool)
    for b in instances:
        rows = np.nonzero(slack_rows(tb, g[b], margin))[0][::2]
        LB[b, rows], UB[b, rows] = -np.inf, np.inf
        free[b, rows] = True
    return LB, UB, free


def mixed_types(tb, X_ref, P, w=0.1, margin=0.5):
    """Per-instance [B, m] bounds whose row types differ between instances.  With k the row's
    position among the inequality rows and g = g(x_ref) of the instance: a row with slack
    (slack_rows) takes type (k + b) % 4 in instance b -- 0 upper-only (as lowered), 1 two-sided
    [g - w, ubg], 2 lower-only [g - w, +inf), 3 free -- and any other row type (k + b) % 2.  Every
    slack row takes every type across four consecutive instances, and x_ref stays a solution of
    every instance; the equality rows stay as they are."""
    B = X_ref.shape[0]
    LB, UB = np.repeat(tb.lbg[None], B, 0), np.repeat(tb.ubg[None], B, 0)
    ineq = np.nonzero(tb.lbg != tb.ubg)[0]
    assert np.isinf(tb.lbg[ineq]).all(), 'mixed_types() expects upper-only inequality rows'
    g = constraint_values(tb, X_ref, P)
    k = np.arange(len(ineq))
    for b in range(B):
        loose = slack_rows(tb, g[b], margin)[ineq]
        kind = np.where(loose, (k + b) % 4, (k + b) % 2)
        lo = np.minimum(g[b, ineq], tb.ubg[ineq]) - w
        LB[b, ineq[kind == 1]] = lo[kind == 1]
        LB[b, ineq[kind == 2]], UB[b, ineq[kind == 2]] = lo[kind == 2], np.inf
        LB[b, ineq[kind == 3]], UB[b, ineq[kind == 3]] = -np.inf, np.inf
    return LB, UB


def row_type_counts(LB, UB):
    """(equality, upper-only, lower-only, two-sided, free) row counts of one bound pair, with the
    solver's classification (|bound| >= 1e19 is no bound)."""
    big = 1e19
    eq = LB == UB
    hL, hU = (LB > -big) & ~eq, (UB < big) & ~eq
    return (int(eq.sum()), int((hU & ~hL).sum()), int((hL & ~hU).sum()), int((hL & hU).sum()),
            int((~eq & ~hL & ~hU).sum()))


def solver(pr, tb, options=None):
    """A B200Solver for tables ``tb`` with the scenario's solver options (the library bound at
    the time of the call: the product's, or the emulation's under the emulation fixture)."""
    from omg_tools_b200.solver.b200 import B200Solver
    opts = translate_solver_options(pr.options)
    opts.update(options or {})
    return B200Solver(tb, opts)
