"""Synthetic NLPs whose condensed KKT structures reach the branches of the sparse kernel's
symbolic analysis (omg_sp_host.cuh) and factorisation (omg_sp.cuh).  No GPU needed.

The scenarios of the suite all lower to one shape -- chains of spline, hyperplane and slack
coefficients under one dense root of 36 or 40 columns -- so they leave most structural branches
of the sparse kernel unused.  Each family here is a function of (size, seed) that builds an NLP
from ``new_symbol`` / ``Poly`` (rows of degree <= 2, quadratic objective), lowers it with
``lower()`` and returns a ``Case``: the tables, instance data for a small batch (the parameters
enter the right-hand sides, so the instances of one launch differ) and the structural property
it is meant to hit -- bounds on the counters of the structure line (``B200Solver.structure``)
or the reason of the fallback to the envelope kernels.

``nlp()`` couples the variables through
  * objective products c x_i x_j (``pairs``) on top of a diagonal 0.5 h x_i^2, h in [2, 3)
    (h = -1.5 for the variables listed in ``neg``);
  * equality rows  sum_k a_k x_k (+ 0.05 x_first x_last) = p_0  (``eqs``: lists of variables);
  * inequality rows  sum_k x_k^2 <= 4 + p_1  (``ineqs``; ``linear_ineq``: sum_k x_k <= 2 + p_1).

``manufactured_qp()`` builds strictly convex QPs whose KKT point is fixed by construction.
"""
import re

import numpy as np

from omg_tools_b200.basics.lowering import lower
from omg_tools_b200.basics.poly import Poly, new_symbol

# packing limits of the sparse kernel (omg_sp.cuh, omg_sp_host.cuh)
SP_MAXCOL = 62       # longest stored column below the root
SP_MAXROOT = 40      # columns of the dense root
SP_NPF = 2           # uint4 words (2 pair records each) of a gather list fetched one level ahead
SP_SNZ = 8           # explicit zeros one supernode may add
SP_SNZ_TOTAL = 400   # ... all supernodes together
SP_MAXN = 2046       # KKT dimension n + n_eq
SP_MAXL = 8191       # stored entries of the factor + the zero slot
NT = 128             # threads per block: block rows one level may hold


class Case(object):
    """A lowered NLP with instance data.  ``target``: {counter: (lo, hi)} (hi None: no upper
    bound) that the structure line must satisfy; ``reject``: the fallback reason instead;
    ``dup``: (equality row, its copy) pairs; ``x_tol``: a looser tolerance on x, if any."""

    def __init__(self, name, tb, X0, P, target=None, reject=None, dup=(), x_tol=None):
        self.name, self.tb, self.X0, self.P = name, tb, X0, P
        self.target, self.reject = dict(target or {}), reject
        self.dup, self.x_tol = tuple(dup), x_tol


def parse_counters(structure):
    """{name: int} of every ``name=<int>`` of a sparse structure line (N, nnz(L), levels, root,
    and the branch counters after the '|'), and ``early-reject``: the leading levels whose
    negative pivots reject a factorisation at once."""
    out = {k: int(v) for k, v in re.findall(r'([\w()%/-]+)=(\d+)', structure)}
    m = re.search(r'\(early-reject (\d+)\)', structure)
    if m:
        out['early-reject'] = int(m.group(1))
    return out


def nlp(n, pairs=(), eqs=(), ineqs=(), seed=0, quad_eq=True, linear_ineq=False, neg=(), dup=(),
        cubic=(), pair_scale=0.2):
    """Lowered tables.  ``dup``: equality rows (indices into ``eqs``) appended once more,
    unchanged -- linearly dependent rows; ``cubic``: variable triples of extra rows
    x_a x_b x_c <= 1 (term degree 3); ``pair_scale``: standard deviation of the coefficients
    of the objective products (small for dense couplings, to keep the objective convex)."""
    rng = np.random.default_rng(seed)
    x = [new_symbol('x%d' % i, 'var') for i in range(n)]
    p = [new_symbol('p%d' % i, 'par') for i in range(2)]
    neg = set(neg)
    f = Poly({})
    for i in range(n):
        h = -1.5 if i in neg else 2.0 + rng.random()
        f = f + 0.5 * h * x[i] * x[i] + rng.standard_normal() * x[i]
    for i, j in pairs:
        f = f + pair_scale * rng.standard_normal() * x[i] * x[j]
    rows, lb, ub = [], [], []
    for vs in eqs:
        r = -p[0] + Poly({})
        for v in vs:
            r = r + (1.0 + rng.random()) * x[v]
        if quad_eq:
            r = r + 0.05 * x[vs[0]] * x[vs[-1]]
        rows.append(r)
    rows += [rows[k] for k in dup]
    lb += [0.0] * len(rows)
    ub += [0.0] * len(rows)
    for vs in ineqs:
        r = -p[1] + Poly({})
        for v in vs:
            r = r + (x[v] if linear_ineq else x[v] * x[v])
        rows.append(r)
        lb.append(-np.inf)
        ub.append(2.0 if linear_ineq else 4.0)
    for a, b, c in cubic:
        rows.append(x[a] * x[b] * x[c])
        lb.append(-np.inf)
        ub.append(1.0)
    var_ids = [next(iter(v.symbols())) for v in x]
    par_ids = [next(iter(v.symbols())) for v in p]
    return lower(var_ids, par_ids, rows, f, np.array(lb), np.array(ub))


def instances(tb, B=3, seed=0):
    """B starting points near 0 and parameters that move both right-hand sides."""
    rng = np.random.default_rng(seed)
    X0 = 0.1 * rng.standard_normal((B, tb.n))
    P = np.column_stack([0.3 * rng.standard_normal(B), 0.5 * rng.random(B)])
    return X0, P


def _case(name, tb, target=None, reject=None, seed=0, **kw):
    X0, P = instances(tb, 3, seed)
    return Case(name, tb, X0, P, target, reject, **kw)


def _at_least(**kw):
    return {k.replace('_', '-'): (v, None) for k, v in kw.items()}


# ---------------------------------------------------------------------------------------
# structure families
# ---------------------------------------------------------------------------------------
def chain(n, seed=0, eq_every=3, **kw):
    """n variables in a chain, an equality row on (i, i + 1) every ``eq_every`` variables and
    inequality rows on (i, i + 2)."""
    return nlp(n, [(i, i + 1) for i in range(n - 1)], [[i, i + 1] for i in range(0, n - 1, eq_every)],
               [[i, i + 2] for i in range(0, n - 2, 4)], seed, **kw)


def arrow(n, n_glob, seed=0, every=3):
    """n local variables in a chain, every ``every``-th one coupled to all n_glob global
    variables; equality rows on two locals and one global."""
    G = list(range(n, n + n_glob))
    pairs = [(i, i + 1) for i in range(n - 1)] + [(i, g) for i in range(0, n, every) for g in G]
    eqs = [[i, i + 1, G[k % n_glob]] for k, i in enumerate(range(0, n - 1, 5))]
    return nlp(n + n_glob, pairs, eqs, [[i, i + 2] for i in range(0, n - 2, 4)], seed)


def fan(K, L=2, seed=0):
    """K hub variables coupled to each other and to each of L leaves: the leaves are eliminated
    first, each a column of exactly K entries; the hubs end in the root (the first K - 40 of
    them in single-column levels above it).  One equality row on two hubs."""
    hubs = list(range(L, L + K))
    pairs = [(a, b) for a in hubs for b in hubs if a < b] + [(l, h) for l in range(L) for h in hubs]
    return nlp(L + K, pairs, [hubs[:2]], [[h] for h in hubs[::3]], seed, pair_scale=0.02)


def clique(n_var, n_eq, seed=0):
    """n_var coupled variables and n_eq equality rows over them: a dense KKT matrix, all of it
    the root when n_var + n_eq <= 40."""
    d = list(range(n_var))
    pairs = [(i, j) for i in d for j in d if i < j]
    eqs = [sorted(set(d[k::n_eq] + [d[(k + 1) % n_var]])) for k in range(n_eq)]
    return nlp(n_var, pairs, eqs, [[i] for i in d], seed)


def blocks(n_blk, width, seed=0):
    """n_blk independent chains of ``width`` variables, each tied to one global variable by its
    last member: one supernode of ``width`` columns per chain, all on one level -- width - 1
    block rows of the panel step each."""
    g = n_blk * width
    pairs, ineqs = [], []
    for b in range(n_blk):
        v = list(range(b * width, (b + 1) * width))
        pairs += [(v[k], v[k + 1]) for k in range(width - 1)] + [(v[-1], g)]
        ineqs.append([v[0]])
    return nlp(g + 1, pairs, (), ineqs, seed)


def band(n, bw, seed=0):
    """A band of half-width bw, no equality rows."""
    pairs = [(i, i + d) for i in range(n) for d in range(1, bw + 1) if i + d < n]
    return nlp(n, pairs, (), [[i] for i in range(0, n, 40)], seed)


def singular_blocks(n_blk, n_rest=5, seed=0):
    """n_blk blocks of two variables a, b with the objective x_a^2 + x_b^2 + c_a x_a + c_b x_b
    and the equality row x_a + x_b = p_0 twice, next to a clique of n_rest variables with
    inequality rows x_i^2 <= 4 + p_1 (eliminated last: the root).  Every value of a block's KKT
    rows is a small power of two, so its elimination is exact in any order: at delta_w =
    delta_c = 0 the pivots are 2, 2, -1 and exactly 0 for the second copy of the row.  Only the
    equality regularisation delta_c (eq_fail, with the pivot flagged as an equality pivot) makes
    that pivot non-zero; delta_w does not change it.  A block is one 4-column supernode at the
    default width (its two equality pivots in the panel step) and four single-column levels at
    OMG_B200_SNW=1; a single block (n_rest = 0) ends, all but its first column, in the root."""
    rng = np.random.default_rng(seed)
    n = 2 * n_blk + n_rest
    x = [new_symbol('x%d' % i, 'var') for i in range(n)]
    p = [new_symbol('p%d' % i, 'par') for i in range(2)]
    f = Poly({})
    for i in range(n):
        h = 2.0 if i < 2 * n_blk else 2.0 + rng.random()
        f = f + 0.5 * h * x[i] * x[i] + rng.standard_normal() * x[i]
    rest = list(range(2 * n_blk, n))
    for i in rest:
        for j in rest:
            if j < i:
                f = f + 0.2 * rng.standard_normal() * x[i] * x[j]
    rows = []
    for b in range(n_blk):
        r = x[2 * b] + x[2 * b + 1] - p[0]
        rows += [r, r]
    n_eq = len(rows)
    rows += [x[i] * x[i] - p[1] for i in rest]
    lb = np.r_[np.zeros(n_eq), np.full(n_rest, -np.inf)]
    ub = np.r_[np.zeros(n_eq), np.full(n_rest, 4.0)]
    return lower([next(iter(v.symbols())) for v in x], [next(iter(v.symbols())) for v in p], rows, f, lb, ub)


def families():
    """{name: zero-argument builder of the Case}; the builders are cheap to call."""
    F = {}

    def add(name, build, target=None, reject=None, **kw):
        F[name] = lambda: _case(name, build(), target, reject, **kw)

    # equality pivots in single-column levels, in 2..4-column panels; a tree of 222 levels
    add('chain-deep', lambda: chain(400), dict(_at_least(eqpiv_level=1, eqpiv_panel=100, levels=200),
                                              zeros=(SP_SNZ_TOTAL, SP_SNZ_TOTAL)))
    add('chain-short', lambda: chain(30), _at_least(eqpiv_panel=5, sn2=1, sn3=1, sn4=1))
    add('chain-dense-eq', lambda: chain(60, eq_every=2), _at_least(eqpiv_panel=20))
    # long gather lists (more than SP_NPF + 4 words), multi-round backward sweep, root of 40
    add('arrow', lambda: arrow(200, 4), dict(_at_least(max_gather=2 * (SP_NPF + 4) + 1, max_nq=5,
                                                       eqpiv_root=40), **{'max-sn-zeros': (SP_SNZ, SP_SNZ)}))
    add('arrow-dense', lambda: arrow(100, 2, every=1), _at_least(max_gather=40, max_nq=2))
    # one column per backward-sweep round count nq = 1 .. 8; exactly SP_MAXCOL
    for K in (5, 12, 20, 28, 36, 44, 52, SP_MAXCOL):
        add('fan-%d' % K, lambda K=K: fan(K), {'max-col': (K, K), 'max-nq': ((K + 7) // 8, (K + 7) // 8)})
    add('fan-wide', lambda: fan(30, L=40), _at_least(max_slices=33, max_gather=40))
    # root sizes 1 .. 40 with every nr % 4, equality pivots inside the root
    for nv, ne in ((1, 0), (2, 0), (2, 1), (3, 1), (4, 1), (4, 2), (5, 2), (9, 4), (10, 3), (17, 5),
                   (30, 8), (33, 6), (35, 5)):
        nr = nv + ne
        add('root-%d-eq%d' % (nr, ne), lambda nv=nv, ne=ne: clique(nv, ne),
            {'root': (nr, nr), 'root-mod4': (nr % 4, nr % 4), 'eqpiv-root': (ne, ne), 'levels': (0, 0)})
    add('root-41', lambda: clique(41, 0), {'root': (SP_MAXROOT, SP_MAXROOT), 'levels': (1, 1)})
    # wide levels: exactly NT block rows on one level, several panel and back-sweep rounds
    add('blocks-128x2', lambda: blocks(NT, 2), {'max-block-rows': (NT, NT), 'max-panel-rounds': (3, None),
                                               'max-back-rounds': (16, None), 'sn2': (NT, NT)})
    add('blocks-64x3', lambda: blocks(NT // 2, 3), {'max-block-rows': (NT, NT), 'sn3': (NT // 2, NT // 2)})
    # size limits: N = SP_MAXN, nnz(L) + 1 = SP_MAXL
    add('band-maxn', lambda: band(SP_MAXN, 1), {'N': (SP_MAXN, SP_MAXN)})
    add('band-maxl', lambda: band(1558, 3), {'nnz(L)': (SP_MAXL - 1, SP_MAXL - 1)})
    # degenerate shapes
    add('no-eq', lambda: nlp(20, [(i, i + 1) for i in range(19)], (), [[i] for i in range(20)], 1),
        {'eqpiv-level': (0, 0), 'eqpiv-panel': (0, 0), 'eqpiv-root': (0, 0)})
    add('no-ineq', lambda: nlp(20, [(i, i + 1) for i in range(19)], [[i, i + 1] for i in range(0, 19, 3)], (), 2),
        _at_least(eqpiv_panel=1))
    add('linear-rows', lambda: chain(40, quad_eq=False, linear_ineq=True), _at_least(eqpiv_panel=1))
    # inertia: negative curvature (bounded by x_i^2 <= 4 + p_1) in the leading levels, which
    # reject a factorisation at their first negative pivot, with equality pivots below the root
    # (the equality rows touch only the variables 60 ..: the levels of the others come first)
    add('nonconvex', lambda: nlp(120, [(i, i + 1) for i in range(119)], [[i, i + 1] for i in range(60, 119, 3)],
                                 [[i] for i in range(120)], 6, neg=range(0, 60, 3)),
        _at_least(eqpiv_panel=1, early_reject=1))
    # linearly dependent equality rows.  Rounded ones: their second pivot is tiny, not zero
    # (delta_c is not needed; it amplifies rounding all the same: x to 1e-8, only the sum of the
    # two rows' multipliers is unique).  Exact ones (singular_blocks): the second pivot is exactly
    # zero, in the panel step, in single-column levels (OMG_B200_SNW=1) or in the root
    add('dependent-panel', lambda: chain(60, dup=(4,)), _at_least(eqpiv_panel=2), dup=[(4, 20)], x_tol=1e-8)
    add('dependent-root', lambda: nlp(9, [(i, j) for i in range(9) for j in range(i)], [[0, 1, 2], [3, 4, 5]],
                                      [[i] for i in range(9)], 3, dup=(1,)), {'eqpiv-root': (3, 3)},
        dup=[(1, 2)], x_tol=1e-8)
    add('singular-panel', lambda: singular_blocks(6), {'eqpiv-panel': (12, 12), 'eqpiv-level': (0, 0),
                                                      'eqpiv-root': (0, 0), 'sn4': (6, None)},
        dup=[(2 * b, 2 * b + 1) for b in range(6)])
    add('singular-root', lambda: singular_blocks(1, 0), {'eqpiv-root': (2, 2), 'levels': (0, 0)}, dup=[(0, 1)])
    # structures the sparse kernel refuses: the envelope kernels take them
    add('fan-63', lambda: fan(SP_MAXCOL + 1), reject='column structure too long for the packed pairs')
    add('blocks-129x2', lambda: blocks(NT + 1, 2), reject='too many supernodes on one level')
    add('blocks-43x4', lambda: blocks(43, 4), reject='too many supernodes on one level')
    add('band-maxn+1', lambda: band(SP_MAXN + 1, 1), reject='factor too large for the packed pairs')
    add('band-maxl+1', lambda: band(1559, 3), reject='factor too large for the packed pairs')
    add('degree3', lambda: nlp(10, [(i, i + 1) for i in range(9)], [[0, 1]], [[2]], 0, cubic=[(3, 4, 5)]),
        reject='term degree > 2')
    return F


# families whose single-column-level equality pivots need OMG_B200_SNW=1 to appear there
SNW1_LEVEL_EQ = ('chain-short', 'chain-dense-eq', 'no-ineq', 'linear-rows', 'nonconvex', 'dependent-panel',
                 'singular-panel')
# families with an exactly singular equality pivot (the copy of a row)
SINGULAR = ('singular-panel', 'singular-root')


# ---------------------------------------------------------------------------------------
# manufactured optima
# ---------------------------------------------------------------------------------------
def manufactured_qp(n, n_eq, n_act, n_inact, seed=0, eq_only=False):
    """A strictly convex QP on a chain with a global variable, whose KKT point is fixed by
    construction for every parameter value p_0:

        min 0.5 x^T Q x + (c0 + p_0 c1)^T x
        s.t. A x - p_0 A d = A x0                                  (linear equality rows)
             0.5 sum_k D_ik (x_k - a_ik)^2 - p_0 e_i - p_0^2 h_i <= u_i   (convex rows)

    with x*(p) = x0 + p_0 d: e_i, h_i make the row's value at x*(p) independent of p_0; the first
    n_act inequality rows are active (u_i = row value, multiplier z_i > 0), the others have
    slack 0.5; the equality multipliers y are drawn; c0 and c1 make the gradient of the
    Lagrangian vanish at x*(p).  Returns (tables, data) with data = dict(Q, A, x0, d, y, z, c0,
    c1, rows = [(variables, D_i, a_i)] of the quadratic rows) for the references."""
    rng = np.random.default_rng(seed)
    x = [new_symbol('x%d' % i, 'var') for i in range(n)]
    p = [new_symbol('p%d' % i, 'par') for i in range(2)]
    Q = np.diag(3.0 + rng.random(n))
    for i in range(n - 1):
        Q[i, i + 1] = Q[i + 1, i] = 0.5 * rng.standard_normal()
    Q[:, -1] += 0.2 * (np.arange(n) % 4 == 0)                    # the global variable
    Q[-1, :] = Q[:, -1]
    Q[-1, -1] = 3.0 + 0.1 * n
    x0 = 0.5 * rng.standard_normal(n)
    d = rng.standard_normal(n)
    A = np.zeros((n_eq, n))
    for k in range(n_eq):
        c = (k * (n - 2)) // max(n_eq, 1)
        A[k, [c, c + 1, n - 1]] = 1.0 + rng.random(3)
    y = rng.standard_normal(n_eq)
    rows, lb, ub = [], [], []
    grad = Q.dot(x0) + A.T.dot(y)
    gd = Q.dot(d)
    z = np.zeros(n_act + n_inact)
    qrows = []
    for k in range(n_eq):
        rows.append(sum((A[k, j] * x[j] for j in np.nonzero(A[k])[0]), Poly({})) - float(A[k].dot(d)) * p[0])
        lb.append(float(A[k].dot(x0)))
        ub.append(float(A[k].dot(x0)))
    for i in range(0 if eq_only else n_act + n_inact):
        vs = sorted(rng.choice(n, 3, replace=False))
        Dv = 1.0 + rng.random(3)
        av = x0[vs] + 0.3 * rng.standard_normal(3)
        qrows.append((vs, Dv, av))
        r = Poly({})
        for v, Dk, ak in zip(vs, Dv, av):
            r = r + 0.5 * Dk * (x[v] - ak) * (x[v] - ak)
        e = float(np.dot(Dv * (x0[vs] - av), d[vs]))
        h = float(0.5 * np.dot(Dv, d[vs] ** 2))
        rows.append(r - e * p[0] - h * p[0] * p[0])
        val = float(0.5 * np.dot(Dv, (x0[vs] - av) ** 2))
        lb.append(-np.inf)
        if i < n_act:
            z[i] = 0.5 + rng.random()
            grad[vs] += z[i] * Dv * (x0[vs] - av)
            gd[vs] += z[i] * Dv * d[vs]
            ub.append(val)
        else:
            ub.append(val + 0.5)
    c0, c1 = -grad, -gd
    f = sum((0.5 * Q[i, i] * x[i] * x[i] for i in range(n)), Poly({}))
    for i in range(n):
        for j in range(i):
            if Q[i, j] != 0.0:
                f = f + Q[i, j] * x[i] * x[j]
    for i in range(n):
        f = f + c0[i] * x[i] + c1[i] * p[0] * x[i]
    tb = lower([next(iter(v.symbols())) for v in x], [next(iter(v.symbols())) for v in p], rows, f,
               np.array(lb), np.array(ub))
    return tb, dict(Q=Q, A=A, x0=x0, d=d, y=y, z=z, c0=c0, c1=c1, rows=qrows)
