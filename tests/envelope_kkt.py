"""Synthetic NLPs for the envelope kernels (omg_ipm_kernel, _2cta, _xl, _xl_2cta in
csrc/omg_b200.cu): the panel shapes of factor_env / back_solve_env, the shared-memory layouts
that omg_problem_create chooses, and the intermediate-derivative paths of the XL kernel.  No
GPU needed.

Every family is a ``Case`` of tests/synthetic_kkt.py plus the environment it runs in (the
envelope kernels forced, optionally one block of 512 threads per SM) and solver options.  Its
``target`` bounds the fields of the envelope layout (``B200Solver.envelope_layout``, read by
``parse_layout``: ``kernel=.. nt=.. K=.. V=.. arrays-in-scratch=.. max-panel-rows=..
min-panel-rows=.. N%8=.. wide=..``); ``table_counters`` gives what the tables hand the kernel
(panel row counts, equality-pivot positions, intermediate lists).

Families:
  * panel shapes: N % 8 = 0 .. 7, N < 8, block-diagonal bands aligned to the panels (panels
    that reach only the right-hand-side row, rows whose envelope starts at a later panel), one
    dense inequality row (J^T Sigma J dense) whose panels reach NT - 1, NT, NT + 1 and well
    over NT rows at 256 threads, and more than 512 rows at 512 threads;
  * pivots: every family of synthetic_kkt.families() on the envelope kernels (equality pivots,
    negative curvature, dependent and exactly singular equality rows), the equality-pivot
    families again under inertia_mode = 1;
  * layouts: the standard kernel at 2 x 256 and 1 x 512 threads and with per-instance arrays in
    scratch; the XL kernel chosen by size with K and the parameter tape V in shared memory or
    scratch (objective products with parameter-expression coefficients make the tape long);
  * intermediates (XL): mids linear in x under parameter-only row coefficients, mids of degree
    2 .. 4 in equality and inequality rows, rows x_k * mid, mid_a * mid_b and mid^2, one mid in
    many rows.  Nested mids are rejected by lower() (tests/test_model.py) and are not a family.
"""
import re

import numpy as np

from omg_tools_b200.basics.lowering import lower
from omg_tools_b200.basics.poly import Poly, new_mid, new_symbol

import synthetic_kkt as sk

NB = 8           # panel width (csrc/omg_b200.cu)
NT2 = 256        # threads per block of the two-blocks-per-SM kernels
NT1 = 512        # ... of the one-block-per-SM kernels
N_ARR_LOW = 4    # per-instance arrays that always live in scratch (lower-bound / equality-only)


class Case(sk.Case):
    """``ctas``: '1' runs with OMG_B200_CTAS=1; ``options``: solver (and oracle) options;
    ``nlp``: the un-lowered rows of an intermediates family (``unlowered_kkt``)."""

    def __init__(self, name, tb, X0, P, target=None, dup=(), x_tol=None, ctas=None, options=None, nlp=None):
        sk.Case.__init__(self, name, tb, X0, P, target, None, dup, x_tol)
        self.ctas, self.options, self.nlp = ctas, dict(options or {}), nlp


def parse_layout(layout):
    """{key: int or str} of the fields of ``B200Solver.envelope_layout``."""
    out = {}
    for k, v in re.findall(r'(\S+)=(\S+)', layout):
        out[k] = int(v) if v.isdigit() else v
    return out


def panel_rows(tb):
    """Rows each panel of factor_env reaches (the last panel reaches only the right-hand side)."""
    return np.diff(tb.kkt_panel_ptr)


def table_counters(tb):
    """Shapes the tables give the kernel: panel row counts and their parity, back-solve panels
    whose rows all start at a later panel (pcmin > 0), equality pivots by position in their
    diagonal block and in a partial last panel; for intermediates the extra Jacobian slots with
    an x factor (n_jxvar, as omg_problem_create counts them), the longest mu = A^T lambda list,
    the cross-Hessian slots (nnz_wx) and their products x_k * mid (xq_b = -1) and mid_a * mid_b
    (xq_b >= 0), constraint slots that receive only chain-rule terms, and equality rows that
    carry a mid (their slots go to the border of K through jdst)."""
    N = tb.kkt_n
    rows = panel_rows(tb)[:-1]
    first = tb.env_first[:N]
    n_pan = (N + NB - 1) // NB
    pcmin = [min(first[pb * NB:(pb + 1) * NB]) for pb in range(n_pan)]
    eqpos = np.asarray(tb.kkt_pos_eq)
    c = {'N': N, 'odd-rows': int((rows % 2 == 1).sum()), 'even-rows': int((rows % 2 == 0).sum()),
         'pcmin>0': int(sum(1 for v in pcmin if v > 0)),
         'eqpiv-mod8': sorted(set(int(p) % NB for p in eqpos)),
         'eqpiv-last-partial': int(N % NB != 0 and (eqpos >= N - N % NB).any()),
         'n_mid': int(tb.n_mid)}
    if tb.n_mid:
        J = tb.J
        c['n_jxvar'] = sum(1 for s in range(tb.nnz_j, tb.nnz_jx)
                           if (J.xi[J.ptr[s]:J.ptr[s + 1]] != tb.n).any())
        c['max-mu'] = int(np.diff(tb.mu_ptr).max())
        c['nnz_wx'] = int(tb.nnz_wx)
        xq_b = np.asarray(tb.xq_b) if tb.nnz_wx else np.zeros(0, int)
        c['xq_b<0'] = int((xq_b < 0).sum())
        c['xq_b>=0'] = int((xq_b >= 0).sum())
        c['chain-only'] = sum(1 for s in range(tb.nnz_j) if J.ptr[s + 1] == J.ptr[s])
        has_mid = np.diff(tb.jp_ptr) > 0
        eq = set(int(i) for i in tb.kkt_eq_rows)
        c['eq-mid-slots'] = int(sum(1 for s in range(tb.nnz_j) if has_mid[s] and int(tb.jrow[s]) in eq))
    return c


# ---------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------
def _symbols(n, tag):
    x = [new_symbol('%sx%d' % (tag, i), 'var') for i in range(n)]
    p = [new_symbol('%sp%d' % (tag, i), 'par') for i in range(2)]
    return x, p


def _ids(polys):
    return [v.single_symbol() for v in polys]


def blocks_diag(n_blk, seed=0):
    """n_blk cliques of NB variables, no coupling between them: the envelope of every row starts
    at its own panel, so a panel reaches only its own rows and the right-hand side (nrows = 1)
    and the back solve of a panel starts at that panel (pcmin > 0)."""
    pairs = [(b * NB + i, b * NB + j) for b in range(n_blk) for i in range(NB) for j in range(i)]
    return sk.nlp(n_blk * NB, pairs, (), [[i] for i in range(0, n_blk * NB, 3)], seed, pair_scale=0.1)


def dense_row(n):
    """One linear inequality row over every variable: J^T Sigma J is dense and panel pb reaches
    N - 8 (pb + 1) + 1 rows.  One equality row on x0 .. x2."""
    return sk.nlp(n, ineqs=[list(range(n))], linear_ineq=True, eqs=[[0, 1, 2]], seed=1)


def with_residue(r, n0=24):
    """A chain with an equality row on every other pair (the last one on the last variables):
    the smallest n >= n0 whose N = n + n_eq is r mod 8."""
    for n in range(n0, n0 + 24):
        eqs = [[i, i + 1] for i in range(0, n - 1, 2)]
        if (n + len(eqs)) % NB == r:
            return sk.nlp(n, [(i, i + 1) for i in range(n - 1)], eqs, [[i, i + 2] for i in range(0, n - 2, 4)], r)
    raise AssertionError(r)


def many_rows(n):
    """Linear inequality rows x_i + x_j <= 2 + p_1 on every pair: m = n (n - 1) / 2 rows, more
    per-instance vectors than shared memory holds next to a small K."""
    return sk.nlp(n, (), (), [[i, j] for i in range(n) for j in range(i)], 2, linear_ineq=True)


def tape_band(n, bw, seed=0):
    """A band of half-width bw whose objective products carry parameter-expression coefficients
    c_ij (1 + 0.1 p_0 + 0.1 r_ij p_1), r_ij distinct: one tape entry each, so the parameter tape
    V has about n bw entries.  Equality rows on (i, i + 1) every 5 variables, x_i^2 <= 4 + p_1
    every 7."""
    rng = np.random.default_rng(seed)
    x, p = _symbols(n, 'tb')
    f = Poly({})
    for i in range(n):
        f = f + 0.5 * (2.0 + rng.random()) * x[i] * x[i] + rng.standard_normal() * x[i]
    cs = 0.3 / bw * rng.standard_normal((n, bw))
    terms = dict(f.t)                    # summed in place: Poly + Poly copies its terms
    k = 0
    for i in range(n):
        for d in range(1, bw + 1):
            if i + d < n:
                k += 1
                coef = 1.0 + 0.1 * p[0] + (0.1 + 1e-4 * k) * p[1]
                terms.update((float(cs[i, d - 1]) * coef * x[i] * x[i + d]).t)
    f = Poly(terms)
    rows, lb, ub = [], [], []
    for i in range(0, n - 1, 5):
        rows.append((1.0 + rng.random()) * x[i] + (1.0 + rng.random()) * x[i + 1] - p[0])
        lb.append(0.0)
        ub.append(0.0)
    for i in range(0, n, 7):
        rows.append(x[i] * x[i] - p[1])
        lb.append(-np.inf)
        ub.append(4.0)
    return lower(_ids(x), _ids(p), rows, f, np.array(lb), np.array(ub))


def mid_nlp(kind, seed=0):
    """NLPs with intermediates ('mid' symbols), 24 variables in a chain (0.5 h x_i^2 + g_i x_i +
    0.1 c x_i x_{i+1}).  Returns (tables, un-lowered data for ``unlowered_kkt``).
      linear: mids linear in x, row coefficients parameter-only (no extra slot depends on x)
      poly:   mids of degree 2, 3 and 4 in equality rows and in inequality rows
      xmid:   rows 0.5 x_k mid + x_j <= 2 + p_1 (cross-Hessian slots, products x_k * mid)
      midmid: rows mid_a mid_b + x_j <= 2 + p_1 and mid^2 - x_j <= 2 + p_1
      shared: one mid in 40 rows (a long mu = A^T lambda list)"""
    rng = np.random.default_rng(seed)
    n = 24 if kind != 'shared' else 44
    x, p = _symbols(n, 'm' + kind)
    f = Poly({})
    for i in range(n):
        f = f + 0.5 * (2.0 + rng.random()) * x[i] * x[i] + rng.standard_normal() * x[i]
    for i in range(n - 1):
        f = f + 0.1 * rng.standard_normal() * x[i] * x[i + 1]
    rows, lb, ub = [], [], []

    def row(r, kind_):
        rows.append(r)
        lb.append(0.0 if kind_ == 'eq' else -np.inf)
        ub.append(0.0 if kind_ == 'eq' else 2.0)

    if kind == 'linear':
        M = [new_mid('ml%d' % k, x[k] + 0.5 * x[k + 1] - 0.3 * x[k + 2]) for k in range(0, 12, 3)]
        for k, mk in enumerate(M):
            row((1.0 + 0.2 * p[0] + (0.1 + 0.05 * k) * p[1]) * mk + x[12 + k] * x[12 + k] - p[1], 'ineq')
            row((1.5 + 0.1 * k * p[1]) * mk - x[16 + k] - p[0], 'eq')
    elif kind == 'poly':
        M = [new_mid('mp0', x[0] * x[1]), new_mid('mp1', x[2] * x[3] * x[4]),
             new_mid('mp2', x[5] * x[6] * x[7] * x[8]), new_mid('mp3', x[9] * x[9] + 0.5 * x[10] * x[11])]
        for k, mk in enumerate(M):
            row(mk + (1.0 + 0.1 * k) * x[12 + k] - p[0], 'eq')
            row(0.5 * mk + x[16 + k] * x[16 + k] - p[1], 'ineq')
    elif kind == 'xmid':
        M = [new_mid('mx%d' % k, x[2 * k] * x[2 * k + 1] + 0.3 * x[2 * k + 2]) for k in range(4)]
        for k, mk in enumerate(M):
            row(0.5 * x[12 + k] * mk + x[16 + k] - p[1], 'ineq')
            row(mk + x[20 + k] - p[0], 'eq')
    elif kind == 'midmid':
        M = [new_mid('mm%d' % k, x[3 * k] * x[3 * k + 1] + 0.5 * x[3 * k + 2]) for k in range(4)]
        for k in range(3):
            row(M[k] * M[k + 1] + x[12 + k] - p[1], 'ineq')
        for k in range(4):
            row(M[k] * M[k] - x[16 + k] - p[1], 'ineq')
        row(M[0] + x[20] - p[0], 'eq')
    elif kind == 'shared':
        M = [new_mid('ms', x[0] * x[1] + x[2])]
        for k in range(3, 43):
            row((1.0 + 0.05 * k) * M[0] + x[k] * x[k] - p[1], 'ineq')
        row(M[0] + x[43] - p[0], 'eq')
    else:
        raise ValueError(kind)
    lb, ub = np.array(lb), np.array(ub)
    tb = lower(_ids(x), _ids(p), rows, f, lb, ub)
    data = dict(x=_ids(x), p=_ids(p), rows=rows, f=f, lbg=lb, ubg=ub)
    return tb, data


# ---------------------------------------------------------------------------------------
# the end-to-end reference of the intermediates families: the un-lowered rows
# ---------------------------------------------------------------------------------------
def _dpoly(poly, sid):
    """d poly / d symbol ``sid`` (Poly without atoms)."""
    out = {}
    for mono, c in poly.t.items():
        k = mono.count(sid)
        if k:
            red = list(mono)
            red.remove(sid)
            red = tuple(red)
            out[red] = out.get(red, 0.0) + k * c
    return Poly({m: c for m, c in out.items() if c != 0.0})


def expand_mids(poly):
    """``poly`` with every mid replaced by its definition (a Poly in x and p)."""
    from omg_tools_b200.basics.poly import resolve, substitute, sym_info
    mapping = {s: sym_info(resolve(s)).arg for s in poly.symbols() if sym_info(resolve(s)).kind == 'mid'}
    return substitute(poly, mapping)


def unlowered_kkt(data, x, p, lam):
    """(||grad f + J^T lam||_inf, max constraint violation) at (x, lam) from the un-lowered
    rows (mids substituted by their definitions) and their symbolic derivatives."""
    vals = dict(zip(data['x'], x))
    vals.update(zip(data['p'], p))
    rows = [expand_mids(r) for r in data['rows']]
    g = np.array([r.evaluate(dict(vals)) for r in rows])
    grad = np.array([_dpoly(data['f'], s).evaluate(dict(vals)) for s in data['x']])
    for r, l in zip(rows, lam):
        grad += l * np.array([_dpoly(r, s).evaluate(dict(vals)) for s in data['x']])
    viol = np.maximum(0.0, np.maximum(g - data['ubg'], data['lbg'] - g)).max()
    return np.abs(grad).max(), viol


# ---------------------------------------------------------------------------------------
# families
# ---------------------------------------------------------------------------------------
def _exact(**kw):
    return {k.replace('_', '-').replace('N-mod8', 'N%8'): (v, v) for k, v in kw.items()}


STD2 = dict(kernel='standard', nt=NT2, K='shared', V='shared')
# synthetic_kkt families with equality pivots that run once more under inertia_mode = 1
INERTIA1 = ['sk-chain-short', 'sk-chain-dense-eq', 'sk-root-17-eq5', 'sk-nonconvex', 'sk-dependent-panel',
            'sk-singular-panel', 'sk-singular-root']


def families():
    """{name: zero-argument builder of the Case}.  Each family that runs at 2 x 256 threads by
    default is also listed as '<name>@ctas1' (OMG_B200_CTAS=1: one block of 512 threads); the
    ones in INERTIA1 and the N % 8 families also as '<name>@inertia1'."""
    F = {}

    def add(name, build, target=None, ctas=None, options=None, twins=(), **kw):
        def make(name=name, build=build, target=target, ctas=ctas, options=options):
            out = build()
            if isinstance(out, sk.Case):          # a synthetic_kkt family: its instances and tolerances
                return Case(name, out.tb, out.X0, out.P, target, out.dup, out.x_tol, ctas, options)
            tb, data = out if isinstance(out, tuple) else (out, None)
            X0, P = sk.instances(tb, 3, seed=0)
            return Case(name, tb, X0, P, target, ctas=ctas, options=options, nlp=data, **kw)
        F[name] = make
        if 'ctas1' in twins:
            t1 = {k: v for k, v in (target or {}).items() if k not in ('nt', 'K', 'V', 'arrays-in-scratch')}
            t1['nt'] = NT1
            add(name + '@ctas1', build, t1, '1', options, **kw)
        if 'inertia1' in twins:
            add(name + '@inertia1', build, target, ctas, dict(options or {}, inertia_mode=1), **kw)

    # ---- panel shapes -------------------------------------------------------------------
    for r in range(NB):
        add('nmod8-%d' % r, lambda r=r: with_residue(r), dict(STD2, **_exact(N_mod8=r)), twins=('ctas1', 'inertia1'))
    add('tiny-1', lambda: sk.nlp(1, (), (), [[0]], 0), dict(STD2, **_exact(N_mod8=1, max_panel_rows=1)),
        twins=('ctas1',))
    add('tiny-5', lambda: sk.nlp(4, [(0, 1), (1, 2), (2, 3)], [[0, 1, 2, 3]], [[0], [3]], 0),
        dict(STD2, **_exact(N_mod8=5, max_panel_rows=1)), twins=('ctas1',))
    add('blocks-diag', lambda: blocks_diag(5), dict(STD2, **_exact(min_panel_rows=1, max_panel_rows=1)),
        twins=('ctas1',))
    add('band-3', lambda: sk.band(64, 3), STD2, twins=('ctas1',))
    add('band-4', lambda: sk.band(64, 4), STD2, twins=('ctas1',))
    # panels reaching NT - 1, NT, NT + 1 and well over NT rows (K in scratch: XL at 256 threads)
    xl2 = dict(kernel='xl', nt=NT2, K='scratch', V='shared')
    for rows in (NT2 - 1, NT2, NT2 + 1, NT2 + 37):
        add('dense-%d' % rows, lambda rows=rows: dense_row(rows + 7), dict(xl2, **_exact(max_panel_rows=rows)),
            twins=('ctas1',))
    add('dense-523@ctas1', lambda: dense_row(530), {'kernel': 'xl', 'nt': NT1, 'max-panel-rows': (523, 523)},
        ctas='1')
    # ---- layouts ------------------------------------------------------------------------
    add('many-rows', lambda: many_rows(64), dict(STD2, **{'arrays-in-scratch': (N_ARR_LOW + 1, None)}),
        twins=('ctas1',))
    add('tape-k-shared', lambda: tape_band(200, 64), dict(kernel='xl', nt=NT1, K='shared', V='scratch'))
    add('tape-k-scratch', lambda: tape_band(400, 70), dict(kernel='xl', nt=NT2, K='scratch', V='scratch'),
        twins=('ctas1',))
    # ---- intermediates ------------------------------------------------------------------
    for kind in ('linear', 'poly', 'xmid', 'midmid', 'shared'):
        add('mid-' + kind, lambda kind=kind: mid_nlp(kind), dict(kernel='xl', K='shared', V='shared'))
    # ---- pivots: every synthetic_kkt family on the envelope kernels ---------------------
    for name, make in sk.families().items():
        add('sk-' + name, make, {}, twins=('inertia1',) if 'sk-' + name in INERTIA1 else ())
    return F
