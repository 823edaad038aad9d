"""The sparse solver kernel on synthetic KKT structures that reach every branch of its symbolic
analysis (omg_sp_host.cuh) and factorisation (omg_sp.cuh).

The families of tests/synthetic_kkt.py put equality pivots into single-column levels, supernode
panels and the root; build roots of every size up to SP_MAXROOT and every nr % 4; long gather
lists and columns of up to SP_MAXCOL entries (backward-sweep rounds nq = 1 .. 8); levels with
exactly 128 block rows and several panel and back-sweep rounds; the explicit-zero budgets; the
SP_MAXN and SP_MAXL limits; degenerate shapes; negative curvature and linearly dependent
equality rows.  Next to each limit sits a structure one step over it, which the envelope
kernels must take.  The structure line's counters (after its '|') show that each family hits
the branch it is meant for.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu); the ones marked gpu
run the same cases through the product library on the device."""
import os
import sys

import numpy as np
import pytest

from oracle import ipm_c

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emu_support                       # noqa: E402
import synthetic_kkt as sk               # noqa: E402

FAMILIES = sk.families()
DENSE_ORACLE_MAX_N = 400       # the dense oracle is O(N^3) per factorisation: larger ones use 'sparse'
TIGHT = {'tol': 1e-8, 'compl_inf_tol': 1e-8, 'constr_viol_tol': 1e-8}
_CASES = {}


def case(name):
    if name not in _CASES:
        _CASES[name] = FAMILIES[name]()
    return _CASES[name]


@pytest.fixture
def emu():
    if not ipm_c.available():
        pytest.skip('C oracle not built')
    saved = emu_support.activate()
    yield
    emu_support.restore(saved)


@pytest.fixture(scope='module')
def gpu():
    import __graft_entry__ as ge
    ge.build()
    if not ipm_c.available():
        pytest.skip('C oracle not built')


@pytest.fixture(params=[None, '1'], ids=['snw-default', 'snw1'])
def snw(request, monkeypatch):
    """Supernode width: the default, and one column per level step."""
    if request.param:
        monkeypatch.setenv('OMG_B200_SNW', request.param)
    return request.param


def solver(tb, options=None):
    from omg_tools_b200.solver.b200 import B200Solver
    return B200Solver(tb, dict(options or {}))


def check_structure(c, structure, snw=None):
    """The family hits its branch: the target counters, or the fallback with its reason."""
    if snw == '1':                       # no supernodes, no explicit zeros: other limits apply
        if not c.reject:                 # (a family that the sparse kernel takes at the default
            assert structure.startswith('sparse LDL^T'), structure     # width takes it here too)
        if structure.startswith('sparse'):
            cnt = sk.parse_counters(structure)
            assert cnt['sn2'] == cnt['sn3'] == cnt['sn4'] == cnt['eqpiv-panel'] == cnt['zeros'] == 0, structure
        return
    if c.reject:
        assert structure == 'envelope kernels (%s)' % c.reject, structure
        return
    cnt = sk.parse_counters(structure)
    assert structure.startswith('sparse LDL^T'), structure
    for key, (lo, hi) in c.target.items():
        assert cnt[key] >= lo and (hi is None or cnt[key] <= hi), (key, cnt[key], structure)


def match(res, ref, x_tol, lam_tol=None, dup=()):
    """Statuses and iteration counts identical; x and f (relative to max(1, |f|)) to x_tol,
    lam_g to lam_tol (default 1e2 x_tol); returns the deviations.  ``dup``: (row, its duplicate) -- only the sum of their
    multipliers is unique."""
    res, ref = dict(res), dict(ref)
    for key in ('lam_g',) if dup else ():
        for d in (res, ref):
            d[key] = d[key].copy()
            for a, b in dup:
                d[key][:, a] += d[key][:, b]
                d[key][:, b] = 0.0
    assert np.array_equal(res['status'], ref['status']), (res['status'], ref['status'])
    assert np.array_equal(res['iters'], ref['iters']), (res['iters'], ref['iters'])
    dx = np.abs(res['x'] - ref['x']).max()
    df = np.abs(res['f'] - ref['f']).max()
    dl = np.abs(res['lam_g'] - ref['lam_g']).max()
    assert dx <= x_tol and df <= x_tol * max(1.0, np.abs(ref['f']).max()), (dx, df)
    assert dl <= (lam_tol if lam_tol is not None else 1e2 * x_tol), dl
    return dx, dl


def oracles(c, X0, P, lbg=None, ubg=None):
    """The C oracle's dense arm (small structures) and its sparse arm (always)."""
    out = []
    if c.tb.kkt_n <= DENSE_ORACLE_MAX_N:
        out.append(ipm_c.solve_batch_full(c.tb, X0, P, threads=8, lbg=lbg, ubg=ubg))
    out.append(ipm_c.solve_batch_full(c.tb, X0, P, threads=8, options={'linear_solver': 'sparse'},
                                      lbg=lbg, ubg=ubg))
    return out


def check_family(name, snw, x_tol, X0=None, P=None, lbg=None, ubg=None, tile=None):
    """``tile``: X0 and P repeat their first ``tile`` instances; the oracle solves those."""
    c = case(name)
    slv = solver(c.tb)
    check_structure(c, slv.structure, snw)
    X0 = c.X0 if X0 is None else X0
    P = c.P if P is None else P
    res = slv.solve_batch(X0, P, lbg, ubg)
    if not c.reject:
        assert (res['status'] == 0).all(), res['status']
    refs = oracles(c, X0[:tile], P[:tile], lbg, ubg) if tile else oracles(c, X0, P, lbg, ubg)
    if tile:
        refs = [{k: np.resize(v, (len(X0),) + v.shape[1:]) for k, v in r.items()} for r in refs]
    devs = [match(res, ref, c.x_tol or x_tol, dup=c.dup) for ref in refs]
    return slv, res, devs


# ---------------------------------------------------------------------------------------
# emulated kernels (CPU)
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(FAMILIES))
def test_family_matches_the_oracle(emu, snw, name):
    """Every family at the default supernode width and at OMG_B200_SNW=1 hits its branch (or
    falls back to the envelope kernels with the expected reason) and matches the C oracle's
    dense and sparse arms: statuses and iteration counts identical, x and f to 1e-12, lam_g to
    1e-10 (measured: x 7.5e-15, lam_g 2.9e-15).  The rounded dependent equality rows: x to 1e-8
    (measured 3.2e-10) and the sum of the two rows' multipliers to 1e-6 (measured 3.6e-11)."""
    check_family(name, snw, 1e-12)


@pytest.mark.parametrize('name', sk.SNW1_LEVEL_EQ)
def test_single_column_levels_take_the_equality_pivots(emu, monkeypatch, name):
    """With one column per level step the equality pivots that the default width puts into
    supernode panels sit in single-column levels (the eq-pivot bit of the gather's entry
    word)."""
    cnt0 = sk.parse_counters(solver(case(name).tb).structure)
    panel, level0 = cnt0['eqpiv-panel'], cnt0['eqpiv-level']
    monkeypatch.setenv('OMG_B200_SNW', '1')
    cnt = sk.parse_counters(solver(case(name).tb).structure)
    assert panel > 0 and cnt['eqpiv-panel'] == 0 and cnt['eqpiv-level'] == panel + level0


def test_negative_curvature_runs_the_early_rejection_and_the_delta_w_schedule(emu):
    """'nonconvex': variables with negative curvature that no equality row touches fill the
    leading levels, which reject a factorisation at their first negative pivot (early-reject > 0),
    and equality pivots sit below the root.  The inertia correction runs: delta_w > 0 (the trace's
    last column, the previous iteration's value) in at least five iterations of instance 0 (18 of
    its 23) -- with the statuses and iteration counts of the oracle
    (test_family_matches_the_oracle)."""
    c = case('nonconvex')
    slv = solver(c.tb, {'trace': 1})
    cnt = sk.parse_counters(slv.structure)
    assert 0 < cnt['early-reject'] < cnt['levels'] and cnt['eqpiv-panel'] > 0
    res = slv.solve_batch(c.X0, c.P)
    assert (res['status'] == 0).all()
    dw = slv.trace(512)[:res['iters'][0] + 1, 7]
    assert (dw > 0).sum() >= 5


@pytest.mark.parametrize('name, snw_', [('singular-panel', None), ('singular-panel', '1'), ('singular-root', None)])
def test_exactly_singular_equality_pivot_takes_the_delta_c_path(emu, monkeypatch, name, snw_):
    """synthetic_kkt.singular_blocks: the copy of an equality row has an exactly zero pivot at
    delta_w = delta_c = 0, in the panel step (default width), in a single-column level
    (OMG_B200_SNW=1) or in the root.  The kernel flags it as a bad EQUALITY pivot (the eq-pivot bit
    of the level entry word, of the panel task, of the root chunk), which sets delta_c; delta_w
    alone leaves that pivot zero.  Shown here: where the pivots are; that the first factorisation
    of the first iteration is rejected (delta_w > 0 in the trace's second row); and that the numpy
    twin of the oracle without delta_c (delta_c_val = 0) does not reproduce the kernel's run, while
    with it it does.  test_family_matches_the_oracle adds the C oracle's statuses, iteration
    counts and solutions."""
    from oracle import ipm_ref
    if snw_:
        monkeypatch.setenv('OMG_B200_SNW', snw_)
    c = case(name)
    slv = solver(c.tb, {'trace': 1})
    cnt = sk.parse_counters(slv.structure)
    n_copy = len(c.dup)
    place = 'eqpiv-root' if name == 'singular-root' else ('eqpiv-level' if snw_ else 'eqpiv-panel')
    assert cnt[place] == 2 * n_copy and cnt['eqpiv-level'] + cnt['eqpiv-panel'] + cnt['eqpiv-root'] == 2 * n_copy
    res = slv.solve_batch(c.X0[:1], c.P[:1])
    assert res['status'][0] == 0 and slv.trace(8)[1, 7] > 0
    twin = ipm_ref.solve(c.tb, c.X0[0], c.P[0])
    assert twin.status == 0 and twin.iters == res['iters'][0] and np.abs(twin.x - res['x'][0]).max() < 1e-12
    plain = ipm_ref.solve(c.tb, c.X0[0], c.P[0], options={'delta_c_val': 0.0})
    assert plain.status != 0 or plain.iters != res['iters'][0]


def test_coverage_table(emu, capsys):
    """One row per family with the counters of its structure line; every branch of the symbolic
    analysis is reached by some family, every packing limit is met exactly by one and exceeded
    by one step by another."""
    keys = ['N', 'nnz(L)', 'levels', 'root', 'root-mod4', 'eqpiv-level', 'eqpiv-panel', 'eqpiv-root',
            'sn1', 'sn2', 'sn3', 'sn4', 'zeros', 'max-sn-zeros', 'max-col', 'max-gather', 'max-nq',
            'max-slices', 'max-block-rows', 'max-panel-rounds', 'max-back-rounds']
    rows, reasons = {}, set()
    for name in FAMILIES:
        s = solver(case(name).tb).structure
        if s.startswith('envelope'):
            reasons.add(s)
        else:
            rows[name] = sk.parse_counters(s)
    with capsys.disabled():
        print('\n%-16s ' % 'family' + ' '.join('%6s' % k[-6:] for k in keys))
        for name, cnt in rows.items():
            print('%-16s ' % name + ' '.join('%6d' % cnt[k] for k in keys))
    col = {k: [cnt[k] for cnt in rows.values()] for k in keys}
    for k in ('eqpiv-level', 'eqpiv-panel', 'eqpiv-root', 'sn1', 'sn2', 'sn3', 'sn4'):
        assert max(col[k]) > 0, k
    assert set(col['root-mod4']) == {0, 1, 2, 3} and min(col['root']) == 1
    assert max(col['root']) == sk.SP_MAXROOT
    assert max(col['zeros']) == sk.SP_SNZ_TOTAL and max(col['max-sn-zeros']) == sk.SP_SNZ
    assert max(col['max-col']) == sk.SP_MAXCOL and set(range(1, 9)) <= set(col['max-nq'])
    assert max(col['max-gather']) > 2 * (sk.SP_NPF + 4)          # the long-list loop of the gather
    assert max(col['max-slices']) > 32 and max(col['max-block-rows']) == sk.NT
    assert max(col['max-panel-rounds']) > 1 and max(col['max-back-rounds']) > 1
    assert max(col['levels']) > 200 and min(col['levels']) == 0
    assert max(col['N']) == sk.SP_MAXN and max(col['nnz(L)']) == sk.SP_MAXL - 1
    assert {r[len('envelope kernels ('):-1] for r in reasons} == {
        'column structure too long for the packed pairs', 'too many supernodes on one level',
        'factor too large for the packed pairs', 'term degree > 2'}


SCHED_SUBSET = ['chain-short', 'arrow', 'fan-62', 'root-7-eq2', 'blocks-128x2', 'nonconvex', 'dependent-root',
                'singular-panel']


def test_results_do_not_depend_on_the_thread_schedule(emu, monkeypatch):
    """A representative subset under the forward, reverse and random fiber schedules of the
    emulation: bit-identical x, lam_g, f, statuses and iteration counts."""
    out = {}
    for sched in ('forward', 'reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        out[sched] = [solver(case(n).tb).solve_batch(case(n).X0, case(n).P) for n in SCHED_SUBSET]
    for sched in ('reverse', 'random:1'):
        for name, a, b in zip(SCHED_SUBSET, out['forward'], out[sched]):
            for key in ('x', 'lam_g', 'f', 'status', 'iters'):
                assert np.array_equal(a[key], b[key]), (name, sched, key)


MANUFACTURED = [('chain', 40, 6, 4, 4), ('wide', 150, 20, 10, 10), ('root', 12, 4, 3, 2)]
P_MANUFACTURED = np.array([[0.0, 0.0], [0.7, 0.0], [-1.3, 0.0]])


def manufactured(n, n_eq, n_act, n_inact, eq_only=False):
    tb, D = sk.manufactured_qp(n, n_eq, n_act, n_inact, seed=n, eq_only=eq_only)
    X0 = np.zeros((len(P_MANUFACTURED), n))
    xs = D['x0'][None] + P_MANUFACTURED[:, :1] * D['d'][None]
    return tb, D, X0, P_MANUFACTURED, xs


def kkt_inverse_norm(D, x, n_act):
    """||K^-1||_2 of the KKT matrix [[H, J^T], [J, 0]] at x: H the Hessian of the Lagrangian,
    J the equality rows and the gradients of the active rows."""
    n = D['Q'].shape[0]
    H = D['Q'].copy()
    J = [D['A']]
    for i, (vs, Dv, av) in enumerate(D['rows'][:n_act]):
        H[vs, vs] += D['z'][i] * Dv
        g = np.zeros(n)
        g[vs] = Dv * (x[vs] - av)
        J.append(g[None])
    J = np.vstack(J)
    K = np.block([[H, J.T], [J, np.zeros((J.shape[0], J.shape[0]))]])
    return 1.0 / np.linalg.svd(K, compute_uv=False).min()


def check_manufactured(n, n_eq, n_act, n_inact):
    """x and the multipliers to 10 ||K^-1|| tol / min(1, z_min) of x*(p), y, z; returns (error
    in x, bound, error in the multipliers)."""
    tb, D, X0, P, xs = manufactured(n, n_eq, n_act, n_inact)
    res = solver(tb, TIGHT).solve_batch(X0, P)
    assert (res['status'] == 0).all(), res['status']
    kinv = max(kkt_inverse_norm(D, x, n_act) for x in xs)
    bound = 10 * kinv * TIGHT['tol'] / min(1.0, D['z'][:n_act].min())
    err = np.abs(res['x'] - xs).max()
    assert err < bound, (err, bound)
    dl = max(np.abs(res['lam_g'][:, :n_eq] - D['y'][None]).max(),
             np.abs(res['lam_g'][:, n_eq:n_eq + n_act] - D['z'][None, :n_act]).max())
    assert dl < bound, (dl, bound)
    return err, bound, dl


@pytest.mark.parametrize('label, n, n_eq, n_act, n_inact', MANUFACTURED)
def test_manufactured_qp_optimum(emu, label, n, n_eq, n_act, n_inact):
    """Strictly convex QPs with linear equality rows and convex quadratic rows whose KKT point
    (x*(p) = x0 + p_0 d, the multipliers, the active set) is fixed by construction
    (synthetic_kkt.manufactured_qp), solved at tol = 1e-8.  When the interior-point run stops,
    the KKT residuals are below tol and so is the complementarity s_i z_i: an active row is off
    by about tol / z_i, and the iterate by at most ||K^-1|| times the residual, K the KKT matrix
    at the optimum; the multipliers likewise.  Asserted for both: 10 ||K^-1|| tol / min(1, z_min),
    1.4e-6 .. 1.0e-5 here; measured 1.1e-8 .. 2.3e-8 in x and 1.1e-7 .. 3.9e-7 in the multipliers
    (the same on an H100)."""
    check_manufactured(n, n_eq, n_act, n_inact)


def mp_kkt_solution(D, p0, dps=50):
    """x of the equality-only QP  min 0.5 x^T Q x + (c0 + p0 c1)^T x, A x = A (x0 + p0 d)
    from its KKT system, in mpmath at ``dps`` digits."""
    import mpmath
    mpmath.mp.dps = dps
    Q, A = D['Q'], D['A']
    n, k = Q.shape[0], A.shape[0]
    K = mpmath.matrix(n + k, n + k)
    rhs = mpmath.matrix(n + k, 1)
    for i in range(n):
        for j in range(n):
            K[i, j] = mpmath.mpf(Q[i, j])
        rhs[i] = -(mpmath.mpf(D['c0'][i]) + mpmath.mpf(p0) * mpmath.mpf(D['c1'][i]))
    for r in range(k):
        for j in range(n):
            K[n + r, j] = K[j, n + r] = mpmath.mpf(A[r, j])
        rhs[n + r] = sum(mpmath.mpf(A[r, j]) * (mpmath.mpf(D['x0'][j]) + mpmath.mpf(p0) * mpmath.mpf(D['d'][j]))
                         for j in range(n))
    sol = mpmath.lu_solve(K, rhs)
    return np.array([float(sol[i]) for i in range(n)])


def check_equality_qp(x_tol):
    tb, D, X0, P, xs = manufactured(30, 8, 0, 0, eq_only=True)
    res = solver(tb, TIGHT).solve_batch(X0, P)
    assert (res['status'] == 0).all()
    ref = np.array([mp_kkt_solution(D, p[0]) for p in P])
    assert np.abs(ref - xs).max() < 1e-14               # the construction is exact
    err = np.abs(res['x'] - ref).max()
    assert err < x_tol, err
    return err


def test_equality_qp_matches_the_mpmath_kkt_solution(emu):
    """An equality-only convex QP is solved by one Newton step of its KKT system: the kernel's x
    against that system solved in mpmath at 50 digits.  ||K^-1|| is 1.1 here and the solve is
    backward stable, so x is right to a few ulps of ||x|| times ||K|| ||K^-1||: asserted 1e-12,
    measured 8.9e-16 (the same on an H100)."""
    check_equality_qp(1e-12)


# ---------------------------------------------------------------------------------------
# the device kernels
# ---------------------------------------------------------------------------------------
def mixed_bounds(tb, B):
    """Per-instance bounds: the inequality rows upper-only as lowered (b % 3 == 0), with the
    upper bound raised by 0.5 (b % 3 == 1), two-sided [-10, ubg] (b % 3 == 2)."""
    LB, UB = np.repeat(tb.lbg[None], B, 0), np.repeat(tb.ubg[None], B, 0)
    ineq = tb.lbg != tb.ubg
    for b in range(B):
        if b % 3 == 1:
            UB[b, ineq] += 0.5
        elif b % 3 == 2:
            LB[b, ineq] = -10.0
    return LB, UB


def gpu_batches(c, slv):
    """(X0, P, LB, UB) at batch 1, at one instance more than the resident blocks, and with mixed
    per-instance bounds."""
    info = slv.info()
    B = info['ctas_per_sm'] * info['n_sm'] + 1
    X1, P1 = sk.instances(c.tb, 6, seed=1)
    LB, UB = mixed_bounds(c.tb, 6)
    return [(c.X0[:1], c.P[:1], None, None, None),
            (np.resize(X1, (B, c.tb.n)), np.resize(P1, (B, 2)), None, None, 6), (X1, P1, LB, UB, None)]


@pytest.mark.gpu
@pytest.mark.parametrize('name', list(FAMILIES))
def test_gpu_family_matches_the_oracle(gpu, snw, name):
    """Every family on the device, default width and OMG_B200_SNW=1, at batch 1, at one instance
    more than the resident blocks (blocks take a second instance) and with mixed per-instance
    bounds: statuses and iteration counts of the C oracle, x and f to 1e-12, lam_g to 1e-10; the
    rounded dependent rows x to 1e-8, the sums of their multipliers to 1e-6.  The large batch
    repeats six instances; the oracle solves those six.  Measured on an H100 80GB HBM3 (700 W
    power limit, 1980 MHz): x within 8.4e-15 and lam_g within 6.7e-16 of the oracle on every
    family but the rounded dependent rows, there 1.1e-9 and 1.0e-10 -- as far as the oracle's
    dense and sparse arms are from each other."""
    c = case(name)
    slv = solver(c.tb)
    check_structure(c, slv.structure, snw)
    worst = worst_l = 0.0
    for X0, P, LB, UB, tile in gpu_batches(c, slv):
        _, _, devs = check_family(name, snw, 1e-12, X0, P, LB, UB, tile)
        worst = max([worst] + [d[0] for d in devs])
        worst_l = max([worst_l] + [d[1] for d in devs])
    print('\n[max |dx|] %s %s %.2e %.2e' % (name, snw or 'default', worst, worst_l))


@pytest.mark.gpu
@pytest.mark.parametrize('label, n, n_eq, n_act, n_inact', MANUFACTURED)
def test_gpu_manufactured_qp_optimum(gpu, label, n, n_eq, n_act, n_inact):
    err, bound, dl = check_manufactured(n, n_eq, n_act, n_inact)
    print('\n[manufactured] %s err %.2e lam %.2e bound %.2e' % (label, err, dl, bound))


@pytest.mark.gpu
def test_gpu_equality_qp_matches_the_mpmath_kkt_solution(gpu):
    print('\n[mpmath] err %.2e' % check_equality_qp(1e-12))
