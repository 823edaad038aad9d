"""The envelope solver kernels (omg_ipm_kernel, _2cta, _xl, _xl_2cta) on synthetic KKT
structures (tests/envelope_kkt.py) that reach every panel shape of factor_env and
back_solve_env, every shared-memory layout that omg_problem_create chooses and every
intermediate-derivative path of the XL kernel, against the C oracle.

Each family is forced onto the envelope kernels (OMG_B200_KERNEL=envelope), some with one block
of 512 threads per SM (OMG_B200_CTAS=1) or inertia_mode = 1.  The envelope layout
(B200Solver.envelope_layout) shows that each family hits the layout and panel shape it is meant
for; the tables show the rest (panel row counts, equality-pivot positions, intermediate lists).

The tests without a mark run the kernel source on the CPU (tools/cpu_emu); the ones marked gpu
run the same cases through the product library on the device."""
import os
import sys

import numpy as np
import pytest

from oracle import ipm_c

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emu_support                       # noqa: E402
import envelope_kkt as ek                # noqa: E402
import synthetic_kkt as sk               # noqa: E402
import test_sparse_structures as ts      # noqa: E402

FAMILIES = ek.families()
MID = [n for n in FAMILIES if n.startswith('mid-')]
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


@pytest.fixture
def envelope(monkeypatch):
    """Sets the environment of a family (the envelope kernels, the block size) for the solvers
    created after the call."""
    def use(c):
        monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
        if c.ctas:
            monkeypatch.setenv('OMG_B200_CTAS', c.ctas)
        else:
            monkeypatch.delenv('OMG_B200_CTAS', raising=False)
        return c
    return use


def check_layout(c, slv):
    """The family runs on the envelope kernels and hits its layout: fields equal to a value, or
    counters within (lo, hi)."""
    assert slv.structure == 'envelope kernels (forced)', slv.structure
    lay = ek.parse_layout(slv.envelope_layout)
    assert lay['wide'] == int(lay['max-panel-rows'] + 2 > lay['nt']), slv.envelope_layout
    for key, want in c.target.items():
        if not isinstance(want, tuple):
            assert lay[key] == want, (key, slv.envelope_layout)
        else:
            lo, hi = want
            assert lay[key] >= lo and (hi is None or lay[key] <= hi), (key, slv.envelope_layout)
    return lay


def oracles(c, X0, P, lbg=None, ubg=None):
    """The C oracle's dense arm (envelope order, small structures) and its sparse arm (minimum-
    degree order; inertia_mode = 1 ties the pivot signs to the envelope order, so not there)."""
    out = []
    if c.tb.kkt_n <= ts.DENSE_ORACLE_MAX_N:
        out.append(ipm_c.solve_batch_full(c.tb, X0, P, threads=8, options=dict(c.options), lbg=lbg, ubg=ubg))
    if not c.options.get('inertia_mode'):
        out.append(ipm_c.solve_batch_full(c.tb, X0, P, threads=8, lbg=lbg, ubg=ubg,
                                          options=dict(c.options, linear_solver='sparse')))
    assert out
    return out


def check_family(name, x_tol, X0=None, P=None, lbg=None, ubg=None, tile=None):
    """``tile``: X0 and P repeat their first ``tile`` instances; the oracle solves those."""
    c = case(name)
    slv = ts.solver(c.tb, c.options)
    check_layout(c, slv)
    X0 = c.X0 if X0 is None else X0
    P = c.P if P is None else P
    res = slv.solve_batch(X0, P, lbg, ubg)
    assert (res['status'] == 0).all(), res['status']
    refs = oracles(c, X0[:tile], P[:tile], lbg, ubg) if tile else oracles(c, X0, P, lbg, ubg)
    if tile:
        refs = [{k: np.resize(v, (len(X0),) + v.shape[1:]) for k, v in r.items()} for r in refs]
    devs = [ts.match(res, ref, c.x_tol or x_tol, dup=c.dup) for ref in refs]
    return slv, res, devs


# ---------------------------------------------------------------------------------------
# emulated kernels (CPU)
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(FAMILIES))
def test_family_matches_the_oracle(emu, envelope, name):
    """Every family hits its layout and matches the C oracle's dense arm (N <= 400) and its
    sparse arm (inertia_mode = 0): statuses and iteration counts identical, x and f to 1e-12,
    lam_g to 1e-10; the rounded dependent equality rows of synthetic_kkt x to 1e-8 and the sum of
    the two rows' multipliers to 1e-6.  The 'dense-*' families are the panels that reach more
    rows than the block has threads: before factor_env solved such panels in a strided loop,
    'dense-293' (293 rows, 256 threads) failed with status 3 at iteration 0.  Measured: x within
    5.8e-15 and lam_g within 4.4e-16 of the oracle, the rounded dependent rows 1.1e-9 and 1.2e-10."""
    envelope(case(name))
    _, _, devs = check_family(name, 1e-12)
    print('\n[max |dx|] %s %.2e %.2e' % (name, max(d[0] for d in devs), max(d[1] for d in devs)))


def check_unlowered(name):
    """The KKT conditions at the returned (x, lam_g) from the un-lowered rows; returns the
    largest dual residual and constraint violation."""
    c = case(name)
    res = ts.solver(c.tb, ts.TIGHT).solve_batch(c.X0, c.P)
    assert (res['status'] == 0).all(), res['status']
    worst = [0.0, 0.0]
    for x, p, lam in zip(res['x'], c.P, res['lam_g']):
        dual, viol = ek.unlowered_kkt(c.nlp, x, p, lam)
        # the stopping test: the scaled dual infeasibility ||grad f + J^T lam|| / s_d below tol,
        # s_d = max(100, sum |multipliers| / (n + m)) / 100 (slack multipliers count twice);
        # the violation below constr_viol_tol on bounds relaxed by bound_relax_factor
        ineq = c.tb.lbg != c.tb.ubg
        s_d = max(100.0, (np.abs(lam).sum() + np.abs(lam[ineq]).sum()) / (c.tb.n + c.tb.m)) / 100.0
        assert dual <= s_d * ts.TIGHT['tol'], (dual, s_d)
        assert viol <= ts.TIGHT['constr_viol_tol'] + 1e-8 * max(1.0, np.abs(c.tb.ubg[ineq]).max()), viol
        worst = [max(worst[0], dual), max(worst[1], viol)]
    return worst


@pytest.mark.parametrize('name', MID)
def test_intermediates_satisfy_the_unlowered_kkt_conditions(emu, envelope, name):
    """An end-to-end reference for the XL kernel's chain rule that does not use the lowered
    tables: the rows with every mid replaced by its definition, differentiated symbolically,
    at the x and lam_g the kernel returns (tol = 1e-8).  ||grad f + J^T lam||_inf is below
    s_d tol (the stopping test, s_d = 1 here) and the constraint violation below
    constr_viol_tol + the bound relaxation (2e-8).  Measured: dual 2.3e-14 .. 1.1e-9 (the mid
    in 40 rows), violation at most 4.6e-11."""
    envelope(case(name))
    dual, viol = check_unlowered(name)
    print('\n[unlowered] %s dual %.2e viol %.2e' % (name, dual, viol))


@pytest.mark.parametrize('label, n, n_eq, n_act, n_inact', ts.MANUFACTURED)
def test_manufactured_qp_optimum(emu, monkeypatch, label, n, n_eq, n_act, n_inact):
    """test_sparse_structures.test_manufactured_qp_optimum on the envelope kernels: x and the
    multipliers within 10 ||K^-1|| tol / min(1, z_min) of the constructed optimum."""
    monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    ts.check_manufactured(n, n_eq, n_act, n_inact)


def test_equality_qp_matches_the_mpmath_kkt_solution(emu, monkeypatch):
    """test_sparse_structures.test_equality_qp_matches_the_mpmath_kkt_solution on the envelope
    kernels: x against the KKT system solved in mpmath at 50 digits, to 1e-12."""
    monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    ts.check_equality_qp(1e-12)


@pytest.mark.parametrize('name', ['sk-nonconvex', 'sk-nonconvex@inertia1', 'sk-singular-panel',
                                  'sk-singular-panel@inertia1'])
def test_inertia_correction_runs(emu, envelope, name):
    """Negative curvature (more negative pivots than equality rows: inertia_mode = 0 stops the
    factorisation early; inertia_mode = 1 fails at the first pivot of the wrong sign) and an
    exactly singular copy of an equality row (delta_c) make the factorisation fail and the
    inertia correction run: delta_w > 0 (the trace's last column) in at least one iteration of
    instance 0 -- with the oracle's statuses and iteration counts (test_family_matches_the_oracle)."""
    c = envelope(case(name))
    slv = ts.solver(c.tb, dict(c.options, trace=1))
    res = slv.solve_batch(c.X0[:1], c.P[:1])
    assert res['status'][0] == 0
    assert (slv.trace(512)[:res['iters'][0] + 1, 7] > 0).any()


SCHED_SUBSET = ['nmod8-3', 'tiny-5', 'blocks-diag', 'dense-257', 'many-rows', 'tape-k-shared', 'mid-xmid',
                'mid-midmid', 'mid-shared', 'sk-singular-panel', 'nmod8-5@inertia1', 'band-4@ctas1']


def test_results_do_not_depend_on_the_thread_schedule(emu, envelope, monkeypatch):
    """A subset under the forward, reverse and random fiber schedules of the emulation:
    bit-identical x, lam_g, f, statuses and iteration counts."""
    out = {}
    for sched in ('forward', 'reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        out[sched] = []
        for n in SCHED_SUBSET:
            c = envelope(case(n))
            out[sched].append(ts.solver(c.tb, c.options).solve_batch(c.X0, c.P))
    for sched in ('reverse', 'random:1'):
        for name, a, b in zip(SCHED_SUBSET, out['forward'], out[sched]):
            for key in ('x', 'lam_g', 'f', 'status', 'iters'):
                assert np.array_equal(a[key], b[key]), (name, sched, key)


def test_coverage_table(emu, envelope, capsys):
    """One row per family with its layout and table counters; every panel shape, layout and
    intermediate path is reached by some family."""
    rows = {}
    for name in FAMILIES:
        c = envelope(case(name))
        lay = ek.parse_layout(ts.solver(c.tb, c.options).envelope_layout)
        rows[name] = dict(lay, **ek.table_counters(c.tb))
        rows[name]['inertia'] = c.options.get('inertia_mode', 0)
    keys = ['kernel', 'nt', 'K', 'V', 'arrays-in-scratch', 'N', 'N%8', 'max-panel-rows', 'min-panel-rows', 'wide',
            'odd-rows', 'even-rows', 'pcmin>0', 'eqpiv-last-partial', 'n_jxvar', 'max-mu', 'nnz_wx', 'xq_b<0',
            'xq_b>=0', 'chain-only', 'eq-mid-slots']
    with capsys.disabled():
        print('\n%-26s ' % 'family' + ' '.join('%8s' % k[-8:] for k in keys))
        for name, r in rows.items():
            print('%-26s ' % name + ' '.join('%8s' % r.get(k, '-') for k in keys))
    R = list(rows.values())
    # panel shapes
    assert {r['N%8'] for r in R} == set(range(8)) and min(r['N'] for r in R) < ek.NB
    assert any(r['min-panel-rows'] == 1 and r['N'] > ek.NB for r in R)
    assert any(r['odd-rows'] for r in R) and any(r['even-rows'] for r in R) and any(r['pcmin>0'] for r in R)
    at256 = {r['max-panel-rows'] for r in R if r['nt'] == ek.NT2}
    assert {ek.NT2 - 1, ek.NT2, ek.NT2 + 1} <= at256 and max(at256) > ek.NT2 + 32
    assert max(r['max-panel-rows'] for r in R if r['nt'] == ek.NT1) > ek.NT1
    assert {r['wide'] for r in R} == {0, 1}            # the strided panel solve of factor_env<true>
    # equality pivots at every position of a diagonal block and in a partial last panel, in
    # both inertia modes
    for mode in (0, 1):
        assert set().union(*[r['eqpiv-mod8'] for r in R if r['inertia'] == mode]) == set(range(ek.NB))
        assert any(r['eqpiv-last-partial'] for r in R if r['inertia'] == mode)
    # layouts
    lays = {(r['kernel'], r['nt'], r['K'], r['V']) for r in R}
    assert {('standard', ek.NT2, 'shared', 'shared'), ('standard', ek.NT1, 'shared', 'shared')} <= lays
    assert any(r['kernel'] == 'standard' and r['arrays-in-scratch'] > ek.N_ARR_LOW for r in R)
    assert {(r['K'], r['V']) for r in R if r['kernel'] == 'xl' and not r['n_mid']} == {
        ('shared', 'scratch'), ('scratch', 'shared'), ('scratch', 'scratch')}
    assert any(r['kernel'] == 'xl' and r['K'] == r['V'] == 'shared' for r in R)   # (with intermediates)
    # intermediates
    M = [r for r in R if r['n_mid']]
    assert min(r['n_jxvar'] for r in M) == 0 and max(r['n_jxvar'] for r in M) > 0
    assert max(r['max-mu'] for r in M) >= 40 and min(r['chain-only'] for r in M) > 0
    assert min(r['eq-mid-slots'] for r in M) > 0
    assert max(r['xq_b<0'] for r in M) > 0 and max(r['xq_b>=0'] for r in M) > 0


# ---------------------------------------------------------------------------------------
# the device kernels
# ---------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('name', list(FAMILIES))
def test_gpu_family_matches_the_oracle(gpu, envelope, name):
    """Every family on the device at batch 1, at one instance more than the resident blocks
    (blocks take a second instance) and with mixed per-instance bounds: statuses and iteration
    counts of the C oracle, x and f to 1e-12, lam_g to 1e-10; the rounded dependent rows x to
    1e-8, the sums of their multipliers to 1e-6.  The large batch repeats six instances; the
    oracle solves those six.  The exactly singular copies of synthetic_kkt.singular_blocks: x to
    1e-5.  Their second pivot is exactly zero only where 1/sqrt is correctly rounded (the oracle,
    the emulation); the device's rsqrt is not, so there the copy is a rounded dependent row and
    the run, with the oracle's statuses and iteration counts, ends elsewhere within the stopping
    tolerance.  Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz): x within 1.2e-14 and
    lam_g within 4.4e-16 of the oracle; the rounded dependent rows 1.1e-9 and 1.1e-10; the singular
    copies 1.5e-10 (panel) and 7.3e-6 (root; the sum of the two multipliers 2.0e-5)."""
    c = envelope(case(name))
    slv = ts.solver(c.tb, c.options)
    check_layout(c, slv)
    x_tol = 1e-5 if name.split('@')[0][len('sk-'):] in sk.SINGULAR else 1e-12
    worst = worst_l = 0.0
    for X0, P, LB, UB, tile in ts.gpu_batches(c, slv):
        _, _, devs = check_family(name, x_tol, X0, P, LB, UB, tile)
        worst = max([worst] + [d[0] for d in devs])
        worst_l = max([worst_l] + [d[1] for d in devs])
    print('\n[max |dx|] %s %.2e %.2e' % (name, worst, worst_l))


@pytest.mark.gpu
@pytest.mark.parametrize('name', MID)
def test_gpu_intermediates_satisfy_the_unlowered_kkt_conditions(gpu, envelope, name):
    envelope(case(name))
    dual, viol = check_unlowered(name)
    print('\n[unlowered] %s dual %.2e viol %.2e' % (name, dual, viol))


@pytest.mark.gpu
@pytest.mark.parametrize('label, n, n_eq, n_act, n_inact', ts.MANUFACTURED)
def test_gpu_manufactured_qp_optimum(gpu, monkeypatch, label, n, n_eq, n_act, n_inact):
    monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    err, bound, dl = ts.check_manufactured(n, n_eq, n_act, n_inact)
    print('\n[manufactured] %s err %.2e lam %.2e bound %.2e' % (label, err, dl, bound))


@pytest.mark.gpu
def test_gpu_equality_qp_matches_the_mpmath_kkt_solution(gpu, monkeypatch):
    monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    print('\n[mpmath] err %.2e' % ts.check_equality_qp(1e-12))
