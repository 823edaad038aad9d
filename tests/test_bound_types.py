"""Lower-bounded, two-sided and free constraint rows through the solver kernels.

Each row gets a type in the kernels' setup: bit 1 lower bound, bit 2 upper bound, bit 4
equality (omg_sp.cuh sp_setup).  The lower bound, z_L, the two-sided starting-point push
and the log(s - s_L) barrier term are used only for rows that have them, and every scenario
of the suite lowers to equality and upper-only rows.  The variants of tests/bound_variants.py
rebuild those scenarios with the same rows under the other bound kinds; the kernels are
compared with the C oracle (oracle/ipm.c) and the numpy twin (oracle/ipm_ref.py).

The tests without a mark run the kernel source on the CPU (tools/cpu_emu, as
tests/test_kernel_emulation.py); the ones marked gpu run the same cases through the
product library on the device."""
import os
import sys

import numpy as np
import pytest

from omg_tools_b200 import scenarios as sc
from oracle import ipm_c, ipm_ref

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bound_variants as bv              # noqa: E402
import emu_support                       # noqa: E402

TIGHT = {'tol': 1e-8, 'compl_inf_tol': 1e-8, 'constr_viol_tol': 1e-8}
MIRROR_MODELS = ['config1', 'config2', 'config5', 'config_freeT', 'config_quadrotor2d']
# non-default starting-point and relaxation options (IPOPT's names), one set per case
BOUND_OPTIONS = [{'bound_push': 1e-2, 'bound_frac': 0.2},
                 {'mult_bound_push': 1e-1},
                 {'bound_relax_factor': 1e-6},
                 {'bound_relax_factor': 0.0},
                 {'bound_push': 0.05, 'bound_frac': 0.05, 'mult_bound_push': 1e-2,
                  'bound_relax_factor': 1e-7}]


@pytest.fixture
def emu():
    """The emulated kernels for the solvers built inside one test (function scope, so that the
    gpu tests of this module always bind the product library)."""
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


_SCENARIOS = {}


def scenario(name):
    """The scenario with its lowered tables (no solver: every test builds its own)."""
    if name not in _SCENARIOS:
        _SCENARIOS[name] = getattr(sc, name)(build_solver=False)
    return _SCENARIOS[name]


def _same(a, b, keys=('x', 'f', 'status', 'iters')):
    for key in keys:
        assert np.array_equal(a[key], b[key]), key


def _match_oracle(res, ref, x_tol, lam_tol=None, hp_tol=None):
    """Identical statuses and iteration counts, the vehicle splines (the first 26 variables) to
    x_tol, the other variables to hp_tol (default x_tol) and lam_g to lam_tol.  The separating
    hyperplanes are not unique at the optimum: there the iteration amplifies rounding."""
    assert np.array_equal(res['status'], ref['status']), (res['status'], ref['status'])
    assert np.array_equal(res['iters'], ref['iters']), (res['iters'], ref['iters'])
    dx = np.abs(res['x'] - ref['x'])
    assert dx[:, :26].max() < x_tol, dx[:, :26].max()
    assert dx.max() < (hp_tol or x_tol), dx.max()
    if lam_tol is not None:
        dl = np.abs(res['lam_g'] - ref['lam_g']).max()
        assert dl < lam_tol, dl


# ---------------------------------------------------------------------------------------
# the cases, shared by the emulated and the device runs
# ---------------------------------------------------------------------------------------
def check_mirror(monkeypatch, name, sel, kernel, x_tol=0.0):
    """The mirrored NLP (sel = every other / every inequality row as -g >= -u) against the
    original through the kernel ``kernel`` ('default' = the solver's choice); x_tol = 0:
    bit for bit, with lam_g negated on the mirrored rows."""
    if kernel == 'envelope':
        monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    pr = scenario(name)
    tb = pr.father.tables
    tbm, idx = bv.mirror(pr, sel)
    n_eq, n_up, n_lo, n_two, n_free = bv.row_type_counts(tbm.lbg, tbm.ubg)
    assert n_lo == len(idx) and n_two == n_free == 0
    assert n_up == (0 if sel == 'all' else tb.m - n_eq - len(idx))
    X0, P = sc.instance_data(pr, 2, jitter=0.1, seed=1)
    a = bv.solver(pr, tb).solve_batch(X0, P)
    b = bv.solver(pr, tbm).solve_batch(X0, P)
    assert (a['status'] == 0).all()
    sign = np.ones(tb.m)
    sign[idx] = -1.0
    assert np.array_equal(a['status'], b['status']) and np.array_equal(a['iters'], b['iters'])
    if x_tol == 0.0:
        _same(a, b)
        assert np.array_equal(b['lam_g'], a['lam_g'] * sign)
    else:
        assert np.abs(a['x'] - b['x']).max() < x_tol
        assert np.abs(a['f'] - b['f']).max() < x_tol
        assert np.abs(b['lam_g'] - a['lam_g'] * sign).max() < 1e3 * x_tol
    return a, b, tbm, sign, X0, P


def check_bands(w, x_tol, lam_tol):
    """Two-sided rows [min(g(x*), u) - w, u] around each instance's solution x* of the
    unchanged config 1 on instances 0, 2 and 3; instance 1 keeps its upper-only rows in the
    same launch."""
    pr = scenario('config1')
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 4, jitter=0.1, seed=1)
    slv = bv.solver(pr, tb)
    a = slv.solve_batch(X0, P)
    LB, UB = bv.band(tb, a['x'], P, w, instances=[0, 2, 3])
    assert bv.row_type_counts(LB[0], UB[0]) == (10, 0, 0, 315, 0)
    assert bv.row_type_counts(LB[1], UB[1]) == (10, 315, 0, 0, 0)
    res = slv.solve_batch(X0, P, LB, UB)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=4, lbg=LB, ubg=UB)
    assert (ref['status'] == 0).all()
    _match_oracle(res, ref, x_tol, lam_tol)
    for key in ('x', 'lam_g', 'f', 'status', 'iters'):       # the one-sided instance
        assert np.array_equal(res[key][1], a[key][1]), key
    return pr, tb, slv, a, res, ref, LB, UB, X0, P


def check_free_rows(x_tol):
    """Rows with slack at the solution are free in instances 1 and 3 only."""
    pr = scenario('config1')
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 4, jitter=0.1, seed=1)
    slv = bv.solver(pr, tb)
    a = slv.solve_batch(X0, P)
    LB, UB, free = bv.free_rows(tb, a['x'], P, [1, 3])
    assert free[1].sum() > 50 and free[3].sum() > 50 and not free[[0, 2]].any()
    assert bv.row_type_counts(LB[1], UB[1])[4] == free[1].sum()
    res = slv.solve_batch(X0, P, LB, UB)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=4, lbg=LB, ubg=UB)
    assert (ref['status'] == 0).all()
    _match_oracle(res, ref, x_tol)
    assert (res['lam_g'][free] == 0.0).all()                 # y of a free row never moves
    for b in (0, 2):                                         # the instances with all bounds
        assert np.array_equal(res['x'][b], a['x'][b]) and res['iters'][b] == a['iters'][b]


def check_mixed(name, B, w, x_tol, hp_tol=None, threads=4, tile=None):
    """mixed_types(): per instance, each inequality row upper-only, two-sided, lower-only or
    free, the type of a row changing from one instance to the next.  ``tile`` > 0 repeats that
    many distinct instances up to the batch size B."""
    pr = scenario(name)
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, tile or B, jitter=0.1, seed=1)
    if tile:
        X0, P = np.resize(X0, (B, tb.n)), np.resize(P, (B, tb.n_par))
    slv = bv.solver(pr, tb)
    a = slv.solve_batch(X0, P)
    assert (a['status'] == 0).all()
    LB, UB = bv.mixed_types(tb, a['x'], P, w)
    counts = np.array([bv.row_type_counts(LB[b], UB[b]) for b in range(min(B, 4))])
    assert (counts[:, 1:] > 0).all()                         # every row type in every instance
    res = slv.solve_batch(X0, P, LB, UB)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=threads, lbg=LB, ubg=UB)
    assert (ref['status'] == 0).all()
    _match_oracle(res, ref, x_tol, hp_tol=hp_tol)


def check_warm_start(variant, x_tol, hp_tol):
    """lam_g0 from a previous solution of the original, the mirrored (multipliers of both
    signs, both one-sided bound kinds) or the banded problem (two-sided rows): statuses,
    iteration counts and x as the oracle, restarting both from the solution and from other
    starting points.  The scaled rows of config 1 (48 rows with gradients above 100) take
    lam0 * fsc / d."""
    pr = scenario('config1')
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 4, jitter=0.1, seed=1)
    LB = UB = None
    if variant == 'mirror':
        tb, _ = bv.mirror(pr, 'alternate')
    slv = bv.solver(pr, tb)
    if variant == 'band':
        LB, UB = bv.band(tb, slv.solve_batch(X0, P)['x'], P, 0.1, instances=[0, 2, 3])
    c = slv.solve_batch(X0, P, LB, UB)
    assert (c['status'] == 0).all()
    lam, ineq = c['lam_g'], tb.lbg != tb.ubg
    # upper-only rows: lam >= 0; lower-bounded rows carry negative multipliers as well
    assert (lam[:, ineq] > 1e-6).any() and ((lam[:, ineq] < -1e-6).any() == (variant != 'original'))
    X1 = sc.instance_data(pr, 4, jitter=0.1, seed=2)[0]
    for x0 in (c['x'], X1):
        w = slv.solve_batch(x0, P, LB, UB, lam_g0=lam)
        ref = ipm_c.solve_batch_full(tb, x0, P, threads=4, lbg=LB, ubg=UB, lam_g0=lam)
        assert (ref['status'] == 0).all()
        _match_oracle(w, ref, x_tol, hp_tol=hp_tol)
    assert (w['iters'] != slv.solve_batch(X1, P, LB, UB)['iters']).any()   # lam0 is used


def check_bound_options(opts, x_tol):
    """Non-default bound_push / bound_frac / mult_bound_push / bound_relax_factor on config 1
    with bands of width 0.1 (instances 0, 2, 3) and upper-only rows (instance 1)."""
    pr = scenario('config1')
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 4, jitter=0.1, seed=1)
    x_ref = bv.solver(pr, tb).solve_batch(X0, P)['x']
    LB, UB = bv.band(tb, x_ref, P, 0.1, instances=[0, 2, 3])
    res = bv.solver(pr, tb, opts).solve_batch(X0, P, LB, UB)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=4, options=opts, lbg=LB, ubg=UB)
    assert (ref['status'] == 0).all()
    _match_oracle(res, ref, x_tol)


# ---------------------------------------------------------------------------------------
# emulated kernels (CPU)
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('sel', ['alternate', 'all'])
@pytest.mark.parametrize('name', MIRROR_MODELS)
def test_mirrored_rows_give_the_same_iterates(emu, monkeypatch, name, sel):
    """Rows g <= u rewritten as -g >= -u (every other inequality row, or all of them: then no
    row has an upper bound only and z_U is never loaded) through the kernel the solver picks
    (the sparse kernel; the envelope kernel for config_freeT, whose rows have degree 3), the
    forced envelope kernel, the C oracle and the numpy twin: x, f, statuses and iteration
    counts bit for bit as the original NLP, lam_g negated on the mirrored rows.  config_freeT
    takes the soft restoration, config_quadrotor2d indefinite pivots."""
    a, b, tbm, sign, X0, P = check_mirror(monkeypatch, name, sel, 'default')
    e = check_mirror(monkeypatch, name, sel, 'envelope')[0]
    tb = scenario(name).father.tables
    r0 = ipm_c.solve_batch_full(tb, X0, P, threads=2)
    r1 = ipm_c.solve_batch_full(tbm, X0, P, threads=2)
    _same(r0, r1)
    assert np.array_equal(r1['lam_g'], r0['lam_g'] * sign)
    assert np.array_equal(r0['iters'], a['iters']) and np.array_equal(r0['iters'], e['iters'])
    t0 = ipm_ref.solve(tb, X0[0], P[0])
    t1 = ipm_ref.solve(tbm, X0[0], P[0])
    assert t0.status == t1.status == 0 and t0.iters == t1.iters == a['iters'][0]
    assert np.array_equal(t0.x, t1.x) and np.array_equal(t1.lam_g, t0.lam_g * sign)


@pytest.mark.parametrize('w', [1e3, 1e-1, 1e-3])
def test_two_sided_bands_match_the_oracle(emu, w):
    """Bands of width w = 1e3 (the upper bound decides), 1e-1 and 1e-3 (narrow: the two-sided
    push min(bound_push * max(1, |l|), bound_frac * (u - l)) sets the starting slacks): the
    statuses and iteration counts of the C oracle, x to 1e-9 (measured 3e-12); the one-sided
    instance bit for bit as without the bands."""
    check_bands(w, 1e-9, 1e-8)


def test_narrow_bands_take_the_feasibility_fallback(emu):
    """At w = 1e-3 the line search of the banded instances fails (Restoration_Failed: the restart
    push of DESIGN.md section 8 moves the slacks across the narrow rows).  Without the
    feasibility phase the emulated kernel, the C oracle and the numpy twin end there alike;
    with the default options solve_batch runs omg_feas_batch and solves again, as the oracle
    does, and every instance succeeds."""
    check_narrow_bands(twin=True)


def check_narrow_bands(twin):
    pr, tb, slv, a, res, ref, LB, UB, X0, P = check_bands(1e-3, 1e-9, 1e-8)
    plain = ipm_c.solve_batch_full(tb, X0, P, threads=4, lbg=LB, ubg=UB, options={'feas_steps': 0})
    assert list(plain['status']) == [2, 0, 2, 2]
    slv.set_options({'feas_steps': 0})
    off = slv.solve_batch(X0, P, LB, UB)
    _match_oracle(off, plain, 1e-9)
    for b in ((0, 2, 3) if twin else ()):
        t = ipm_ref.solve(tb, X0[b], P[b], LB[b], UB[b])
        assert t.status == 2 and t.iters == plain['iters'][b]
        assert np.abs(t.x - plain['x'][b]).max() < 1e-9
    assert (res['iters'][[0, 2, 3]] > plain['iters'][[0, 2, 3]]).all()   # the fallback ran


def test_wide_bands_keep_the_solution_at_tight_tolerance(emu):
    """Bands 1e3 wide leave the optimum where it was: at tol = 1e-8 the vehicle splines of the
    banded instances equal those of the upper-only problem."""
    check_wide_bands_tight()


def check_wide_bands_tight():
    pr = scenario('config1')
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 2, jitter=0.1, seed=2)
    slv = bv.solver(pr, tb, TIGHT)
    a = slv.solve_batch(X0, P)
    LB, UB = bv.band(tb, a['x'], P, 1e3)
    res = slv.solve_batch(X0, P, LB, UB)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=2, options=TIGHT, lbg=LB, ubg=UB)
    assert (a['status'] == 0).all() and (res['status'] == 0).all()
    _match_oracle(res, ref, 1e-9)
    assert np.abs(res['x'] - a['x'])[:, :26].max() < 1e-7


def test_rows_free_in_some_instances(emu):
    """Free rows (-inf, +inf) in two of four instances: the C oracle instance by instance,
    zero multipliers on the free rows, and the other instances as without free rows."""
    check_free_rows(1e-9)


@pytest.mark.parametrize('name, w, hp_tol', [('config1', 1.0, None), ('config1', 0.1, None),
                                             ('config2', 0.1, 1e-4)])
def test_row_types_mixed_across_instances(emu, name, w, hp_tol):
    """Upper-only, two-sided, lower-only and free rows in one launch, every row changing type
    between instances: the C oracle instance by instance -- statuses, iteration counts, the
    vehicle splines to 1e-9; config 2's hyperplanes to 1e-4 (measured 7.5e-6)."""
    check_mixed(name, 4, w, 1e-9, hp_tol)


@pytest.mark.parametrize('variant', ['original', 'mirror', 'band'])
def test_warm_start_with_multipliers_matches_the_oracle(emu, variant):
    """The vehicle splines to 1e-9, the hyperplanes to 1e-7 (measured 2.1e-9)."""
    check_warm_start(variant, 1e-9, 1e-7)


@pytest.mark.parametrize('opts', BOUND_OPTIONS, ids=lambda o: '-'.join(sorted(o)))
def test_bound_options_on_two_sided_rows(emu, opts):
    """x to 1e-7 (measured 2.6e-9 with bound_relax_factor = 1e-6)."""
    check_bound_options(opts, 1e-7)


# ---------------------------------------------------------------------------------------
# the device kernels
# ---------------------------------------------------------------------------------------
@pytest.fixture(params=[None, '1'], ids=['snw-default', 'snw1'])
def snw(request, monkeypatch):
    """Supernode width of the sparse kernel: the default, and one column per level step."""
    if request.param:
        monkeypatch.setenv('OMG_B200_SNW', request.param)
    return request.param


@pytest.mark.gpu
@pytest.mark.parametrize('sel', ['alternate', 'all'])
@pytest.mark.parametrize('name', MIRROR_MODELS)
def test_gpu_mirrored_rows(gpu, snw, monkeypatch, name, sel):
    """The mirrored NLP on the device: statuses and iteration counts as the original, x to
    1e-12.  Measured on an H100: bit for bit (x, f and lam_g negated on the mirrored rows) on all
    ten cases, with the default supernodes and with OMG_B200_SNW=1 -- nvcc's contraction treats
    the lower- and the upper-bound branches alike."""
    check_mirror(monkeypatch, name, sel, 'default', x_tol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize('w', [1e3, 1e-1, 1e-3])
def test_gpu_two_sided_bands(gpu, snw, w):
    check_bands(w, 1e-9, 1e-8)


@pytest.mark.gpu
def test_gpu_narrow_bands_take_the_feasibility_fallback(gpu, snw):
    """omg_ipm_kernel_sp and omg_feas_kernel on narrow two-sided rows: Restoration_Failed
    without the feasibility phase, success after it, as the C oracle."""
    check_narrow_bands(twin=False)


@pytest.mark.gpu
def test_gpu_wide_bands_keep_the_solution_at_tight_tolerance(gpu, snw):
    check_wide_bands_tight()


@pytest.mark.gpu
def test_gpu_rows_free_in_some_instances(gpu, snw):
    check_free_rows(1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize('name, w, x_tol, hp_tol', [('config1', 1.0, 1e-9, None), ('config1', 0.1, 1e-9, None),
                                                    ('config2', 0.1, 1e-6, 5e-3)])
def test_gpu_row_types_mixed_across_instances(gpu, snw, name, w, x_tol, hp_tol):
    """On the device config 2's splines to 1e-6 (measured 1.5e-8 with OMG_B200_SNW=1) and its
    hyperplanes to tol-size 5e-3 (measured 2.1e-4), as tests/test_gpu_parity.py."""
    check_mixed(name, 4, w, x_tol, hp_tol)


@pytest.mark.gpu
@pytest.mark.parametrize('name, x_tol', [('config1', 1e-9), ('config2', 1e-6)])
def test_gpu_row_types_mixed_above_the_resident_slots(gpu, snw, name, x_tol):
    """1100 instances (more than the 528 resident blocks of config 2 and the 924 of config 1 on
    an H100): blocks that take a new instance meet other row types.  config 2's splines to 1e-6
    (measured 8.6e-8 with OMG_B200_SNW=1), its hyperplanes to 5e-3 (measured 5.3e-4)."""
    check_mixed(name, 1100, 0.1, x_tol, 5e-3, threads=16, tile=12)


@pytest.mark.gpu
@pytest.mark.parametrize('variant', ['original', 'mirror', 'band'])
def test_gpu_warm_start_with_multipliers(gpu, snw, variant):
    check_warm_start(variant, 1e-9, 1e-7)


@pytest.mark.gpu
@pytest.mark.parametrize('opts', BOUND_OPTIONS, ids=lambda o: '-'.join(sorted(o)))
def test_gpu_bound_options_on_two_sided_rows(gpu, snw, opts):
    check_bound_options(opts, 1e-7)
