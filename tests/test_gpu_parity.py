"""GPU parity tests (call through the C-ABI): CUDA solver vs the CPU oracle on
seeded instances and committed golden vectors; size-independent properties at
BASELINE batch sizes."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from omg_tools_b200 import scenarios as sc
from oracle import ipm_ref, ipm_c
from oracle.nlp_eval import TableEval


def oracle_solve(tb, x0, p, options=None, lam_g0=None):
    """CPU oracle: the C restatement (fast) when built, else the numpy twin."""
    if ipm_c.available():
        r = ipm_c.solve_batch_full(tb, x0[None], p[None], threads=1, options=options,
                                   lam_g0=None if lam_g0 is None else lam_g0[None])
        res = ipm_ref.Result()
        res.x, res.lam_g, res.f = r['x'][0], r['lam_g'][0], r['f'][0]
        res.status, res.iters = int(r['status'][0]), int(r['iters'][0])
        return res
    return ipm_ref.solve(tb, x0, p, options=options, lam_g0=lam_g0)

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'p2p_golden.npz'))
TIGHT = {'tol': 1e-8, 'compl_inf_tol': 1e-8, 'constr_viol_tol': 1e-8}
# GPU and oracle run the same algorithm in fp64 with different summation order
# and a different factorisation blocking; rounding differences are amplified by
# the interior-point iteration on ill-conditioned instances (non-unique
# separating hyperplanes).  X_TOL is for well-conditioned instances; the
# north-star criterion is 1e-4 on the spline coefficients.
X_TOL = 1e-5
NORTH_STAR_TOL = 1e-4


@pytest.fixture(scope='module')
def solvers():
    import __graft_entry__ as ge
    ge.build()
    out = {}
    for name in ('config1', 'config2', 'config5'):
        out[name] = getattr(sc, name)()
    return out


@pytest.mark.parametrize('name', ['config1', 'config2', 'config5'])
def test_matches_golden_default_tolerance(solvers, name):
    """tol = 1e-3 (the reference's setting): both runs stop somewhere in the tol-
    neighbourhood of the optimum.  The vehicle's spline coefficients (unique at the
    optimum) must agree to the north-star tolerance, the non-unique hyperplane /
    slack variables to tol-size."""
    pr = solvers[name]
    res = pr.problem.solve_batch(G[name + '_X0'], G[name + '_P'])
    assert np.array_equal(res['status'], G[name + '_loose_status'])
    assert np.abs(res['iters'] - G[name + '_loose_iters']).max() <= 2
    dx = np.abs(res['x'] - G[name + '_loose_x'])
    assert dx[:, :26].max() < NORTH_STAR_TOL
    assert dx.max() < 5e-3
    assert np.abs(res['f'] - G[name + '_loose_f']).max() < 1e-5
    assert np.abs(res['lam_g'] - G[name + '_loose_lam']).max() < 2e-2


def test_matches_golden_tight_tolerance(solvers):
    pr = solvers['config2']
    pr.problem.set_options(TIGHT)
    try:
        res = pr.problem.solve_batch(G['config2_X0'], G['config2_P'])
    finally:
        pr.problem.set_options({'tol': 1e-3, 'compl_inf_tol': 1e-4,
                                'constr_viol_tol': 1e-4})
    assert np.array_equal(res['status'], G['config2_tight_status'])
    # the separating hyperplanes (a, b) are not unique at the optimum: two correct solvers with
    # different pivot orders end 1.3e-4 apart there (measured; the envelope kernel 0.9e-4)
    assert np.abs(res['x'] - G['config2_tight_x']).max() < 5e-4
    # IPOPT-parity criterion of the north star: 1e-4 on the spline coefficients -- at tight
    # tolerance the vehicle splines are unique and agree far better (measured 4e-9)
    assert np.abs(res['x'][:, :26] - G['config2_tight_x'][:, :26]).max() < 1e-6


def test_matches_live_oracle_on_fresh_seed(solvers):
    pr = solvers['config1']
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 3, jitter=0.3, seed=7)
    res = pr.problem.solve_batch(X0, P)
    for b in range(3):
        ref = oracle_solve(tb, X0[b], P[b])
        assert res['status'][b] == ref.status and res['iters'][b] == ref.iters
        assert np.abs(res['x'][b] - ref.x).max() < X_TOL


def test_full_batch_properties_config2(solvers):
    """BASELINE config 2 at full size (batch 1024): identical instances give
    bit-identical results; jittered instances all satisfy the KKT conditions."""
    pr = solvers['config2']
    tb = pr.father.tables
    ev = TableEval(tb)
    X0, P = sc.instance_data(pr, 1, jitter=0.0)
    B = 1024
    res = pr.problem.solve_batch(np.repeat(X0, B, 0), np.repeat(P, B, 0))
    assert np.all(res['status'] == 0)
    assert np.all(res['x'] == res['x'][0]) and np.all(res['iters'] == res['iters'][0])
    assert np.abs(res['x'][0] - G['config2_loose_x'][0])[:26].max() < NORTH_STAR_TOL
    Xj, Pj = sc.instance_data(pr, 256, jitter=0.2, seed=11)
    rj = pr.problem.solve_batch(Xj, Pj)
    ok = rj['status'] == 0
    assert ok.mean() > 0.95
    eq = tb.lbg == tb.ubg
    for b in np.nonzero(ok)[0][:24]:
        V = ev.tape(Pj[b])
        g = ev.g(rj['x'][b], V)
        assert np.abs(g[eq]).max() < 2e-4 and g[~eq].max() < 2e-4
        stat = ev.gradf(rj['x'][b], V) + ev.jac_dense(rj['x'][b], V).T @ rj['lam_g'][b]
        assert np.abs(stat).max() < 1.0 + 1e-9          # dual_inf_tol (unscaled)
        assert abs(ev.f(rj['x'][b], V) - rj['f'][b]) < 1e-10
        assert np.abs(rj['lam_g'][b][~eq] * g[~eq]).max() < 1e-3


def test_edge_cases(solvers):
    pr = solvers['config1']
    tb = pr.father.tables
    X0, P = G['config1_X0'], G['config1_P']
    # per-instance bounds == shared bounds
    LB, UB = np.repeat(tb.lbg[None], 4, 0), np.repeat(tb.ubg[None], 4, 0)
    a = pr.problem.solve_batch(X0, P)
    b = pr.problem.solve_batch(X0, P, LB, UB)
    assert np.array_equal(a['x'], b['x'])
    # batch of one / ragged batch sizes around the SM count
    one = pr.problem.solve_batch(X0[:1], P[:1])
    assert np.array_equal(one['x'][0], a['x'][0])
    many = pr.problem.solve_batch(np.repeat(X0, 75, 0), np.repeat(P, 75, 0))  # 300
    assert np.array_equal(many['x'][::75], a['x'])
    # max_iter exhaustion is reported, not hidden
    pr.problem.set_options({'max_iter': 5})
    try:
        r = pr.problem.solve_batch(X0[:2], P[:2])
    finally:
        pr.problem.set_options({'max_iter': 3000})
    assert np.all(r['status'] == 1) and np.all(r['iters'] == 5)
    ref = oracle_solve(tb, X0[0], P[0], options={'max_iter': 5})
    assert np.abs(r['x'][0] - ref.x).max() < 1e-10
    # NaN parameters -> Invalid_Number_Detected, other instances unaffected
    Pn = P.copy()
    Pn[1, 0] = np.nan
    r = pr.problem.solve_batch(X0, Pn)
    assert r['status'][1] == 4 and r['status'][0] == 0
    assert np.array_equal(r['x'][0], a['x'][0])
    # warm start from the solution converges in far fewer iterations
    w = pr.problem.solve_batch(a['x'], P, lam_g0=a['lam_g'])
    assert np.all(w['status'] == 0) and np.all(w['iters'] < a['iters'])


def test_problem_solve_dropin(solvers):
    """Problem.solve() -- the reference's call (problem.py:103-136)."""
    pr = sc.config1()
    tb = pr.father.tables
    x0 = pr.father.get_variables().cat.copy()
    p = pr.father.set_parameters(0.).cat.copy()
    pr.solve(0., 0.1)
    assert pr.problem.stats()['return_status'] == 'Solve_Succeeded'
    ref = oracle_solve(tb, x0, p)
    assert np.abs(pr.father.get_variables().cat - ref.x).max() < X_TOL
    assert np.abs(pr.father.get_dual_variables().cat - ref.lam_g).max() < 1e-6
    splines = pr.father.get_variables(pr.vehicles[0], 'splines_seg0')
    assert abs(splines[0](0.)[0] + 1.5) < 1e-6 and abs(splines[0](1.)[0] - 2.) < 1e-2


def test_device_pointer_api_and_shift(solvers):
    import torch
    pr = solvers['config1']
    tb, slv = pr.father.tables, pr.problem
    dev = torch.device('cuda:0')
    X0 = torch.tensor(G['config1_X0'], device=dev)
    P = torch.tensor(G['config1_P'], device=dev)
    LB, UB = torch.tensor(tb.lbg, device=dev), torch.tensor(tb.ubg, device=dev)
    B = X0.shape[0]
    X = torch.empty_like(X0)
    LAM = torch.empty((B, tb.m), dtype=torch.float64, device=dev)
    F = torch.empty(B, dtype=torch.float64, device=dev)
    ST = torch.empty(B, dtype=torch.int32, device=dev)
    IT = torch.empty(B, dtype=torch.int32, device=dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        slv.solve_batch_device(X0, P, LB, UB, X, LAM, F, ST, IT)
    side.synchronize()
    assert np.abs(X.cpu().numpy() - G['config1_loose_x']).max() < X_TOL
    ms, launches = slv.last_timing()
    assert ms > 0 and launches == 1
    # warm-start knot shift on device == T.dot(coeffs) of the reference
    blocks = [(off, shape[0], shape[1], T) for (_, _, off, shape, T)
              in pr.father.shifted_entries()]
    Xs = X.clone()
    slv.shift_batch_device(Xs, blocks)
    want = X.cpu().numpy().copy()
    for off, L, nc, T in blocks:
        for c in range(nc):
            seg = slice(off + c * L, off + (c + 1) * L)
            want[:, seg] = X.cpu().numpy()[:, seg] @ np.asarray(T).T
    assert np.abs(Xs.cpu().numpy() - want).max() < 1e-13


def test_receding_horizon_config1(solvers):
    """10 MPC steps of the p2p_holonomic scenario through Problem.solve(),
    each checked against the oracle started from the same warm start."""
    pr = sc.config1()
    tb = pr.father.tables
    pr.initialize(0.)
    t, dt = 0., 0.1
    for k in range(12):
        pr.predict(t, dt, 0.01)
        pr.init_step(t, dt)
        x0 = pr.father.get_variables().cat.copy()
        p = pr.father.set_parameters(t).cat.copy()
        ref = oracle_solve(tb, x0, p)
        pr.solve(t, dt)
        assert pr.problem.stats()['return_status'] == ipm_ref.STATUS[ref.status]
        assert np.abs(pr.father.get_variables().cat - ref.x).max() < X_TOL
        pr.store(t, dt, 0.01)
        pr.simulate(t, dt, 0.01)
        t += dt
    # vehicle moved towards the goal and stayed on its trajectory
    assert pr.vehicles[0].signals['state'][0, -1] > -1.5


def test_batched_receding_horizon_config5(solvers):
    """BASELINE config 5 (revolving door, rotating obstacles): the batched
    device-resident MPC loop equals the reference-style sequential loop
    Problem.predict/solve/store/simulate, step by step."""
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    seq = sc.config5()
    seq.initialize(0.)
    bat = BatchMPC(sc.config5(), batch=3, update_time=0.1)
    t, dt = 0., 0.1
    for k in range(15):                      # crosses the first knot at t = 1.0
        seq.predict(t, dt, 0.01)
        seq.solve(t, dt)
        bat.step()
        Xb = bat.X.cpu().numpy()
        xs = seq.father.get_variables().cat
        assert seq.problem.stats()['return_status'] == 'Solve_Succeeded'
        assert np.all(bat.history['status'][-1] == 0)
        assert np.abs(Xb - xs[None]).max() < NORTH_STAR_TOL, k
        assert np.abs(Xb[:, :26] - xs[None, :26]).max() < X_TOL, k
        seq.store(t, dt, 0.01)
        seq.simulate(t, dt, 0.01)
        t = np.round(t + dt, 6)
    assert np.abs(bat.state[0] - seq.vehicles[0].signals['state'][:, -1]).max() < 1e-5


def test_receding_horizon_batch256_50_steps(solvers):
    """Config 5 at BASELINE size: 256 jittered instances, 50 MPC steps on device."""
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(sc.config5(), batch=256, update_time=0.1, jitter=0.1, seed=3)
    start = bat.state.copy()
    hist = bat.run(50)
    status = np.array(hist['status'])
    assert (status == 0).mean() > 0.90
    # every vehicle made progress towards its goal
    d0 = np.linalg.norm(start - bat.poseT, axis=1)
    d1 = np.linalg.norm(bat.state - bat.poseT, axis=1)
    assert np.all(d1 < d0)
    assert np.isfinite(bat.state).all()


@pytest.mark.parametrize('opts', [None, {'nesterov_acceleration': True},
                                  {'nesterov_acceleration': True, 'nesterov_reset': True}])
def test_formation_admm_matches_oracle(solvers, opts):
    """BASELINE config 3 (4 agents as in the reference example): batched x-update +
    consensus kernel vs the sequential ADMM oracle, iteration by iteration; plain
    ADMM and the fast (Nesterov) variants of admm.py:510-554."""
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    from oracle.admm_ref import ADMMOracle
    pr = sc.config3(4, opts)
    run = FormationADMMRunner(pr)
    orc = ADMMOracle(sc.config3(4, opts, build_solver=False))
    for it in range(6):
        rg = run.dual_update(0.)
        ro = orc.dual_update(0.)
        st, _ = run.status()
        assert np.all(st == 0) and np.all(orc.status == 0)
        assert np.abs(run.x_i.cpu().numpy() - orc.x_i).max() < NORTH_STAR_TOL, it
        assert np.abs(run.z_i.cpu().numpy() - orc.z_i).max() < NORTH_STAR_TOL
        assert np.abs(run.z_ij.cpu().numpy() - orc.z_ij).max() < NORTH_STAR_TOL
        assert np.abs(run.l_i.cpu().numpy() - orc.l_i).max() < 10 * NORTH_STAR_TOL
        assert np.abs(run.z_ji.cpu().numpy() - orc.z_ji).max() < NORTH_STAR_TOL
        assert abs(rg[0] - ro[0]) < 1e-3 * max(1., ro[0]) and abs(rg[1] - ro[1]) < 1e-3 * max(1., ro[1])


def test_formation_admm_64_agents(solvers):
    """Config 3 at BASELINE size: 64 agents on a ring; residuals and formation
    error shrink, every x-update succeeds."""
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    pr = sc.config3(64)
    run = FormationADMMRunner(pr)
    hist, spread = [], []
    for it in range(10):
        hist.append(run.dual_update(0.))
        st, _ = run.status()
        assert np.all(st == 0)
        cen = run.x_i.cpu().numpy().reshape(64, 2, 13) + pr.relp[:, :, None]
        # consensus spreads one neighbour per iteration on a 64-ring: measure the
        # mismatch between adjacent agents' views of the formation centre
        spread.append(np.abs(cen - np.roll(cen, 1, axis=0)).max())
    assert hist[-1][2] < hist[1][2]          # combined residual shrinks
    assert spread[-1] < spread[0]            # adjacent agents agree better than at start


def test_formation_admm_64_agents_matches_oracle(solvers):
    """Config 3 at BASELINE size against the sequential ADMM oracle (64 agent NLPs per iteration
    through the C oracle), iteration by iteration: shared variables, consensus variables and
    residuals to the tolerance of the reference's own formation test (5e-3,
    export/tests/formation/test.cpp:200-207).

    Tighter where it can be justified: in the first x-update every agent whose interior-point
    iteration count equals the oracle's agrees to 1e-6 (summation-order
    rounding of the factorisation carried through ~10 Newton steps; 1e-10 in the CPU emulation).  A few of the 64 agents end one iteration
    earlier or later than the oracle (a termination test decided by the last bits, tol = 1e-3,
    problem.py:57): those differ by tol-size (measured 2.7e-4 on agent 24) and their difference
    then travels through the consensus, so later iterations carry the 5e-3 bound only."""
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    from oracle.admm_ref import ADMMOracle
    run = FormationADMMRunner(sc.config3(64))
    orc = ADMMOracle(sc.config3(64, build_solver=False))
    for it in range(5):
        rg, ro = run.dual_update(0.), orc.dual_update(0.)
        st, its = run.status()
        assert np.all(st == 0) and np.all(orc.status == 0)
        d = np.abs(run.x_i.cpu().numpy() - orc.x_i).max(1)
        dz = np.abs(run.z_i.cpu().numpy() - orc.z_i).max()
        assert d.max() < 5e-3 and dz < 5e-3, (it, d.max(), dz)
        if it == 0:
            same = its == orc.iters
            assert same.sum() >= 58, (its, orc.iters)            # at most 10 % decided by rounding
            assert d[same].max() < 1e-6, d[same].max()
        assert abs(rg[0] - ro[0]) < 1e-2 * max(1., ro[0])


def test_quadrotor3d_config4_baseline_size_matches_oracle():
    """BASELINE config 4 at its stated size (5 plate obstacles: n = 406, m = 2039; the XL kernel
    with K in the L2-resident scratch): statuses and iteration counts as the C oracle, flat-output
    splines to the north-star tolerance on the nominal instance, all instances to tol-size."""
    pr = sc.config4(n_obstacles=5)
    tb = pr.father.tables
    assert (tb.n, tb.m) == (406, 2039)
    X0, P = sc.instance_data(pr, 4, jitter=0.05, seed=4)
    X0[0], P[0] = sc.instance_data(pr, 1)[0][0], sc.instance_data(pr, 1)[1][0]
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=4)
    assert np.array_equal(res['status'], ref['status']) and res['status'][0] == 0
    ok = ref['status'] == 0
    assert np.abs(res['iters'] - ref['iters'])[ok].max() <= 3
    err = np.abs(res['x'] - ref['x'])[:, :36].max(axis=1)
    assert err[0] < NORTH_STAR_TOL
    assert err[ok].max() < 5e-2 and np.abs(res['f'] - ref['f'])[ok].max() < 1e-4


def test_device_trajectory_sampling(solvers):
    """Post-solve extraction on device == scipy splev of the reference's
    sample_splines (spline_extra.py:406-410), state and input trajectories."""
    import torch
    from omg_tools_b200.solver.b200 import sample_batch
    from omg_tools_b200.basics.spline import BSpline
    from omg_tools_b200.basics.spline_extra import sample_splines
    pr = solvers['config1']
    veh = pr.vehicles[0]
    X = torch.tensor(G['config1_loose_x'], device='cuda:0')
    tau = np.linspace(0., 1., 101)
    basis = veh.basis
    S0 = basis.eval_basis(tau)
    Bd, P1 = basis.derivative(1)
    S1 = Bd.eval_basis(tau).dot(P1) / 10.
    out = sample_batch(X, [(0, 13, 2, S0), (0, 13, 2, S1)]).cpu().numpy()
    for b in range(X.shape[0]):
        for c in range(2):
            coeffs = G['config1_loose_x'][b, c * 13:(c + 1) * 13]
            ref = sample_splines(BSpline(basis, coeffs), tau)
            dref = sample_splines(BSpline(basis, coeffs).derivative(), tau) / 10.
            assert np.abs(out[b, c * 101:(c + 1) * 101] - ref).max() < 1e-12
            assert np.abs(out[b, 202 + c * 101:202 + (c + 1) * 101] - dref).max() < 1e-10


@pytest.mark.gpu
def test_holonomic3d_matches_oracle():
    """examples/p2p_holonomic_3d.py (Plate vehicle, Cuboid + rising prism,
    3D separating hyperplanes): same table format, the kernel needs no 3D
    special case.  8 jittered instances vs the CPU oracle."""
    # the example's own start/goal put the plate exactly on the room limit, so
    # jittered copies would be infeasible: interior start/goal here
    pr = sc.config_holonomic3d(start=(-1.7, -1.7, -1.7), goal=(1.7, 1.7, -1.7))
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 8, jitter=0.1, seed=1)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=8)
    assert np.array_equal(res['status'], ref['status'])
    assert (res['status'] == 0).all()
    # long solves (50-130 iterations) on degenerate hyperplanes: compare the
    # vehicle trajectory (first 39 coefficients) at the north-star tolerance
    # and the objective tightly
    assert np.abs(res['x'][:, :39] - ref['x'][:, :39]).max() < NORTH_STAR_TOL
    assert np.abs(res['f'] - ref['f']).max() < 1e-5
    ev = TableEval(tb)
    for b in range(8):
        g = ev.g(res['x'][b], ev.tape(P[b]))
        assert (g <= tb.ubg + 1e-4).all() and (g >= tb.lbg - 1e-4).all()   # constr_viol_tol


@pytest.mark.gpu
def test_quadrotor3d_config4_matches_oracle():
    """BASELINE config 4 (examples/p2p_3dquadrotor.py): rows up to degree 5,
    236 shared intermediates (acceleration product-spline coefficients) that
    the XL kernel differentiates through by the chain rule.  8 jittered
    instances vs the CPU oracle; same iteration counts, coefficients within
    the north-star tolerance."""
    pr = sc.config4()
    tb = pr.father.tables
    assert (tb.n, tb.m, tb.n_mid) == (238, 1319, 236)
    X0, P = sc.instance_data(pr, 8, jitter=0.1, seed=3)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=8)
    assert np.array_equal(res['status'], ref['status'])
    assert (res['status'] == 0).all()
    # (one instance of this set sits on a filter / barrier decision: 73 iterations in the oracle;
    #  75, 77, 80 on the GPU with three successive summation orders of the same assembly -- every
    #  other instance takes the oracle's count exactly)
    assert (res['iters'] == ref['iters']).sum() >= 7
    assert np.abs(res['iters'] - ref['iters']).max() <= 0.12 * ref['iters'].max()
    # This NLP is ill-conditioned (+-1e-3 bands tie two double integrals, free
    # separating planes): rounding differences (summation order, factorisation
    # blocking) are amplified along the interior-point path, on one instance of
    # this set up to a changed filter/barrier decision, and the two runs then stop
    # at two different points of the tol=1e-3 neighbourhood of the same optimum
    # (the numpy and C oracles differ from each other in the same way).  Most
    # instances must agree to the north-star tolerance, all of them in the
    # objective and to tol-size in x.
    err = np.abs(res['x'] - ref['x']).max(axis=1)
    assert (err < NORTH_STAR_TOL).sum() >= 6
    assert np.median(err) < X_TOL
    assert err.max() < 5e-2
    assert np.abs(res['f'] - ref['f']).max() < 1e-4
    ev = TableEval(tb)
    for b in range(8):
        g = ev.g(res['x'][b], ev.tape(P[b]))
        assert (g <= tb.ubg + 1e-4).all() and (g >= tb.lbg - 1e-4).all()


@pytest.mark.gpu
def test_quadrotor3d_receding_horizon_dropin():
    """Problem.solve() drop-in on config 4: six MPC steps (one knot crossing,
    warm starts), each solve compared with the oracle from the same start."""
    pr = sc.config4()
    tb = pr.father.tables
    pr.initialize(0.)
    t, dt = 0., 0.4
    for k in range(6):
        pr.predict(t, dt, 0.01)
        pr.init_step(t, dt)
        x0 = pr.father.get_variables().cat.copy()
        p = pr.father.set_parameters(t).cat.copy()
        ref = oracle_solve(tb, x0, p)
        pr.solve(t, dt)
        assert pr.problem.stats()['return_status'] == ipm_ref.STATUS[ref.status] == 'Solve_Succeeded'
        x = pr.father.get_variables().cat
        # vehicle part (flat outputs + acceleration slacks) of the solution
        assert np.abs(x[:78] - ref.x[:78]).max() < 5e-3
        assert abs(pr.problem.stats()['iter_count'] - ref.iters) <= 3
        pr.store(t, dt, 0.01)
        pr.simulate(t, dt, 0.01)
        t += dt
    assert pr.vehicles[0].signals['state'][1, -1] > -1.0     # moved towards the goal


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['config4', 'holonomic3d'])
def test_matches_vehicle_goldens(name):
    """CUDA path against the committed numpy-oracle solutions of config 4 and
    the Holonomic3D example at tight tolerance (end point solver independent)."""
    GV = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'vehicles_golden.npz'))
    if name == 'config4':
        pr = sc.config4()
    else:
        pr = sc.config_holonomic3d(start=(-1.7, -1.7, -1.7), goal=(1.7, 1.7, -1.7))
    pr.problem.set_options(TIGHT)
    res = pr.problem.solve_batch(GV[name + '_X0'], GV[name + '_P'])
    assert np.array_equal(res['status'], GV[name + '_tight_status'])
    assert np.abs(res['iters'] - GV[name + '_tight_iters']).max() <= 2
    assert np.abs(res['x'] - GV[name + '_tight_x']).max() < NORTH_STAR_TOL
    assert np.abs(res['f'] - GV[name + '_tight_f']).max() < 1e-6


@pytest.mark.gpu
def test_freeT_point2point_matches_oracle():
    """FreeTPoint2point: cold solves of jittered instances and a receding-
    horizon run (warm starts need the soft restoration path) vs the oracle."""
    pr = sc.config_freeT()
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 8, jitter=0.1, seed=2)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=8)
    assert np.array_equal(res['status'], ref['status'])
    ok = ref['status'] == 0
    assert ok.sum() >= 6
    assert np.abs(res['iters'] - ref['iters'])[ok].max() <= 2
    iT = pr.father._var_struct.entries[(pr.label, 'T')][0]
    assert np.abs(res['x'][ok, iT] - ref['x'][ok, iT]).max() < 1e-5      # motion time
    assert np.median(np.abs(res['x'] - ref['x'])[ok].max(axis=1)) < NORTH_STAR_TOL
    pr.initialize(0.)
    t, dt = 0., 0.5
    for k in range(8):
        pr.predict(t, dt, 0.01)
        pr.init_step(t, dt)
        x0 = pr.father.get_variables().cat.copy()
        p = pr.father.set_parameters(t).cat.copy()
        r = oracle_solve(tb, x0, p)
        pr.solve(t, dt)
        assert pr.problem.stats()['return_status'] == ipm_ref.STATUS[r.status] == 'Solve_Succeeded'
        assert abs(pr.horizon_time() - r.x[iT]) < 1e-4
        # (iteration counts may differ by a few: the bilinear T terms make the
        # path sensitive to rounding once the soft restoration is active)
        pr.store(t, dt, 0.01)
        pr.simulate(t, dt, 0.01)
        t += dt


@pytest.mark.gpu
def test_native_cpp_caller(tmp_path):
    """examples/native/native_solve.cpp: a C++ program that links only
    libomgb200.so, loads a table file and solves -- the twin of the reference's
    exported C++ runtime (Point2Point.cpp:80-91, 207-231).  Same result as the
    Python binding."""
    import subprocess
    from omg_tools_b200.solver import b200
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pr = sc.config1()
    tb = pr.father.tables
    exe = str(tmp_path / 'native_solve')
    lib_dir = os.path.join(root, 'omg_tools_b200', 'csrc')
    subprocess.check_call(['g++', '-O2', '-I', os.path.join(root, 'include'),
                           os.path.join(root, 'examples', 'native', 'native_solve.cpp'),
                           '-o', exe, '-L', lib_dir, '-lomgb200', '-Wl,-rpath,' + lib_dir])
    X0, P = sc.instance_data(pr, 3, jitter=0.2, seed=4)
    b200.save_tables(tb, str(tmp_path / 'p.omgtbl'))
    X0.tofile(str(tmp_path / 'x0.f64'))
    P.tofile(str(tmp_path / 'p.f64'))
    out = subprocess.check_output([exe, str(tmp_path / 'p.omgtbl'), str(tmp_path / 'x0.f64'),
                                   str(tmp_path / 'p.f64'), '3', str(tmp_path / 'x.f64')])
    res = pr.problem.solve_batch(X0, P)
    x = np.fromfile(str(tmp_path / 'x.f64')).reshape(3, tb.n)
    assert np.array_equal(x, res['x'])
    lines = out.decode().strip().splitlines()
    assert len(lines) == 3
    for b, line in enumerate(lines):
        tok = line.split()
        assert int(tok[3]) == res['status'][b] and int(tok[5]) == res['iters'][b]


@pytest.mark.gpu
def test_batched_receding_horizon_config4():
    """BASELINE config 4 in the batched device-resident MPC loop: equals the
    reference-style sequential loop step by step (identical instances), and a
    jittered batch of 64 flies towards its goals."""
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    seq = sc.config4()
    seq.initialize(0.)
    bat = BatchMPC(sc.config4(), batch=2, update_time=0.4)
    t, dt = 0., 0.4
    for k in range(5):                       # crosses the first knot at t = 0.5
        seq.predict(t, dt, 0.01)
        seq.init_step(t, dt)
        seq.solve(t, dt)
        bat.step()
        assert seq.problem.stats()['return_status'] == 'Solve_Succeeded'
        assert np.all(bat.history['status'][-1] == 0)
        xs = seq.father.get_variables().cat
        Xb = bat.X.cpu().numpy()
        assert np.abs(Xb[:, :78] - xs[None, :78]).max() < 5e-3, k
        seq.store(t, dt, 0.01)
        seq.simulate(t, dt, 0.01)
        t = np.round(t + dt, 6)
    assert np.abs(bat.state[0] - seq.vehicles[0].signals['state'][:, -1]).max() < 5e-3
    big = BatchMPC(sc.config4(), batch=64, update_time=0.4, jitter=0.1, seed=7)
    start = big.veh.position().copy()
    hist = big.run(6)
    assert (np.array(hist['status']) == 0).mean() > 0.95
    d0 = np.linalg.norm(start - big.poseT[:, :3], axis=1)
    d1 = np.linalg.norm(big.veh.position() - big.poseT[:, :3], axis=1)
    assert np.all(d1 < d0)


@pytest.mark.gpu
def test_planar_quadrotor_matches_oracle():
    """examples/p2p_quadrotor.py (vehicles/quadrotor.py): non-convex thrust
    bound, the case IPOPT's inertia test (number of negative pivots) is needed
    for.  8 jittered instances vs the CPU oracle."""
    pr = sc.config_quadrotor2d()
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 8, jitter=0.2, seed=11)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=8)
    assert np.array_equal(res['status'], ref['status'])
    ok = ref['status'] == 0
    assert ok.sum() >= 7
    assert np.median(res['iters'][ok]) < 80           # 140 with the positional inertia test
    # the flat outputs (vehicle splines, first 28 coefficients) and the objective
    assert np.median(np.abs(res['x'] - ref['x'])[ok][:, :28].max(axis=1)) < NORTH_STAR_TOL
    assert np.abs(res['f'] - ref['f'])[ok].max() < 1e-3


@pytest.mark.gpu
def test_rk4_state_prediction():
    """omg_integrate_rk4 (non-ideal prediction, Vehicle.predict / integrate_ode;
    C++ twin Vehicle::integrate): batch RK4 on the device vs numpy RK4 with the
    vehicle classes' own ode(), and vs the exact spline integral for the
    holonomic model."""
    import torch
    from omg_tools_b200 import Holonomic, Quadrotor, Quadrotor3D
    from omg_tools_b200.solver.b200 import integrate_rk4

    def rk4(veh, x, U, dt):
        for i in range(U.shape[0] - 1):
            k1 = veh.ode(x, U[i])
            k2 = veh.ode(x + 0.5 * dt * k1, U[i])
            k3 = veh.ode(x + 0.5 * dt * k2, U[i])
            k4 = veh.ode(x + dt * k3, U[i + 1])
            x = x + dt / 6. * (k1 + 2 * k2 + 2 * k3 + k4)
        return x

    rng = np.random.default_rng(5)
    B, steps, dt = 17, 40, 0.01
    for veh, ns, ni in ((Holonomic(), 2, 2), (Quadrotor3D(0.5), 8, 3), (Quadrotor(), 5, 2)):
        x0 = 0.3 * rng.standard_normal((B, ns))
        U = 0.5 * rng.standard_normal((B, steps + 1, ni))
        if ni == 3:
            U[:, :, 0] += 9.81
        out = integrate_rk4(type(veh).__name__, torch.tensor(x0, device='cuda:0'),
                            torch.tensor(U, device='cuda:0'), dt).cpu().numpy()
        ref = np.array([rk4(veh, x0[b], U[b], dt) for b in range(B)])
        assert np.abs(out - ref).max() < 1e-12
    # holonomic model on a solved trajectory.  The scheme of the reference's C++ twin uses
    # input[i] for the stages 1-3 and input[i+1] for the stage 4, i.e. the quadrature
    # dt*(5 u_i + u_{i+1})/6 per sample: exact for that rule, first order w.r.t. the spline.
    pr = sc.config1()
    res = pr.problem.solve_batch(G['config1_X0'], G['config1_P'])
    basis = pr.vehicles[0].basis
    tau = np.linspace(0., 0.04, steps + 1)            # 0.4 s of the 10 s horizon
    Bd, P1 = basis.derivative(1)
    V = Bd.eval_basis(tau).dot(P1) / 10.
    X = res['x']
    vel = np.stack([X[:, :13].dot(V.T), X[:, 13:26].dot(V.T)], axis=2)     # [B, steps+1, 2]
    b0, b1 = basis.eval_basis([0.])[0], basis.eval_basis([0.04])[0]
    pos0 = np.stack([X[:, :13].dot(b0), X[:, 13:26].dot(b0)], 1)
    pos1 = np.stack([X[:, :13].dot(b1), X[:, 13:26].dot(b1)], 1)
    out = integrate_rk4('Holonomic', torch.tensor(pos0, device='cuda:0'),
                        torch.tensor(np.ascontiguousarray(vel), device='cuda:0'), 0.01).cpu().numpy()
    rule = pos0 + 0.01 * (5. * vel[:, :-1] + vel[:, 1:]).sum(axis=1) / 6.
    assert np.abs(out - rule).max() < 1e-13
    assert np.abs(out - pos1).max() < 5e-3             # and close to the spline itself


@pytest.mark.gpu
def test_dubins_matches_oracle():
    """vehicles/dubins.py (substitution form, 116 shared intermediates): the XL
    kernel vs the CPU oracle on 8 jittered instances."""
    pr = sc.config_dubins()
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 8, jitter=0.1, seed=1)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=8)
    assert np.array_equal(res['status'], ref['status'])
    ok = ref['status'] == 0
    assert ok.sum() >= 7
    err = np.abs(res['x'] - ref['x'])[ok][:, :26].max(axis=1)       # v~ and tan(theta/2) splines
    assert np.median(err) < NORTH_STAR_TOL
    assert np.abs(res['f'] - ref['f'])[ok].max() < 1e-3


@pytest.mark.gpu
def test_retry_mu_option_on_the_references_quadrotor_warm_start():
    """Solver option ``retry_mu`` (host level, solver/b200.py): the infeasible warm start
    the reference's Quadrotor3D loop produces at a knot crossing (loop_golden.npz) fails
    by default and converges with the retry, to the oracle's point."""
    L = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'loop_golden.npz'))
    pr = sc.config4()
    tb = pr.father.tables
    X0 = np.vstack([L['config4_x0'][2], L['config4_x0'][0]])
    P = np.vstack([L['config4_p'][2], L['config4_p'][0]])
    pr.problem.set_options({'feas_steps': 0})       # (the feasibility phase does not rescue this one)
    plain = pr.problem.solve_batch(X0, P)
    assert plain['status'][0] != 0 and plain['status'][1] == 0
    pr.problem.set_options({'retry_mu': 1e-3})
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=2, options={'retry_mu': 1e-3, 'feas_steps': 0})
    assert np.array_equal(res['status'], [0, 0]) and np.array_equal(ref['status'], [0, 0])
    assert np.abs(res['f'] - ref['f']).max() < 1e-4
    assert np.abs(res['x'][1] - plain['x'][1]).max() == 0.0        # untouched instance
    assert np.abs(res['x'] - ref['x'])[:, :78].max() < 5e-3
