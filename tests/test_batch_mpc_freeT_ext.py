"""BatchMPC with a free motion time (FreeTPoint2point) for HolonomicOrient, the planar Quadrotor and
SimpleQuadrotor3D, ideal and closed through the vehicle's own dynamics.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu): the model rows against
the reference's modelling code (golden/model_golden_freeT_ext.npz), the reference's own ideal and
closed free-T loops (golden/freeT_loop_golden_ext.npz, freeT_closed_loop_golden_ext.npz, made by
make_freeT_loop_golden_ext.py and make_freeT_closed_loop_golden_ext.py) and instance independence.
The ones marked gpu run the golden loops with the solver on the device and jittered batches of 256."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'freeT_loop_golden_ext.npz')
GOLDEN_CLOSED = os.path.join(HERE, 'golden', 'freeT_closed_loop_golden_ext.npz')
GOLDEN_MODEL = os.path.join(HERE, 'golden', 'model_golden_freeT_ext.npz')
DT = 0.5
NAMES = ['config_holonomic_orient_freeT', 'config_quadrotor2d_freeT', 'config_quadrotor3d_simple_freeT']
CLOSED = {'ideal_prediction': False, 'ideal_update': False}
DISTURBED = dict(CLOSED, **{'1storder_delay': True, 'time_constant': 0.1,
                            'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(3)}})
# the tolerances of test_batch_mpc_freeT.py (ideal: x0, p and T; the final state) and
# test_batch_mpc_freeT_closed.py (x0 and T, p, the plant)
FINAL_TOL = 1e-4
GOLDEN_TOL = (1e-5, 5e-6, 5e-6)
# The quadrotors' closed runs need test_batch_mpc_vehicles.py's SimpleQuadrotor3D tolerance: the error
# of the reference's odeint (at its default tolerances) in the plant grows over the 0.5 s updates, step
# by step, to 1.3e-5 (planar Quadrotor) and 2.0e-5 (SimpleQuadrotor3D) in the plant and 8.9e-6 and
# 1.6e-5 in p, the prediction from that plant (measured under the CPU emulation).
QUAD_TOL = (5e-5, 5e-5, 5e-5)
# closed golden run -> (scenario, vehicle options, tolerances); the reference's defaults are both
# ideal flags off
CLOSED_RUNS = {'config_holonomic_orient_freeT': ('config_holonomic_orient_freeT', CLOSED, GOLDEN_TOL),
               'config_quadrotor2d_freeT': ('config_quadrotor2d_freeT', CLOSED, QUAD_TOL),
               'config_quadrotor3d_simple_freeT': ('config_quadrotor3d_simple_freeT', CLOSED, QUAD_TOL),
               'config_holonomic_orient_freeT_ideal_update': (
                   'config_holonomic_orient_freeT', {'ideal_update': True, 'ideal_prediction': False}, GOLDEN_TOL),
               'config_holonomic_orient_freeT_disturbed': ('config_holonomic_orient_freeT', DISTURBED, GOLDEN_TOL)}


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _batch(scenario, batch, device, vehicle_options=None, seed=0, jitter=0.):
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    pr = getattr(sc, scenario)()
    pr.vehicles[0].set_options(vehicle_options or {})
    return BatchMPC(pr, batch=batch, update_time=DT, device=device, seed=seed, jitter=jitter)


# ---------------------------------------------------------------------------------------------
# model rows
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', NAMES)
def test_model_rows_equal_the_references(name):
    """The reference's own modelling code (make_model_golden_freeT_ext.py) on a numeric stand-in for
    casadi.MX: this framework's layout, bounds, every constraint row, the objective, the host's
    parameter vector and initial guess are the reference's, at T_parameter = T_variable (the
    reference's unset T parameter is dropped, as for config_freeT in test_model.py)."""
    import re
    from oracle.nlp_eval import TableEval
    M = np.load(GOLDEN_MODEL)
    pr = getattr(sc, name)(build_solver=False)
    tb, f = pr.father.tables, pr.father
    norm = lambda s: re.sub(r'(vehicle|obstacle|p2p|environment)\d+', r'\1#', str(s))
    layout = lambda st: [norm('%s|%s|%dx%d' % (k[0], k[1], v[2][0], v[2][1])) for k, v in st.entries.items()]
    assert layout(f._var_struct) == [norm(s) for s in M[name + '_var_layout']]
    ref_par = [norm(s) for s in M[name + '_par_layout']]
    k_T = ref_par.index('p2p#|T|1x1')
    size = lambda e: int(e.split('|')[2].split('x')[0]) * int(e.split('|')[2].split('x')[1])
    keep = np.ones(M[name + '_P'].shape[1], dtype=bool)
    keep[sum(size(e) for e in ref_par[:k_T])] = False
    ref_par.pop(k_T)
    assert layout(f._par_struct) == ref_par
    assert np.array_equal(tb.lbg, M[name + '_lb']) and np.array_equal(tb.ubg, M[name + '_ub'])
    ev = TableEval(tb)
    for k in range(M[name + '_X'].shape[0]):
        x, p = M[name + '_X'][k], M[name + '_P'][k][keep]
        V = ev.tape(p)
        g_ref = M[name + '_G'][k]
        err = np.abs(ev.g(x, V) - g_ref) / np.maximum(1., np.abs(g_ref))
        assert err.max() < 1e-7 and np.median(err) < 1e-12, (k, int(np.argmax(err)), err.max())
        assert abs(ev.f(x, V) - M[name + '_F'][k]) < 1e-10
    assert np.array_equal(f.set_parameters(0.37).cat, M[name + '_host_P'][keep])
    assert np.array_equal(f.get_variables().cat, M[name + '_host_X0'])


# ---------------------------------------------------------------------------------------------
# the reference's loops
# ---------------------------------------------------------------------------------------------
def _replay(bat, G, name, solve):
    """Record what every solve is handed (x0 and p of the instances solved) and hand back the
    reference's solution of step k (G[name + '_x'][k]).  With ``solve`` the solver runs first and its
    statuses stay; without it the solver is not called and the reference's status and iteration
    count are reported."""
    import torch
    calls = []
    solver = bat.solver.solve_batch_device
    x, st, it = G[name + '_x'], G[name + '_status'], G[name + '_iters']

    def rec(X0, P, LB, UB, Xn, LAM, F, ST, IT):
        k = len(calls)
        calls.append((X0.cpu().numpy().copy(), P.cpu().numpy().copy()))
        if solve:
            solver(X0, P, LB, UB, Xn, LAM, F, ST, IT)
        else:
            ST.fill_(int(st[k]))
            IT.fill_(int(it[k]))
        Xn.copy_(torch.from_numpy(np.repeat(x[k][None], Xn.shape[0], 0)).to(Xn.device))
    bat.solver.solve_batch_device = rec
    return calls


def _check_x0_p_T(bat, calls, G, name, rows, n_steps, tol=GOLDEN_TOL):
    err = np.zeros(3)
    for k in range(n_steps):
        X0, P = calls[k][0][rows], calls[k][1][rows]
        e = [np.abs(X0 - G[name + '_x0'][k][None]).max(), np.abs(P - G[name + '_p'][k][None]).max(),
             np.abs(bat.history['T'][k][rows] - G[name + '_T'][k]).max()]
        assert e[0] < tol[0] and e[1] < tol[1] and e[2] < tol[0], (name, k, e)
        err = np.maximum(err, e)
    return err


def _statuses(bat, G, name, rows, n_steps):
    """(step, device status, reference status) of every solve where they differ."""
    return [(k, bat.history['status'][k][rows].tolist(), int(G[name + '_status'][k])) for k in range(n_steps)
            if np.any(bat.history['status'][k][rows] != G[name + '_status'][k])]


def _check_golden(name, batch, device, solve):
    """BatchMPC against the reference's ideal free-T loop on the reference's solutions: x0, p and T at
    every step, the stop step and the final state (within 1e-4: the reference's last update moves the
    vehicle by T rounded to its 0.01 s samples, this loop by T).  Returns the steps whose device
    statuses differ from the reference's (with ``solve``)."""
    import torch
    G = np.load(GOLDEN)
    n_steps = len(G[name + '_status'])
    bat = _batch(name, batch, torch.device(device))
    calls = _replay(bat, G, name, solve)
    bat.run(n_steps + 5)
    assert len(calls) == n_steps and not bat.active.any(), (name, len(calls), n_steps)
    err = _check_x0_p_T(bat, calls, G, name, slice(None), n_steps)
    e_final = np.abs(bat.state - G[name + '_state'][None]).max()
    print('%s batch %d: x0 %.1e, p %.1e, T %.1e, final state %.1e' % ((name, batch) + tuple(err) + (e_final,)))
    assert e_final < FINAL_TOL, e_final
    return _statuses(bat, G, name, slice(None), n_steps) if solve else []


def _check_golden_closed(name, batch, device, solve):
    """BatchMPC against the reference's closed free-T loop on the reference's solutions: x0, p, T, the
    plant state and input at every update boundary and the stop step."""
    import torch
    G = np.load(GOLDEN_CLOSED)
    scenario, vopt, tol = CLOSED_RUNS[name]
    n_steps = len(G[name + '_status'])
    bat = _batch(scenario, batch, torch.device(device), vopt)
    calls = _replay(bat, G, name, solve)
    bat.run(n_steps + 5)
    assert len(calls) == n_steps and not bat.active.any(), (name, len(calls), n_steps)
    # the golden's noise is instance 0's: with the disturbance only instance 0 repeats its loop
    rows = slice(0, 1) if vopt.get('input_disturbance') else slice(None)
    err = _check_x0_p_T(bat, calls, G, name, rows, n_steps, tol)
    assert len(bat.history['plant']) == n_steps + 1
    e_plant = 0.
    for k in range(n_steps + 1):
        e = np.abs(bat.history['plant'][k][rows] - G[name + '_plant_state'][k][None]).max()
        # (the reference's first plant input is the first plan's input at t = 0, which the quadrotors'
        # initial constraints do not fix; the plant starts from the vehicle's initial input, as the
        # fixed-T loop does and as test_batch_mpc_vehicles.py compares it: from the first update on)
        if k > 0:
            e = max(e, np.abs(bat.history['plant_input'][k][rows] - G[name + '_plant_input'][k][None]).max())
        assert e < tol[2], (name, k, e)
        e_plant = max(e_plant, e)
    print('%s batch %d: x0 %.1e, p %.1e, T %.1e, plant %.1e' % ((name, batch) + tuple(err) + (e_plant,)))
    return _statuses(bat, G, name, rows, n_steps) if solve else []


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('name', NAMES)
def test_batch_mpc_follows_the_references_freeT_loop(emu, name, batch):
    """The reference's ideal free-T loop at batch 1 and 3 of identical copies.  The solver is not
    emulated: the reference's solutions, statuses and iteration counts are replayed through the loop.
    The emulated interior-point solves of these problems take minutes (SimpleQuadrotor3D's cold start
    takes the oracle 1235 iterations, and both quadrotor runs have solves that stop at the
    3000-iteration cap); the GPU test runs the solver."""
    _check_golden(name, batch, 'cpu', solve=False)


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('name', sorted(CLOSED_RUNS))
def test_batch_mpc_follows_the_references_closed_freeT_loop(emu, name, batch):
    """The reference's closed free-T loop at its own vehicle defaults for the three vehicles,
    HolonomicOrient with ideal_update on and ideal_prediction off, and HolonomicOrient with the lag and
    the disturbance on the device generator's noise; batch 1 and 3, the solutions replayed as in the
    ideal test.  The quadrotors' stop tests read the position part of the plant and the planned dspl."""
    _check_golden_closed(name, batch, 'cpu', solve=False)


def _identity_solver(bat):
    """Stand-in for the solver that returns the warm start, with T lowered by 0.2, as the solution
    (status 0): the loop around it -- warm start, prediction, plant step and stop test -- runs per
    instance as with a real solve, at the cost of the emulation's kernels other than the solver.  (The
    warm start alone keeps a T between dt and 2 dt: the reference's rule re-targets it to T.)"""
    def solve(X0, P, LB, UB, Xn, LAM, F, ST, IT):
        Xn.copy_(X0)
        Xn[:, bat.t_index] -= 0.2
        ST.fill_(0)
        IT.fill_(1)
    bat.solver.solve_batch_device = solve


def _jittered(scenario, B, vopt, device):
    """A jittered batch whose instances start from motion times 10, 8.7, 7.4, ... (so they stop at
    different steps), and a batch of B rows for each instance b in which only row b runs."""
    bat = _batch(scenario, B, device, vopt, seed=7, jitter=0.6)
    _identity_solver(bat)
    T0 = 10. - 1.3 * np.arange(B)
    bat.X[:, bat.t_index] = bat.torch.from_numpy(T0)
    ones = []
    for b in range(B):
        one = _batch(scenario, B, device, vopt, seed=7, jitter=0.6)
        _identity_solver(one)
        one.X.copy_(bat.X)
        one.active[:b] = one.active[b + 1:] = False
        ones.append(one)
    return bat, ones


@pytest.mark.parametrize('scenario, vopt', [('config_holonomic_orient_freeT', None),
                                            ('config_holonomic_orient_freeT', DISTURBED),
                                            ('config_quadrotor2d_freeT', CLOSED),
                                            ('config_quadrotor3d_simple_freeT', None),
                                            ('config_quadrotor3d_simple_freeT', CLOSED)])
def test_instances_are_independent(emu, scenario, vopt):
    """A jittered batch of 3 whose instances stop at different steps: each instance's history (T,
    state, plant) and final x are those of a run in which it is the only instance running, bit for bit.
    The solver is the identity (the warm start is the plan): this test is about the loop around it;
    the GPU batch tests compare instance 0 of a solved batch of 256 with a batch-1 run."""
    import torch
    dev = torch.device('cpu')
    bat, ones = _jittered(scenario, 3, vopt, dev)
    bat.run(40)
    assert not bat.active.any()
    stops = np.array(bat.history['active']).sum(axis=0)
    assert len(set(stops.tolist())) > 1, stops
    keys = ['T', 'state'] + (['plant', 'plant_input'] if bat.closed_loop else [])
    for b, one in enumerate(ones):
        one.run(40)
        n = len(one.history['T'])
        assert n == stops[b], (b, n, stops[b])
        for key in keys:
            for k in range(min(len(bat.history[key]), len(one.history[key]))):
                assert np.array_equal(bat.history[key][k][b], one.history[key][k][b]), (b, key, k)
        assert np.array_equal(bat.X[b].numpy(), one.X[b].numpy())


def test_unsupported_free_T_vehicles_raise():
    """Quadrotor3D, Bicycle and AGV have no per-instance prediction with a free motion time, and the
    Trailer's problem has a second, unsimulated vehicle: BatchMPC raises for each."""
    import torch
    from omg_tools_b200 import (Quadrotor3D, Bicycle, AGV, Environment, Point2point, Cuboid, Square)
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    cpu = torch.device('cpu')
    for vehicle, room in ((Quadrotor3D(0.5), Cuboid(8, 6, 8)), (Bicycle(length=0.4), Square(5.)),
                          (AGV(length=0.8), Square(5.))):
        pr = Point2point(vehicle, Environment(room={'shape': room}), options={'verbose': 0}, freeT=True)
        with pytest.raises(NotImplementedError, match='free end time .* for %s' % type(vehicle).__name__):
            BatchMPC(pr, 1, device=cpu)
    with pytest.raises(NotImplementedError, match='free end time'):
        BatchMPC(sc.config_trailer(build_solver=False), 1, device=cpu)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_batch_mpc_follows_the_references_freeT_loops():
    """Every golden loop at batch 1 with the solver on the device (its solutions replaced by the
    reference's after each solve).  The statuses that differ from the oracle's are printed."""
    for name in NAMES:
        print('ideal %s: differing statuses %s' % (name, _check_golden(name, 1, 'cuda', solve=True)))
    for name in sorted(CLOSED_RUNS):
        print('closed %s: differing statuses %s' % (name, _check_golden_closed(name, 1, 'cuda', solve=True)))


def _failed(bat):
    return int(sum((s > 0).sum() for s in bat.history['status']))


def _batch_256(scenario, vopt):
    """A jittered batch of 256 and the batch-1 run of its instance 0, 40 steps at most."""
    import torch
    dev = torch.device('cuda')
    bat = _batch(scenario, 256, dev, vopt, seed=3, jitter=0.1)
    one = _batch(scenario, 1, dev, vopt, seed=3)
    bat.run(40)
    one.run(40)
    n = len(one.history['status'])
    for key in ['status', 'iters', 'T', 'state'] + (['plant', 'plant_input'] if bat.closed_loop else []):
        assert all(np.array_equal(bat.history[key][k][0], one.history[key][k][0]) for k in range(n)), key
    assert np.array_equal(bat.X[0].cpu().numpy(), one.X[0].cpu().numpy())
    return bat


def _report(bat, scenario, vopt):
    """Print the batch's stop steps, failed solves and every instance that failed a solve or did not
    stop, with its statuses; returns the distance of every instance to its goal at the end."""
    st, act = np.array(bat.history['status']), np.array(bat.history['active'])
    nd = bat.veh.position().shape[1]
    pos = bat.history['plant'][-1][:, :nd] if bat.closed_loop else bat.veh.position()
    d = np.linalg.norm(pos - bat.poseT[:, :nd], axis=1)
    print('%s %s batch 256: stopped after %s steps (%d stopped), failed solves %d, max distance to goal %.2e'
          % (scenario, 'closed' if bat.closed_loop else 'ideal', np.unique(act.sum(axis=0)), (~bat.active).sum(),
             _failed(bat), d.max()))
    for b in range(256):
        if (st[:, b] > 0).any() or bat.active[b]:
            print('  instance %d: statuses %s, T %s, distance %.2e' % (
                b, st[act[:, b], b].tolist(), np.round(np.array(bat.history['T'])[act[:, b], b], 3).tolist(), d[b]))
    return d


@pytest.mark.gpu
@pytest.mark.parametrize('vopt', [None, CLOSED], ids=['ideal', 'closed'])
def test_gpu_batch_256_holonomic_orient_freeT(vopt):
    """A jittered batch of 256 of examples/p2p_holonomic_orient.py as written, ideal and at the
    reference's vehicle defaults: every instance stops within 40 steps at its goal (1e-2), and instance 0
    is a batch-1 run bit for bit.  T drops by the update time per step in the median over an instance's
    consecutive successful solves (within 0.15, as for config_freeT): not at every step, because the
    reference's own loop re-plans around the moving circle and raises T by 0.38 s and 1.2 s at its
    steps 6 and 8 (golden/freeT_loop_golden_ext.npz), and a failed solve hands on an arbitrary T.  On an
    H100 the batch fails 328 solves in the ideal loop and 317 in the closed loop; every instance stops
    after 21 to 31 steps within 5e-5 of its goal."""
    bat = _batch_256('config_holonomic_orient_freeT', vopt)
    d = _report(bat, 'config_holonomic_orient_freeT', vopt)
    assert not bat.active.any()
    assert d.max() < 1e-2
    T, act, st = np.array(bat.history['T']), np.array(bat.history['active']), np.array(bat.history['status'])
    ok = act & (st == 0)
    for b in range(256):
        pairs = ok[:-1, b] & ok[1:, b]
        dT = (T[1:, b] - T[:-1, b])[pairs]
        assert abs(np.median(dT) + DT) < 0.15, (b, T[act[:, b], b])


@pytest.mark.gpu
@pytest.mark.parametrize('scenario', ['config_quadrotor2d_freeT', 'config_quadrotor3d_simple_freeT'])
@pytest.mark.parametrize('vopt', [None, CLOSED], ids=['ideal', 'closed'])
def test_gpu_batch_256_quadrotors_freeT(scenario, vopt):
    """The same jittered batch of 256 for the two quadrotors, ideal and at the reference's defaults:
    every instance whose solves all succeed stops within 40 steps, and instance 0 is a batch-1 run bit
    for bit.  The instances that fail a solve are printed with their statuses and motion times: the
    reference's own loops fail solves on these problems (golden/freeT_loop_golden_ext.npz), and a failed
    solve hands on a long T, so such an instance may not stop within 40 steps (DESIGN.md section 8)."""
    bat = _batch_256(scenario, vopt)
    _report(bat, scenario, vopt)
    failed = (np.array(bat.history['status']) > 0).any(axis=0)
    assert not (bat.active & ~failed).any(), np.nonzero(bat.active & ~failed)[0]
