"""BatchMPC for problems with several vehicles in one NLP, and the fleet plant step
(omg_closed_loop_step_fleet): inter-vehicle avoidance (scenarios.config_interveh_offset, two
Holonomic vehicles swapping places) and the central formation (config_formation_central, four
Holonomic vehicles on the XL kernel), ideal and closed through the vehicles' dynamics.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu) against the numpy
twin (tests/plant_twin_fleet.py) and the reference's recorded loops (golden/fleet_loop_golden.npz,
make_fleet_loop_golden.py).  The ones marked gpu run the same checks on the device."""
import os
import sys
import types

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
import plant_twin as tw                  # noqa: E402
import plant_twin_fleet as twf           # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'fleet_loop_golden.npz')
CLOSED = {'ideal_prediction': False, 'ideal_update': False}
DISTURBED = dict(CLOSED, **{'1storder_delay': True, 'time_constant': 0.1,
                            'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}})
# x0, p and plant tolerances of the closed-loop goldens (tests/test_closed_loop.py)
TOL = (1e-5, 5e-6, 5e-6)
# The closed inter-vehicle runs take x0 to 2e-5: the plant follows the reference's odeint to
# 1.8e-6, and the knot-crossing shift at 1.0 s extrapolates the g splines with rows of up to
# 9.25, which takes x0 of that step to 1.4e-5 (measured on the CPU).  With the disturbance the
# solve of step 9 takes 27 iterations where the reference's takes 25 (p agrees to 6e-7) and ends
# 2.4e-2 away in the non-unique separating hyperplane; that run REPLAYS the reference's solutions
# (every step's solution is replaced by the golden's, as tests/test_batch_mpc_vehicles.py does for
# HolonomicOrient), so x0, p and the plant are compared on the reference's own trajectories and
# iteration counts are not compared.
# golden run -> (scenario, vehicle options of every vehicle, x0 tolerance, replay)
RUNS = {'config_interveh_offset_ideal': ('config_interveh_offset', None, TOL[0], False),
        'config_interveh_offset': ('config_interveh_offset', CLOSED, 2e-5, False),
        'config_interveh_offset_disturbed': ('config_interveh_offset', DISTURBED, 2e-5, True),
        'config_formation_central_ideal': ('config_formation_central', None, TOL[0], False),
        'config_formation_central': ('config_formation_central', CLOSED, TOL[0], False)}
# model, n_state, n_input of the kernel cases: Holonomic, Holonomic3D, Dubins
KERNEL_CASES = [(0, 2, 2), (0, 3, 3), (3, 3, 2)]


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _case(model, ni, rng, B, n_veh=3):
    """A batch whose rows hold n_veh vehicles' input splines at non-contiguous offsets with other
    variables between them, and the derivative rows [2, n_samp + 1, L] of an update across a knot."""
    from omg_tools_b200.execution.batch_mpc import plant_rows_der
    from omg_tools_b200.vehicles.dubins import Dubins
    from omg_tools_b200.vehicles.holonomic import Holonomic
    basis, T = (Dubins() if model == 3 else Holonomic()).basis, 10.
    L = len(basis)
    offsets = [3 + v * (ni * L + 7) for v in range(n_veh)]
    X = rng.standard_normal((B, offsets[-1] + ni * L + 5))
    for off in offsets:
        walk = np.cumsum(0.3 * rng.standard_normal((B, ni, L)), axis=2)
        if model == 3:                      # v~ > 0, tg small
            walk[:, 0] = 0.3 + 0.1 * rng.standard_normal((B, L))
            walk[:, 1] *= 0.3
        X[:, off:off + ni * L] = walk.reshape(B, ni * L)
    return X, offsets, L, plant_rows_der(basis, T, 0.95, 0.01, 10)[:2]


def _fleet(model, X, offsets, L, R, px, pu, step, seed=0, tau=None, dist=None, dt=0.01, device='cpu'):
    """The fleet kernel through the binding; dist = (filt, mean, stdev, n_traj).  Returns numpy."""
    import torch
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=device)
    X, px, pu = t(X), t(px), t(pu)
    out = [torch.empty_like(px), torch.empty_like(pu), torch.empty_like(px), torch.empty_like(pu)]
    d = None
    if dist is not None:
        filt, mean, sd, n_traj = dist
        scratch = torch.empty(px.shape[0] * px.shape[1] * pu.shape[2] * (n_traj + 24), dtype=torch.float64,
                              device=device)
        d = (filt, mean, sd, n_traj, scratch)
    b200.closed_loop_step_fleet(model, X, offsets, L, R, dt, px, pu, out, step, seed=seed, time_constant=tau,
                                disturbance=d)
    return [o.cpu().numpy() for o in out]


def _twin_case(model, ns, ni, rng, B, n_veh=3, idx=None):
    X, offsets, L, R = _case(model, ni, rng, B, n_veh)
    px = 0.1 * rng.standard_normal((B, n_veh, ns))
    pu = 0.05 * rng.standard_normal((B, n_veh, ni))
    return X, offsets, L, R, px, pu


# ---------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('lag, disturb', [(False, False), (True, False), (False, True), (True, True)])
def test_fleet_kernel_matches_the_twin(emu, lag, disturb):
    """Three vehicles at non-contiguous offsets: plant and predicted state and input of every
    vehicle against the twin, 1e-13 relative to the largest value."""
    rng = np.random.default_rng(7)
    for model, ns, ni in KERNEL_CASES:
        X, offsets, L, R, px, pu = _twin_case(model, ns, ni, rng, 4)
        spec = (0.05, 0.02 * np.ones(ni), 0.1 * np.ones(ni), 150) if disturb else None
        dist = (b200.disturbance_filter(0.05),) + spec[1:] if disturb else None
        out = _fleet(model, X, offsets, L, R, px, pu, 6, seed=9, tau=0.1 if lag else None, dist=dist)
        ref = twf.plant_step(model, X, offsets, L, R, 0.01, px, pu, 6, seed=9, time_constant=0.1 if lag else None,
                             disturbance_spec=spec)
        for o, r in zip(out, ref):
            err = np.abs(o - r).max() / max(1., np.abs(r).max())
            print('model %d n_state %d lag %d disturb %d: %.1e' % (model, ns, lag, disturb, err))
            assert err < 1e-13, (model, ns)
        if not lag and not disturb:
            assert np.array_equal(out[0], out[2]) and np.array_equal(out[1], out[3])


@pytest.mark.parametrize('model, ns, ni', KERNEL_CASES)
def test_one_vehicle_fleet_is_the_single_vehicle_step(emu, model, ns, ni):
    """A fleet of one vehicle at offset 0 gives omg_closed_loop_step_der's four outputs bit for bit,
    with the lag and the disturbance on."""
    import torch
    rng = np.random.default_rng(20 + ns + model)
    X, offsets, L, R, px, pu = _twin_case(model, ns, ni, rng, 3, n_veh=1)
    X = X[:, offsets[0]:]
    dist = (b200.disturbance_filter(0.05), 0.01 * np.ones(ni), 0.1 * np.ones(ni), 120)
    fleet = _fleet(model, X, [0], L, R, px, pu, 2, seed=4, tau=0.1, dist=dist)
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float64))
    scratch = torch.empty(3 * ni * 144, dtype=torch.float64)
    single = [t(np.zeros_like(px[:, 0])), t(np.zeros_like(pu[:, 0])), t(np.zeros_like(px[:, 0])),
              t(np.zeros_like(pu[:, 0]))]
    b200.closed_loop_step(model, t(X), L, R[0], R[1], 0.01, t(px[:, 0]), t(pu[:, 0]), single, 2, seed=4,
                          time_constant=0.1, disturbance=dist[:3] + (120, scratch),
                          higher=np.zeros((2,) + R.shape[1:]))        # (-> omg_closed_loop_step_der)
    for f, s in zip(fleet, single):
        assert np.array_equal(f[:, 0], s.numpy())


def test_each_vehicle_draws_its_own_signals(emu):
    """Through an identity filter and without lag, the applied input of vehicle v at sample s is
    its planned input plus the white noise of signal v * n_input + j of the instance: zero planned
    input shows plant_twin.normals(seed, step, b, v * n_input + j) itself (to the last bits of log,
    cos and sin)."""
    B, nv, ns, ni, L, n_traj, seed, step = 3, 3, 2, 2, 4, 20, 11, 5
    offsets = [1, 12, 30]
    X = np.zeros((B, 40))
    ident = np.r_[1., 0., 0., 0., 1., 0., 0., 0., 0., 0., 0.]
    px, pu = np.zeros((B, nv, ns)), np.zeros((B, nv, ni))
    for s in (0, 1, 7):
        R = np.full((2, s + 1, L), 0.25)
        out = _fleet(0, X, offsets, L, R, px, pu, step, seed=seed, dist=(ident, np.zeros(ni), np.ones(ni), n_traj))
        for b in range(B):
            for v in range(nv):
                for j in range(ni):
                    z = tw.normals(seed, step, b, v * ni + j, n_traj)[s]
                    assert abs(out[1][b, v, j] - z) < 1e-14, (s, b, v, j)
        assert np.array_equal(out[3], np.zeros_like(out[3]))


def _fleet_args(buf, n_veh=3, offsets=(0, 9, 20), n=30):
    """A valid argument list of omg_closed_loop_step_fleet (model 0, B = 2, host pointers)."""
    def p(name, a, dtype=np.float64):
        buf[name] = np.ascontiguousarray(a, dtype=dtype)
        return buf[name].ctypes.data
    B, ns, ni, L, n_samp, n_traj = 2, 2, 2, 3, 2, 20
    filt = np.r_[1., 0., 0., 0., 1., 0., 0., 0., 0., 0., 0.]
    plant = lambda k: p(k, np.zeros((B, n_veh, ni)))
    return [0, B, n_veh, ns, ni, n, p('x', np.ones((B, n))), p('off', offsets, np.int32) if offsets is not None
            else None, L, n_samp, 2, p('R', 0.1 * np.ones((2, n_samp + 1, L))), 0.01, 1, 0.1, 1, n_traj, p('filt', filt),
            p('mean', np.zeros(ni)), p('sd', np.ones(ni)), 1, 0, plant('px'), plant('pu'), plant('px1'), plant('pu1'),
            plant('qx'), plant('qu'), p('scr', np.zeros(B * n_veh * ni * (n_traj + 24))), None]


def test_bad_fleet_arguments_are_rejected(emu):
    """The valid call passes; n_veh < 1, null offsets, an offset < 0 or one whose input splines
    leave x, a null decision vector and a model the sizes do not fit are rejected with a message."""
    buf = {}
    assert emu.omg_closed_loop_step_fleet(*_fleet_args(buf)) == 0, emu.omg_last_error()
    assert emu.omg_closed_loop_step_fleet(*_fleet_args(buf, offsets=(0, 9, 24))) == 0, emu.omg_last_error()
    cases = [(dict(n_veh=0, offsets=(0,)), 'n_veh must be >= 1, got 0'),
             (dict(offsets=None), 'null argument (vehicle offsets)'),
             (dict(offsets=(0, -1, 20)), 'vehicle 1 at offset -1'),
             (dict(offsets=(0, 9, 25)), 'vehicle 2 at offset 25: its 2 input splines of length 3 leave x of 30')]
    for kw, message in cases:
        assert emu.omg_closed_loop_step_fleet(*_fleet_args(buf, **kw)) == -1, kw
        err = emu.omg_last_error().decode()
        assert err.startswith('omg_closed_loop_step_fleet: ') and message in err, err
    for index, value, message in ((6, None, 'null argument'), (3, 3, 'sizes'), (0, 7, 'unknown vehicle model 7'),
                                  (10, 1, 'derivative rows, got 1')):
        args = _fleet_args(buf)
        args[index] = value
        assert emu.omg_closed_loop_step_fleet(*args) == -1, (index, value)
        err = emu.omg_last_error().decode()
        assert err.startswith('omg_closed_loop_step_fleet: ') and message in err, err


# ---------------------------------------------------------------------------------------------
# BatchMPC
# ---------------------------------------------------------------------------------------------
def _batch(name, batch, device, seed=0, vehicle_options=None, **kw):
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    pr = getattr(sc, name)()
    for veh in pr.vehicles:
        veh.set_options(vehicle_options or {})
    return BatchMPC(pr, batch=batch, update_time=kw.pop('update_time', 0.1), device=device, seed=seed, **kw)


def _record_solves(bat, replay=None):
    """Record what every solve is handed; with ``replay`` (the golden's solutions x [steps, n])
    the solution of step k is replaced by the reference's."""
    import torch
    calls = []
    solve = bat.solver.solve_batch_device

    def rec(X0, P, LB, UB, Xn, *a, **kw):
        calls.append((X0.cpu().numpy().copy(), P.cpu().numpy().copy()))
        r = solve(X0, P, LB, UB, Xn, *a, **kw)
        if replay is not None:
            Xn.copy_(torch.from_numpy(np.repeat(replay[len(calls) - 1][None], Xn.shape[0], 0)))
        return r
    bat.solver.solve_batch_device = rec
    return calls


def _check_golden(run, batch, device):
    """BatchMPC hands the solver the reference's x0 and p at every step, statuses and iteration
    counts are equal, and in the closed runs every vehicle's plant state and applied input follow
    the reference's simulated signals (instance 0 only with the disturbance: the others draw their
    own noise)."""
    import torch
    G = np.load(GOLDEN)
    name, vopt, tx, replay = RUNS[run]
    n_steps = len(G[run + '_status'])
    bat = _batch(name, batch, torch.device(device), update_time=float(G[run + '_dt']), vehicle_options=vopt)
    assert bat.closed_loop == (vopt is not None)
    calls = _record_solves(bat, G[run + '_x'] if replay else None)
    bat.run(n_steps)
    b = slice(0, 1) if vopt and 'input_disturbance' in vopt else slice(None)
    err = np.zeros(3)
    for k in range(n_steps):
        X0, P = calls[k]
        e = [np.abs(X0[b] - G[run + '_x0'][k][None]).max(), np.abs(P[b] - G[run + '_p'][k][None]).max(), 0.]
        if bat.closed_loop:
            h = lambda key: bat.history[key][k + 1][b]
            e[2] = max(np.abs(h('plant') - G[run + '_plant_state'][k + 1][None]).max(),
                       np.abs(h('plant_input') - G[run + '_plant_input'][k + 1][None]).max())
        err = np.maximum(err, e)
        assert e[0] < tx and e[1] < TOL[1] and e[2] < TOL[2], (run, k, e)
        assert np.all(bat.history['status'][k][b] == G[run + '_status'][k]), (run, k)
        if not replay:
            assert np.all(bat.history['iters'][k][b] == G[run + '_iters'][k]), (run, k, bat.history['iters'][k])
    print('%s batch %d: x0 %.1e, p %.1e, plant %.1e' % ((run, batch) + tuple(err)))
    return bat


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('run', [r for r in sorted(RUNS) if r.startswith('config_interveh')])
def test_interveh_follows_the_references_loop(emu, run, batch):
    """config_interveh_offset, 12 x 0.1 s across the knot crossing at 1.0 s: ideal, at the
    reference's non-ideal defaults, and with the lag and the disturbance on both vehicles."""
    bat = _check_golden(run, batch, 'cpu')
    if bat.closed_loop:
        assert bat.history['plant'][-1].shape == (batch, 2, 2)
    assert bat.state.shape == bat.inp.shape == bat.poseT.shape == (batch, 2, 2)


@pytest.mark.parametrize('batch', [1, 2])
@pytest.mark.parametrize('run', ['config_formation_central', 'config_formation_central_ideal'])
def test_formation_follows_the_references_loop(emu, run, batch):
    """config_formation_central on the XL kernel, 4 x 0.5 s across the knot crossing at 1.5 s, ideal
    and at the reference's non-ideal defaults (batch 1 and 2: the emulated XL kernel is slow)."""
    _check_golden(run, batch, 'cpu')


def _rebased(name, vopt, state, poseT, **kw):
    """A batch-1 run that starts from one instance's start and goal."""
    import torch
    bat = _batch(name, 1, torch.device('cpu'), vehicle_options=vopt, **kw)
    for v, a in enumerate(bat.vehs):
        a.state[0], a.poseT[0] = state[v], poseT[v]
    X0 = np.repeat(bat.father.get_variables().cat[None], 1, 0)
    for a in bat.vehs:
        a.cold_start(X0)
    bat.X.copy_(torch.from_numpy(X0))
    bat.history['state'][0] = bat.state.copy()
    if bat.closed_loop:
        bat.plant_x.copy_(torch.from_numpy(bat.state))
        bat.history['plant'][0] = bat.plant_x.numpy().copy()
    return bat


def test_jittered_instances_are_independent(emu):
    """Instance b of a jittered fleet batch (one shift of all starts, one of all goals) equals a
    batch-1 run from that instance's start and goal, bit for bit, in the closed loop with the lag."""
    import torch
    vopt = dict(CLOSED, **{'1storder_delay': True, 'time_constant': 0.1})
    bat = _batch('config_interveh_offset', 3, torch.device('cpu'), seed=2, jitter=0.1, vehicle_options=vopt)
    st, goal = bat.state.copy(), bat.poseT.copy()
    # the jitter keeps the geometry: the same shift for every vehicle of an instance
    for b in (1, 2):
        assert np.allclose(st[b] - st[b, :1], st[0] - st[0, :1], atol=1e-15)
        assert np.allclose(goal[b] - goal[b, :1], goal[0] - goal[0, :1], atol=1e-15)
        assert not np.array_equal(st[b], st[0])
    bat.run(3)
    for b in (1, 2):
        one = _rebased('config_interveh_offset', vopt, st[b], goal[b])
        one.run(3)
        for key in ('plant', 'plant_input', 'state', 'iters', 'status'):
            assert all(np.array_equal(x[b], y[0]) for x, y in zip(bat.history[key], one.history[key])), (b, key)
        assert np.array_equal(bat.X.numpy()[b], one.X.numpy()[0])


def test_fleet_schedules_agree(emu, monkeypatch):
    """A disturbed fleet batch: the reversed and random thread schedules of the emulation give
    bit-identical plant histories."""
    import torch
    run = lambda: _batch('config_interveh_offset', 2, torch.device('cpu'), seed=5, jitter=0.05,
                         vehicle_options=DISTURBED).run(2)
    a = run()
    for sched in ('reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        d = run()
        for key in ('plant', 'plant_input', 'state'):
            assert all(np.array_equal(x, y) for x, y in zip(a[key], d[key])), (sched, key)


def _two_holonomic(**opts):
    from omg_tools_b200 import Holonomic
    vehicles = [Holonomic(), Holonomic()]
    for v, o in zip(vehicles, ({}, opts)):
        v.set_options(o)
    return vehicles


def test_unsupported_fleets_are_rejected():
    """BatchMPC names the cause for every multi-vehicle problem it does not run."""
    from omg_tools_b200 import Holonomic, Environment, Square, Rectangle
    from omg_tools_b200.basics.shape import Plate
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    from omg_tools_b200.vehicles.dubins import Dubins
    from omg_tools_b200.vehicles.holonomic3d import Holonomic3D
    fleet = lambda vehicles: types.SimpleNamespace(vehicles=vehicles)
    knots = _two_holonomic()
    knots[1].define_knots(knot_intervals=12)
    cases = [(fleet([Dubins(), Dubins()]), 'Holonomic or Holonomic3D only, not Dubins'),
             (fleet([Holonomic(), Holonomic3D(Plate(Rectangle(0.5, 1.), height=0.1))]),
              'mixed fleet of Holonomic, Holonomic3D'),
             (fleet(knots), 'one spline basis only'),
             (fleet(_two_holonomic(ideal_update=False)), "option 'ideal_update'"),
             (fleet(_two_holonomic(time_constant=0.2)), "option 'time_constant'"),
             (fleet(_two_holonomic(input_disturbance={'fc': 0.01, 'stdev': 0.05 * np.ones(2)})),
              "option 'input_disturbance'"),
             (fleet(_two_holonomic()[:1] + [types.SimpleNamespace(to_simulate=False)]), 'to_simulate = False'),
             (sc.config_trailer(build_solver=False), 'free end time (FreeTPoint2point) for one vehicle only')]
    vehicles = _two_holonomic()
    for k, v in enumerate(vehicles):
        v.set_initial_conditions([-1.5, k - 0.5])
        v.set_terminal_conditions([1.5, k - 0.5])
    free = sc._p2p(vehicles, Environment(room={'shape': Square(5.)}), {}, build_solver=False, freeT=True)
    cases.append((free, 'free end time (FreeTPoint2point) for one vehicle only, this problem has 2'))
    for problem, message in cases:
        with pytest.raises(NotImplementedError, match='BatchMPC') as e:
            BatchMPC(problem, batch=1, device='cpu')
        assert message in str(e.value), (message, str(e.value))


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 1024, 4096])
def test_gpu_fleet_kernel_matches_the_twin(B):
    """The device kernel with four vehicles, lag and disturbance against the twin on a spread of
    instances of each batch: 5e-13 relative, the bound of test_batch_mpc_vehicles.py's device test
    for the integrator and Dubins models (nvcc fuses the multiply-adds of the filter recursion)."""
    rng = np.random.default_rng(B)
    for model, ns, ni in KERNEL_CASES:
        X, offsets, L, R, px, pu = _twin_case(model, ns, ni, rng, B, n_veh=4)
        spec = (0.01, 0.02 * np.ones(ni), 0.05 * np.ones(ni), 901)
        out = _fleet(model, X, offsets, L, R, px, pu, 3, seed=12, tau=0.1,
                     dist=(b200.disturbance_filter(0.01),) + spec[1:], device='cuda')
        idx = np.unique(np.r_[0, B - 1, rng.integers(0, B, 4)])
        ref = twf.plant_step(model, X[idx], offsets, L, R, 0.01, px[idx], pu[idx], 3, seed=12, time_constant=0.1,
                             disturbance_spec=spec, instances=idx)
        for o, r in zip(out, ref):
            err = np.abs(o[idx] - r).max() / max(1., np.abs(r).max())
            print('model %d n_state %d B %d: %.1e' % (model, ns, B, err))
            assert err < 5e-13, (model, ns, B)


@pytest.mark.gpu
def test_gpu_batch_mpc_follows_the_references_fleet_loops():
    for run in sorted(RUNS):
        _check_golden(run, 1, 'cuda')


@pytest.mark.gpu
@pytest.mark.parametrize('name, dt', [('config_formation_central', 0.5), ('config_interveh_offset', 0.1)])
def test_gpu_fleet_batch_256_closed_loop(name, dt):
    """A jittered batch of 256, 20 MPC steps at the reference's non-ideal defaults: the closed loop
    fails no instance that the ideal loop on the same batch solves, instance 0 equals a batch-1 run
    bit for bit, and every vehicle of every instance whose solves all succeed ends closer to its
    goal.  (One formation instance, 160, fails every solve in both loops on the XL kernel:
    DESIGN.md section 8.)"""
    import torch
    dev = torch.device('cuda')
    closed = _batch(name, 256, dev, seed=3, jitter=0.1, update_time=dt, vehicle_options=CLOSED)
    ideal = _batch(name, 256, dev, seed=3, jitter=0.1, update_time=dt)
    one = _batch(name, 1, dev, seed=3, update_time=dt, vehicle_options=CLOSED)
    start = closed.state.copy()
    extra, failed = [], [0, 0]
    for k in range(20):
        for bat in (closed, ideal, one):
            bat.step()
        bad_closed, bad_ideal = closed.history['status'][k] != 0, ideal.history['status'][k] != 0
        failed[0] += int(bad_closed.sum())
        failed[1] += int(bad_ideal.sum())
        extra.append(bad_closed & ~bad_ideal)
        for key in ('plant', 'plant_input', 'iters', 'status'):
            assert np.array_equal(closed.history[key][-1][0], one.history[key][-1][0]), (k, key)
    print('%s: failed solves closed %d, ideal %d' % (name, failed[0], failed[1]))
    extra = np.array(extra)
    assert not extra.any(), np.argwhere(extra)
    solved = np.all(np.array(closed.history['status']) == 0, axis=0)
    print('%s: instances with a failed solve: %s' % (name, np.nonzero(~solved)[0].tolist()))
    d0 = np.linalg.norm(start - closed.poseT, axis=2)[solved]
    d1 = np.linalg.norm(closed.history['plant'][-1] - closed.poseT, axis=2)[solved]
    assert np.all(d1 < d0), (np.argwhere(d1 >= d0), d0[d1 >= d0], d1[d1 >= d0])
