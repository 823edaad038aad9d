"""BatchMPC with a free motion time closed through the vehicle's own dynamics, and its plant kernel
omg_closed_loop_step_free (every instance samples its plan on its own time axis, for its own
number of samples, and filters its disturbance over its own trajectory length).

The tests without a mark run the kernel source on the CPU (tools/cpu_emu) against the numpy twin
(tests/plant_twin_free.py), the fixed-T kernel and the reference's own closed free-T loop
(golden/freeT_closed_loop_golden.npz, make_freeT_closed_loop_golden.py).  The ones marked gpu run
the same checks on the device."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
import plant_twin_free as twf            # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'freeT_closed_loop_golden.npz')
DT, ST = 0.5, 0.01
CLOSED = {'ideal_prediction': False, 'ideal_update': False}
DIST = {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}
DISTURBED = dict(CLOSED, **{'1storder_delay': True, 'time_constant': 0.1, 'input_disturbance': DIST})
# golden run -> (scenario, vehicle options); the reference's defaults are both ideal flags off
RUNS = {'config_freeT_moving': ('config_freeT_moving', CLOSED),
        'config_dubins_freeT': ('config_dubins_freeT', CLOSED),
        'config_freeT_disturbed': ('config_freeT', DISTURBED)}
X0_TOL, P_TOL, PLANT_TOL = 1e-5, 5e-6, 5e-6
# model -> (scenario whose vehicle basis is used, n_state, n_input, n_der, twin tolerance relative to
# the largest value: test_batch_mpc_vehicles.py's for models 2-5)
MODELS = {0: ('config_freeT', 2, 2, 2, 1e-13), 1: ('config4', 8, 3, 2, 1e-12),
          2: ('config_quadrotor2d', 5, 2, 4, 1e-12), 3: ('config_dubins_freeT', 3, 2, 2, 1e-13),
          4: ('config_holonomic_orient', 3, 3, 2, 1e-13), 5: ('config_quadrotor3d_simple', 8, 3, 4, 1e-12)}
# one launch: T below the sample time (n_samp 0), between dt and 2 dt, n_traj = 13, long horizons,
# a stopped instance (n_samp 0 at any T), T off the sample grid
T_MIX = [0.005, 0.7, 0.12, 10., 24., 3.7, 2.0, 0.437]
STOPPED = 6


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _t(a, device):
    import torch
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=device)


def _counts(T, stopped=()):
    """n_samp and n_traj per instance as BatchMPC computes them."""
    T = np.asarray(T, dtype=float)
    n_samp = np.where(T >= ST, np.round(np.minimum(DT, T) / ST, 6), 0).astype(np.int32)
    n_traj = np.where(T >= ST, np.round(T / ST, 6) + 1, 0).astype(np.int32)
    n_samp[list(stopped)] = 0
    n_traj[n_traj <= 12] = 0
    return n_samp, n_traj


def _case(model, rng, Ts):
    """Spline coefficients of the model's vehicle basis (a walk not far from a flight), T in the
    last entry of x, and the block of the input splines."""
    name, ns, ni, nd, _ = MODELS[model]
    basis = getattr(sc, name)(build_solver=False).vehicles[0].basis
    L, B = len(basis), len(Ts)
    walk = np.cumsum(0.3 * rng.standard_normal((B, ni, L)), axis=2)
    if model == 1:
        walk[:, 0] += 9.81
    if model == 3:
        walk[:, 0] = 0.3 + 0.1 * rng.standard_normal((B, L))
        walk[:, 1] *= 0.3
    if model == 4:
        walk[:, 2] *= 0.3
    X = np.c_[walk.reshape(B, ni * L), Ts]
    return X, (0, L, ni, basis.degree, basis.knots), ni * L


def _run(model, X, block, t_index, n_samp, px, pu, out0, step, seed, tau, dist, device):
    """The kernel through the binding; dist = (fc, mean, stdev, n_traj).  Returns numpy outputs."""
    import torch
    ni, nd = MODELS[model][2], MODELS[model][3]
    out = [_t(o, device) for o in out0]
    d = None
    if dist is not None:
        fc, mean, sd, n_traj = dist
        scratch = torch.empty(X.shape[0] * ni * (int(n_traj.max()) + 24), dtype=torch.float64, device=device)
        d = (b200.disturbance_filter(fc), mean, sd, n_traj, scratch)
    b200.closed_loop_step_free(model, _t(X, device), block, t_index, nd, n_samp, ST, _t(px, device), _t(pu, device),
                               out, step, seed=seed, time_constant=tau, disturbance=d)
    return [o.cpu().numpy() for o in out]


def _check_twin(model, lag, disturb, Ts, device, rng, check=None):
    """Kernel against the twin on one launch with motion times Ts; returns the largest relative error."""
    name, ns, ni, nd, tol = MODELS[model]
    X, block, ti = _case(model, rng, Ts)
    B = len(Ts)
    n_samp, n_traj = _counts(Ts, [b for b in range(B) if b % len(T_MIX) == STOPPED])
    px, pu = 0.1 * rng.standard_normal((B, ns)), 0.1 * rng.standard_normal((B, ni))
    out0 = [rng.standard_normal((B, ns)), rng.standard_normal((B, ni)), rng.standard_normal((B, ns)),
            rng.standard_normal((B, ni))]
    spec = (0.05, 0.02 * np.ones(ni), 0.1 * np.ones(ni), n_traj) if disturb else None
    tau = 0.1 if lag else None
    got = _run(model, X, block, ti, n_samp, px, pu, out0, 6, 9, tau, spec, device)
    if check is None:
        idx = np.arange(B)
        ref = twf.plant_step_free(model, X, block, ti, n_samp, ST, px, pu, out0, 6, seed=9, time_constant=tau,
                                  disturbance_spec=spec)
    else:
        idx = np.asarray(check)
        ref = _twin_rows(model, X, block, ti, n_samp, px, pu, out0, tau, spec, idx)
    err = 0.
    for o, r, o0 in zip(got, ref, out0):
        r = r[idx] if check is None else r
        for b in idx:
            if n_samp[b] == 0:
                assert np.array_equal(o[b], o0[b]), (model, b)
        e = np.abs(o[idx] - r).max() / max(1., np.abs(r).max())
        err = max(err, e)
        assert e < tol, (model, lag, disturb, e)
    return err


def _twin_rows(model, X, block, ti, n_samp, px, pu, out0, tau, spec, idx):
    """The twin on the rows idx of a launch, each with its own global instance id."""
    res = [np.array(o[idx], copy=True) for o in out0]
    for j, b in enumerate(idx):
        sel = np.zeros(len(X), dtype=bool)
        sel[b] = True
        ns_b = np.where(sel, n_samp, 0)
        r = twf.plant_step_free(model, X, block, ti, ns_b, ST, px, pu, out0, 6, seed=9, time_constant=tau,
                                disturbance_spec=None if spec is None else spec[:3] + (np.where(sel, spec[3], 0),))
        for o, v in zip(res, r):
            o[j] = v[b]
    return res


@pytest.mark.parametrize('lag, disturb', [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_the_twin(emu, lag, disturb):
    """All six models, one launch with mixed motion times: below the sample time and stopped
    (outputs untouched bit for bit), between dt and 2 dt, n_traj = 13, long horizons and T off the
    sample grid; the four outputs against the twin to test_batch_mpc_vehicles.py's tolerances."""
    rng = np.random.default_rng(3)
    for model in MODELS:
        err = _check_twin(model, lag, disturb, T_MIX, 'cpu', rng)
        print('model %d lag %d disturb %d: %.1e' % (model, lag, disturb, err))


def _check_fixed_T(model, device, rng):
    """Every T equal: the free-T kernel against omg_closed_loop_step_der on the host's rows."""
    import torch
    name, ns, ni, nd, _ = MODELS[model]
    B, T = 3, 4.0
    X, block, ti = _case(model, rng, [T] * B)
    n_samp, n_traj = _counts([T] * B)
    px, pu = 0.1 * rng.standard_normal((B, ns)), 0.1 * rng.standard_normal((B, ni))
    spec = (0.05, np.zeros(ni), 0.1 * np.ones(ni), n_traj)
    zeros = [np.zeros((B, ns)), np.zeros((B, ni))] * 2
    free = _run(model, X, block, ti, n_samp, px, pu, zeros, 2, 4, 0.1, spec, device)
    R = twf.rows(_basis(block), T, ST, int(n_samp[0]), nd)
    out = [_t(z, device) for z in zeros]
    scratch = torch.empty(B * ni * (int(n_traj[0]) + 24), dtype=torch.float64, device=device)
    b200.closed_loop_step(model, _t(X, device), block[1], R[0], R[1], ST, _t(px, device), _t(pu, device), out, 2,
                          seed=4, time_constant=0.1,
                          disturbance=(b200.disturbance_filter(0.05), spec[1], spec[2], int(n_traj[0]), scratch),
                          higher=R[2:] if nd > 2 else None)
    err = 0.
    for o, f in zip(out, free):
        o = o.cpu().numpy()
        e = np.abs(o - f).max() / max(1., np.abs(o).max())
        err = max(err, e)
        assert e < 1e-13, (model, e)
    return err


def _basis(block):
    from omg_tools_b200.basics.spline import BSplineBasis
    return BSplineBasis(block[4], block[3])


@pytest.mark.parametrize('model', sorted(MODELS))
def test_equal_motion_times_match_the_fixed_T_kernel(emu, model):
    """With every T equal, omg_closed_loop_step_free is omg_closed_loop_step_der on the host's basis
    rows to rounding (1e-13 relative), lag and disturbance on."""
    print('model %d: %.1e' % (model, _check_fixed_T(model, 'cpu', np.random.default_rng(20 + model))))


def _free_args(buf, **kw):
    """A valid argument list of omg_closed_loop_step_free: Dubins, B = 2, host pointers."""
    def p(name, a, dtype=np.float64):
        buf[name] = np.ascontiguousarray(a, dtype=dtype)
        return buf[name].ctypes.data
    x = np.r_[0.2 * np.ones(5), 0.1 * np.ones(5), 1.0]
    x = np.tile(x, 2)
    filt = np.r_[1., 0., 0., 0., 1., 0., 0., 0., 0., 0., 0.]
    a = dict(model=3, B=2, ns=3, ni=2, n=11, x=p('x', x), off=0, L=5, nc=2, degree=3,
             knots=p('k', np.r_[0., 0, 0, 0, .5, 1, 1, 1, 1]), t_index=10, n_der=2,
             n_samp=p('ns', [20, 0], np.int32), n_traj=p('nt', [101, 0], np.int32), st=0.01, lag=1, tc=0.1,
             disturb=1, filt=p('filt', filt), mean=p('mean', np.zeros(2)), sd=p('sd', np.ones(2)), seed=1, step=0,
             px=p('px', np.zeros(6)), pu=p('pu', np.ones(4)), px1=p('px1', np.zeros(6)), pu1=p('pu1', np.zeros(4)),
             qx=p('qx', np.zeros(6)), qu=p('qu', np.zeros(4)), scr=p('scr', np.zeros(2 * 2 * (101 + 24))), stream=None)
    for key, val in kw.items():
        if isinstance(val, tuple):          # (array, dtype)
            val = p(key, *val)
        a[key] = val
    return list(a.values())


def test_bad_arguments_are_rejected(emu):
    """The valid call passes (also with n_traj 0: no disturbance); each refusal comes with its
    message, including every one omg_closed_loop_step_der makes."""
    buf = {}
    assert emu.omg_closed_loop_step_free(*_free_args(buf)) == 0, emu.omg_last_error()
    assert emu.omg_closed_loop_step_free(*_free_args(buf, n_traj=([0, 0], np.int32))) == 0
    assert emu.omg_closed_loop_step_free(*_free_args(buf, disturb=0, n_traj=None)) == 0
    i32 = np.int32
    cases = [
        (dict(model=6), 'unknown vehicle model 6'), (dict(model=-1), 'unknown vehicle model -1'),
        (dict(ns=4), 'bad state / input sizes'), (dict(ni=3), 'bad state / input sizes'),
        (dict(n_der=1), 'derivative rows, got 1'), (dict(n_der=5), 'derivative rows, got 5'),
        (dict(x=None), 'null argument'), (dict(knots=None), 'null argument'), (dict(n_samp=None), 'null argument'),
        (dict(n_traj=None), 'null argument'), (dict(scr=None), 'null argument'), (dict(px=None), 'null argument'),
        (dict(qu=None), 'null argument'), (dict(filt=None), 'null argument'),
        (dict(knots=(np.r_[0., 0, 0, 0, .5, 1, .9, 1, 1], np.float64)), 'knots not non-decreasing'),
        (dict(off=2), 'columns outside x'), (dict(n=9, t_index=8), 'columns outside x'),
        (dict(degree=9), 'degree 9'), (dict(L=3), 'basis length 3'),
        (dict(degree=2, knots=(np.r_[0., 0, 0, .4, .7, 1, 1, 1], np.float64), n_der=4),
         'n_der 4 above degree + 1 = 3'),
        (dict(nc=1), 'the spline block has 1 columns, the model reads 2'),
        (dict(t_index=11), 't_index 11 outside [0, 11)'), (dict(t_index=-1), 't_index -1 outside'),
        (dict(st=0.), 'sample_time must be > 0'), (dict(st=-0.01), 'sample_time must be > 0'),
        (dict(tc=0.), 'time_constant must be > 0 with the lag on'),
        (dict(n_samp=([-1, 0], i32)), 'instance 0: n_samp < 0'),
        (dict(n_traj=([12, 0], i32)), 'instance 0: n_traj must be 0 or exceed the filter padding of 12'),
        (dict(n_traj=([101, 5], i32)), 'instance 1: n_traj must be 0 or exceed the filter padding'),
        (dict(n_traj=([-1, 0], i32)), 'instance 0: n_traj must be 0'),
        (dict(n_traj=([20, 0], i32)), 'instance 0: n_traj < n_samp + 1'),
        (dict(n_samp=([0, 1024], i32), n_traj=([0, 2000], i32)),
         '(max n_samp + 1) * n_input exceeds 2048 samples per update')]
    for kw, message in cases:
        assert emu.omg_closed_loop_step_free(*_free_args(buf, **kw)) == -1, kw
        err = emu.omg_last_error().decode()
        assert err.startswith('omg_closed_loop_step_free: ') and message in err, (kw, err)
    # the lag off takes any time constant; n_samp 1023 with 2 inputs is the largest update
    assert emu.omg_closed_loop_step_free(*_free_args(buf, tc=0., lag=0)) == 0
    assert emu.omg_closed_loop_step_free(*_free_args(buf, n_samp=([0, 1023], i32), n_traj=([0, 2000], i32),
                                                     scr=(np.zeros(2 * 2 * 2024), np.float64))) == 0


# ---------------------------------------------------------------------------------------------
# BatchMPC
# ---------------------------------------------------------------------------------------------
def _batch(scenario, batch, device, vehicle_options, seed=0, jitter=0., **kw):
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    pr = getattr(sc, scenario)(**kw)
    pr.vehicles[0].set_options(vehicle_options)
    return BatchMPC(pr, batch=batch, update_time=DT, device=device, seed=seed, jitter=jitter)


def _replay(bat, x):
    """Record what every solve is handed (x0 and p of the instances solved) and replace the solution
    of step k by x[k], so the loop around the solver runs on those trajectories."""
    import torch
    calls = []
    solve = bat.solver.solve_batch_device

    def rec(X0, P, LB, UB, Xn, *a, **kw):
        calls.append((X0.cpu().numpy().copy(), P.cpu().numpy().copy()))
        r = solve(X0, P, LB, UB, Xn, *a, **kw)
        Xn.copy_(torch.from_numpy(np.repeat(x[len(calls) - 1][None], Xn.shape[0], 0)).to(Xn.device))
        return r
    bat.solver.solve_batch_device = rec
    return calls


def _check_golden(name, batch, device):
    """BatchMPC against the reference's closed free-T loop on the reference's solutions (replayed):
    x0 (without Dubins' dx, dy, which the reference does not shift), p, T, the plant state and input
    at every update boundary, the stop step and the statuses (but for Dubins' cold first solve)."""
    import torch
    G = np.load(GOLDEN)
    scenario, vopt = RUNS[name]
    n_steps = len(G[name + '_status'])
    bat = _batch(scenario, batch, torch.device(device), vopt)
    calls = _replay(bat, G[name + '_x'])
    bat.run(n_steps + 5)
    assert len(calls) == n_steps and not bat.active.any(), (name, len(calls), n_steps)
    keep = np.ones(bat.tb.n, dtype=bool)
    if 'dubins' in name:
        ent = bat.father._var_struct.entries
        for nm in ('dx', 'dy'):
            off, size, _ = ent[(bat.vehicle.label, nm)]
            keep[off:off + size] = False
    # the golden's noise is instance 0's: with the disturbance only instance 0 repeats its loop
    rows = slice(0, 1) if vopt.get('input_disturbance') else slice(None)
    err = np.zeros(4)
    for k in range(n_steps):
        X0, P = calls[k]
        X0, P = X0[rows], P[rows]
        e = [np.abs(X0 - G[name + '_x0'][k][None])[:, keep].max(), np.abs(P - G[name + '_p'][k][None]).max(),
             np.abs(bat.history['T'][k] - G[name + '_T'][k]).max()]
        assert e[0] < X0_TOL and e[1] < P_TOL and e[2] < X0_TOL, (name, k, e)
        if not ('dubins' in name and k == 0):
            assert np.all(bat.history['status'][k][rows] == G[name + '_status'][k]), (name, k)
        err[:3] = np.maximum(err[:3], e)
    assert len(bat.history['plant']) == n_steps + 1
    for k in range(n_steps + 1):
        e = max(np.abs(bat.history['plant'][k][rows] - G[name + '_plant_state'][k][None]).max(),
                np.abs(bat.history['plant_input'][k][rows] - G[name + '_plant_input'][k][None]).max())
        assert e < PLANT_TOL, (name, k, e)
        err[3] = max(err[3], e)
    print('%s batch %d: x0 %.1e, p %.1e, T %.1e, plant %.1e' % ((name, batch) + tuple(err)))


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('name', sorted(RUNS))
def test_batch_mpc_follows_the_references_closed_freeT_loop(emu, name, batch):
    """The reference's closed free-T loop with its own vehicle options (the moving-obstacle holonomic
    variant, p2p_dubins.py as written, and config_freeT with lag and disturbance on the device
    generator's noise) at batch 1 and 3 of identical copies."""
    _check_golden(name, batch, 'cpu')


def _instance_alone(bat, b, device, vopt):
    """A BatchMPC in which only row b runs, with the start and goal of instance b of ``bat``: rows
    0..b-1 are stopped from the start, so row b draws instance b's noise."""
    one = _batch('config_freeT', b + 1, device, vopt, seed=7)
    one.veh.state[b], one.veh.poseT[b] = bat.veh.state[b], bat.veh.poseT[b]
    X0 = np.repeat(one.father.get_variables().cat[None], b + 1, 0)
    one.veh.cold_start(X0)
    one.X.copy_(_t(X0, device))
    one.plant_x.copy_(_t(one.state, device))
    one.plant_u.copy_(_t(one.inp, device))
    one.active[:b] = False
    for key in ('state', 'plant', 'plant_input'):
        one.history[key] = [np.array(bat.history[key][0], copy=True)]
    return one


def _check_independent(bat, ones, steps):
    act = np.array(bat.history['active'])
    stops = act.sum(axis=0)
    for b, one in enumerate(ones):
        one.run(steps)
        n = len(one.history['status'])
        assert n == stops[b], (b, n, stops[b])
        for key in ('status', 'iters', 'T'):
            assert all(np.array_equal(bat.history[key][k][b], one.history[key][k][b]) for k in range(n)), (b, key)
        for key in ('state', 'plant', 'plant_input'):
            for k in range(len(bat.history[key])):
                assert np.array_equal(bat.history[key][k][b], one.history[key][min(k, n)][b]), (b, key, k)
        assert np.array_equal(bat.X[b].cpu().numpy(), one.X[b].cpu().numpy())
    return stops


def test_instances_are_independent(emu, monkeypatch):
    """A jittered batch of 4 with lag and disturbance whose instances stop at different steps: each
    instance's history (statuses, iterations, T, prediction, plant) is that of a run in which it is
    the only instance running, bit for bit; the reversed and random thread schedules of the
    emulation give the same histories."""
    import torch
    dev = torch.device('cpu')
    bat = _batch('config_freeT', 4, dev, DISTURBED, seed=7, jitter=0.6)
    ones = [_instance_alone(bat, b, dev, DISTURBED) for b in range(4)]
    bat.run(40)
    assert not bat.active.any()
    stops = _check_independent(bat, ones, 40)
    assert len(set(stops.tolist())) > 1, stops
    for sched in ('reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        other = _batch('config_freeT', 4, dev, DISTURBED, seed=7, jitter=0.6)
        other.run(40)
        for key in ('state', 'T', 'iters', 'status', 'plant', 'plant_input'):
            assert all(np.array_equal(x, y) for x, y in zip(bat.history[key], other.history[key])), (sched, key)
        assert np.array_equal(bat.X.numpy(), other.X.numpy())


def test_ideal_update_with_the_closed_prediction(emu):
    """ideal_update on, ideal_prediction off: the plant is the spline's own state and input at every
    boundary (the ideal loop's prediction), and state0 of every solve is the kernel's prediction from
    that plant over the plan just solved."""
    import torch
    dev = torch.device('cpu')
    opt = {'ideal_update': True, 'ideal_prediction': False}
    from omg_tools_b200.execution.batch_mpc import _HolonomicAdapter
    bat = _batch('config_freeT', 2, dev, opt, jitter=0.3, seed=5)
    spline = _HolonomicAdapter(None, bat.vehicle, 2, 0., None)
    for k in range(40):
        if not bat.active.any():
            break
        act = bat.active.copy()
        plant0 = bat.plant_x.numpy().copy()
        bat.step()
        T = bat.history['T'][-1]
        idx = np.nonzero(act & (T >= ST))[0]
        if not len(idx):
            continue
        # the plant follows the spline: the ideal prediction (predict_free) of the solution
        spline.predict_free(bat.X[torch.from_numpy(idx)], idx, np.minimum(DT, T[idx]) / T[idx], T[idx],
                            bat.veh_blocks)
        assert np.abs(bat.history['plant'][-1][idx] - spline.state[idx]).max() < 1e-12, k
        assert np.abs(bat.history['plant_input'][-1][idx] - spline.inp[idx]).max() < 1e-12, k
        # state0 of the next solve: the kernel's prediction from the plant at the start of the update
        assert np.array_equal(bat.state[idx], bat.pred_x.numpy()[idx]), k
        n_samp = np.zeros(2, dtype=np.int32)
        n_samp[idx] = _counts(T[idx])[0]
        zeros = [np.zeros((2, 2))] * 4
        pred = twf.plant_step_free(0, bat.X.numpy(), bat.veh_blocks[0], bat.t_index, n_samp, ST, plant0,
                                   np.zeros((2, 2)), zeros, k)
        assert np.abs(pred[2][idx] - bat.state[idx]).max() < 1e-12, k
    assert not bat.active.any()
    assert np.abs(bat.history['plant'][-1] - bat.poseT).max() < 1e-2


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 1024, 4096])
def test_gpu_kernel_matches_the_twin(B):
    """The kernel on the device against the twin, all six models, lag and disturbance off and on;
    the mixed motion times tiled over the batch (beyond the resident blocks at 4096), checked on a
    sample of instances with their own noise keys."""
    rng = np.random.default_rng(B)
    Ts = np.resize(np.array(T_MIX), B) if B >= len(T_MIX) else np.array([3.7])
    check = np.unique(np.r_[np.arange(min(B, len(T_MIX))), rng.integers(0, B, 8), B - 1])
    for model in MODELS:
        for lag, disturb in ((False, False), (True, True)):
            err = _check_twin(model, lag, disturb, Ts, 'cuda', rng, check=check)
            print('B %d model %d lag %d disturb %d: %.1e' % (B, model, lag, disturb, err))
        print('B %d model %d fixed T: %.1e' % (B, model, _check_fixed_T(model, 'cuda', rng)))


@pytest.mark.gpu
@pytest.mark.parametrize('batch', [1, 1024, 4096])
def test_gpu_batch_mpc_follows_the_references_closed_freeT_loop(batch):
    for name in sorted(RUNS):
        _check_golden(name, batch, 'cuda')


def _failed(bat):
    return int(sum((s > 0).sum() for s in bat.history['status']))


@pytest.mark.gpu
@pytest.mark.parametrize('scenario, kw, vopt, max_failed, min_stopped', [
    ('config_freeT', {}, DISTURBED, 24, 256), ('config_dubins_freeT', {'init_v_til': 0.3}, CLOSED, 67, 255)])
def test_gpu_batch_256_closed_freeT(scenario, kw, vopt, max_failed, min_stopped):
    """A jittered batch of 256 closed free-T loops: config_freeT with lag and disturbance, and
    config_dubins_freeT (init_v_til = 0.3) at the reference's defaults; instance 0 is a batch-1 run
    bit for bit.  The closed loops fail more solves than the ideal loops on the same batches, and
    not every Dubins instance stops within 40 steps; measured on an H100 and asserted as such:
    config_freeT fails 24 solves against none in the ideal loop, every instance stops after 16 to 19
    steps; config_dubins_freeT fails 67 against 41, 255 of 256 instances stop within 40 steps.  (With
    lag and disturbance the Dubins batch stops only 93 of 256 instances within 40 steps and fails
    2887 solves: the open disturbed-Dubins item of DESIGN.md section 8.)"""
    import torch
    dev = torch.device('cuda')
    bat = _batch(scenario, 256, dev, vopt, seed=3, jitter=0.1, **kw)
    one = _batch(scenario, 1, dev, vopt, seed=3, **kw)
    ideal = _batch(scenario, 256, dev, {}, seed=3, jitter=0.1, **kw)
    for b in (bat, one, ideal):
        b.run(40)
    act = np.array(bat.history['active'])
    print('%s batch 256: stopped after %s steps (%d stopped), failed solves %d closed / %d ideal'
          % (scenario, np.unique(act.sum(axis=0)), (~bat.active).sum(), _failed(bat), _failed(ideal)))
    assert (~bat.active).sum() >= min_stopped
    n = len(one.history['status'])
    for key in ('status', 'iters', 'T', 'state', 'plant', 'plant_input'):
        assert all(np.array_equal(bat.history[key][k][0], one.history[key][k][0]) for k in range(n)), key
    assert np.array_equal(bat.X[0].cpu().numpy(), one.X[0].cpu().numpy())
    assert _failed(bat) <= max_failed
