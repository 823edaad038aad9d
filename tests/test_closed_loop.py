"""Closed-loop MPC through the vehicle's own dynamics: omg_closed_loop_step (non-ideal
Vehicle.simulate / predict with input disturbance and first-order actuator lag) and the
closed-loop path of execution/batch_mpc.py.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu) against the numpy
twin (tests/plant_twin.py), scipy and the reference's recorded closed loop
(golden/closed_loop_golden.npz, make_closed_loop_golden.py); the ones marked gpu run the same
checks on the device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
import plant_twin as tw                  # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'closed_loop_golden.npz')
IDENTITY = np.r_[1., 0., 0., 0., 1., 0., 0., 0., 0., 0., 0.]     # b = a = [1, 0, 0, 0], zi = 0
DIST = {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _call(model, X, L, R0, R1, px, pu, step, seed=0, tau=None, dist=None, dt=0.01, device='cpu'):
    """The kernel through the binding; dist = (filt, mean, stdev, n_traj).  Returns numpy."""
    import torch
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=device)
    X, px, pu = t(X), t(px), t(pu)
    out = [torch.empty_like(px), torch.empty_like(pu), torch.empty_like(px), torch.empty_like(pu)]
    d = None
    if dist is not None:
        filt, mean, sd, n_traj = dist
        scratch = torch.empty(X.shape[0] * pu.shape[1] * (n_traj + 24), dtype=torch.float64, device=device)
        d = (filt, mean, sd, n_traj, scratch)
    b200.closed_loop_step(model, X, L, R0, R1, dt, px, pu, out, step, seed=seed, time_constant=tau,
                          disturbance=d)
    return [o.cpu().numpy() for o in out]


def _kernel_disturbance(filt, B, ni, n_traj, samples, seed, step, mean, sd, device='cpu'):
    """Disturbance samples [B, ni, len(samples)] as the kernel draws and filters them: with
    zero planned input and no lag, the applied input at sample s is the disturbance itself."""
    out = []
    for s in samples:
        Z = np.zeros((s + 1, 1))
        r = _call(0, np.zeros((B, ni)), 1, Z, Z, np.zeros((B, ni)), np.zeros((B, ni)), step, seed=seed,
                  dist=(filt, mean, sd, n_traj), device=device)
        out.append(r[1])
    return np.stack(out, axis=2)


def _twin_disturbance(B, ni, n_traj, seed, step, fc, mean, sd):
    return np.array([tw.disturbance(seed, step, b, ni, n_traj, fc, mean, sd) for b in range(B)])


# ---------------------------------------------------------------------------------------------
# generator and filter
# ---------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's known-answer vectors of philox4x32-10."""
    z = tw.philox4x32_10(np.zeros((1, 4), np.uint64), (0, 0))[0]
    assert [int(v) for v in z] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    f = tw.philox4x32_10(np.full((1, 4), 0xffffffff, np.uint64), (0xffffffff, 0xffffffff))[0]
    assert [int(v) for v in f] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    c = np.array([[0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344]], np.uint64)
    p = tw.philox4x32_10(c, (0xa4093822, 0x299f31d0))[0]
    assert [int(v) for v in p] == [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_kernel_white_noise_matches_the_twin(emu):
    """Identity filter, mean 0, stdev 1: the kernel's disturbance is its raw normals.  The
    uniforms are the same bits (Philox and the 52-bit conversion are integer and exact), so the
    normals differ only by the last bits of log, cos and sin: at most 4 ulp of max(|z|, 1)."""
    B, ni, n_traj = 3, 3, 40
    k = _kernel_disturbance(IDENTITY, B, ni, n_traj, range(n_traj), 11, 4, np.zeros(ni), np.ones(ni))
    t = np.array([[tw.normals(11, 4, b, j, n_traj) for j in range(ni)] for b in range(B)])
    assert np.all(np.abs(k - t) <= 4 * np.spacing(np.maximum(np.abs(t), 1.)))


def test_kernel_filter_matches_scipy_filtfilt(emu):
    """butter(3, fc) + filtfilt over the whole stored trajectory, first samples kept: the
    kernel's passes match scipy.signal.filtfilt on the same white noise to 1e-12."""
    B, ni, n_traj = 2, 2, 301
    mean, sd = np.array([0.1, -0.2]), np.array([0.05, 0.3])
    for fc in (0.01, 0.3):
        samples = list(range(0, 12)) + [40, 150, 300]
        k = _kernel_disturbance(b200.disturbance_filter(fc), B, ni, n_traj, samples, 3, 7, mean, sd)
        t = _twin_disturbance(B, ni, n_traj, 3, 7, fc, mean, sd)[:, :, samples]
        assert np.abs(k - t).max() < 1e-12, fc


def test_normal_statistics_and_keys():
    """Raw draws: mean and standard deviation within 4 sigma of 0 and 1; the uniforms lie in
    (0, 1).  Changing the seed, step, instance or signal changes the whole stream."""
    n = 200000
    z = np.concatenate([tw.normals(1, s, 0, 0, n // 4) for s in range(4)])
    assert abs(z.mean()) < 4 / np.sqrt(n)
    assert abs(z.std() - 1.) < 4 * np.sqrt(0.5 / n)
    u1, u2 = tw.uniforms(1, 0, 0, 0, n)
    assert 0 < min(u1.min(), u2.min()) and max(u1.max(), u2.max()) < 1
    base = tw.normals(1, 2, 3, 1, 64)
    for key in ((2, 2, 3, 1), (1, 3, 3, 1), (1, 2, 4, 1), (1, 2, 3, 0), (1 << 40, 2, 3, 1)):
        other = tw.normals(*key, 64)
        assert np.count_nonzero(other == base) == 0, key


# ---------------------------------------------------------------------------------------------
# inputs and integrator
# ---------------------------------------------------------------------------------------------
def _holonomic_case(rng, B=4):
    from omg_tools_b200.execution.batch_mpc import plant_rows
    pr = sc.config1(build_solver=False)
    veh, T = pr.vehicles[0], pr.options['horizon_time']
    L = len(veh.basis)
    X = np.cumsum(0.2 * rng.standard_normal((B, 2, L)), axis=2).reshape(B, 2 * L)
    R0, R1 = plant_rows(veh.basis, T, 0.3, 0.01, 10)
    return veh, T, L, X, R0, R1


def _quadrotor_case(rng, B=4):
    from omg_tools_b200.execution.batch_mpc import plant_rows
    pr = sc.config4(build_solver=False)
    veh, T = pr.vehicles[0], pr.options['horizon_time']
    L = len(veh.basis)
    X = np.zeros((B, pr.father.tables.n))
    X[:, :L] = 9.81 / 1.0 + 0.5 * rng.standard_normal((B, L))
    X[:, L:3 * L] = 0.1 * rng.standard_normal((B, 2 * L))
    R0, R1 = plant_rows(veh.basis, T, 0.2, 0.01, 40)
    return veh, T, L, X, R0, R1


def test_input_samples_match_splines2signals(emu):
    """The planned inputs on the device (and the twin's) are the vehicle's own splines2signals
    at the samples of one update, to 1e-13."""
    from omg_tools_b200.basics.spline import BSpline
    rng = np.random.default_rng(2)
    for model, case, ns, ni, t_rel, n_samp in ((0, _holonomic_case, 2, 2, 0.3, 10), (1, _quadrotor_case, 8, 3, 0.2, 40)):
        veh, T, L, X, R0, R1 = case(rng)
        time = t_rel + 0.01 * np.arange(n_samp + 1)
        px = np.zeros((X.shape[0], ns))
        if model == 1:
            veh.prediction['state'] = np.zeros(8)
        out = _call(model, X, L, R0, R1, px, np.zeros((X.shape[0], ni)), 0, dt=0.01)
        for b in range(X.shape[0]):
            spl = [BSpline(veh.basis, X[b, c * L:(c + 1) * L]).scale(T) for c in range(ni)]
            ref = np.atleast_2d(veh.splines2signals(spl, time)['input'])
            twin = tw.planned_inputs(model, X[b], L, R0, R1, ni).T
            scale = max(1., np.abs(ref).max())
            assert np.abs(twin - ref).max() < 1e-13 * scale, (model, b)
            assert np.abs(out[3][b] - ref[:, -1]).max() < 1e-13 * scale, (model, b)


@pytest.mark.parametrize('lag, disturb', [(False, False), (True, False), (False, True), (True, True)])
def test_kernel_matches_the_twin(emu, lag, disturb):
    """Plant and predicted state and input against the twin, with and without the lag and the
    disturbance: 1e-13 for the integrator model, 1e-12 (relative to the largest value) for
    Quadrotor3D."""
    rng = np.random.default_rng(3)
    for model, case, ns, ni, tol in ((0, _holonomic_case, 2, 2, 1e-13), (1, _quadrotor_case, 8, 3, 1e-12)):
        veh, T, L, X, R0, R1 = case(rng)
        B = X.shape[0]
        px = 0.1 * rng.standard_normal((B, ns))
        pu = tw.planned_inputs(model, X[0], L, R0, R1, ni)[0] + 0.05 * rng.standard_normal((B, ni))
        n_traj = 150
        spec = (0.05, 0.02 * np.ones(ni), 0.1 * np.ones(ni), n_traj) if disturb else None
        dist = (b200.disturbance_filter(0.05),) + spec[1:] if disturb else None
        out = _call(model, X, L, R0, R1, px, pu, 6, seed=9, tau=0.1 if lag else None, dist=dist)
        ref = tw.plant_step(model, X, L, R0, R1, 0.01, px, pu, 6, seed=9, time_constant=0.1 if lag else None,
                            disturbance_spec=spec)
        for o, r in zip(out, ref):
            assert np.abs(o - r).max() < tol * max(1., np.abs(r).max()), model
        if not lag and not disturb:
            assert np.array_equal(out[0], out[2]) and np.array_equal(out[1], out[3])


def test_twin_integrator_matches_odeint():
    """The RK4 rule on the linearly interpolated input against scipy's odeint on the same input
    (what the reference integrates): the difference is odeint's own error at its default
    tolerances.  Measured: 2.2e-7 for the integrator model over 0.1 s (RK4 is exact there) and
    3.4e-7 for its lag; 5.7e-7 for Quadrotor3D over 0.4 s and 1.8e-6 for its lag (thrust ~10)."""
    from scipy.integrate import odeint
    rng = np.random.default_rng(4)
    dt = 0.01
    for model, case, ns, ni in ((0, _holonomic_case, 2, 2), (1, _quadrotor_case, 8, 3)):
        veh, T, L, X, R0, R1 = case(rng, B=1)
        U = tw.planned_inputs(model, X[0], L, R0, R1, ni)
        n = U.shape[0] - 1
        tg = dt * np.arange(n + 1)
        interp = lambda t: np.array([np.interp(t, tg, U[:, c]) for c in range(ni)])
        x0 = np.r_[0.1 * rng.standard_normal(ns)]
        ref = odeint(lambda x, t: tw.ode(model, x, interp(t)), x0, tg)
        mine = tw.rk4(lambda x, u: tw.ode(model, x, u), x0, U, dt)
        err = np.abs(mine - ref).max()
        lag_ref = odeint(lambda u, t: (interp(t) - u) / 0.1, U[0] + 0.3, tg)
        lag_mine = tw.rk4(lambda u, c: (c - u) / 0.1, U[0] + 0.3, U, dt)
        err_lag = np.abs(lag_mine - lag_ref).max()
        print('odeint vs RK4, model %d: state %.1e, lag %.1e' % (model, err, err_lag))
        assert err < 1e-6 and err_lag < 5e-6, model


def _valid_args(buf):
    """A valid argument list of omg_closed_loop_step (integrator, B = 1, host pointers)."""
    def p(name, a):
        buf[name] = np.ascontiguousarray(a, dtype=np.float64)
        return buf[name].ctypes.data
    L, n_samp, n_traj = 3, 2, 20
    return [0, 1, 2, 2, 2 * L, p('x', np.ones(2 * L)), L, n_samp, p('R0', np.ones((3, L))), p('R1', np.ones((3, L))),
            0.01, 1, 0.1, 1, n_traj, p('filt', IDENTITY), p('mean', np.zeros(2)), p('sd', np.ones(2)), 1, 0,
            p('px', np.zeros(2)), p('pu', np.zeros(2)), p('px1', np.zeros(2)), p('pu1', np.zeros(2)),
            p('qx', np.zeros(2)), p('qu', np.zeros(2)), p('scr', np.zeros(2 * (n_traj + 24))), None]


@pytest.mark.parametrize('index, value, message', [
    (0, 2, 'unknown vehicle model'), (0, 7, 'unknown vehicle model'), (0, -1, 'unknown vehicle model'),
    (14, 12, 'n_traj'), (14, 5, 'n_traj'), (12, 0.0, 'time_constant'), (12, -0.1, 'time_constant'),
    (10, 0.0, 'sample_time'), (2, 3, 'sizes'), (7, -1, 'sizes'), (7, 1024, 'exceeds 2048'),
    (5, None, 'null'), (8, None, 'null'), (20, None, 'null'), (23, None, 'null'), (26, None, 'null'),
    (15, None, 'null')])
def test_bad_arguments_are_rejected(emu, index, value, message):
    buf = {}
    args = _valid_args(buf)
    assert emu.omg_closed_loop_step(*args) == 0
    args[index] = value
    assert emu.omg_closed_loop_step(*args) == -1
    assert message in emu.omg_last_error().decode()


def test_lag_and_disturbance_switches_relax_their_checks(emu):
    """n_traj, the filter and the scratch only matter with the disturbance, the time constant
    only with the lag."""
    buf = {}
    args = _valid_args(buf)
    args[11], args[12], args[13], args[14] = 0, 0.0, 0, 0
    args[15] = args[16] = args[17] = args[26] = None
    assert emu.omg_closed_loop_step(*args) == 0


# ---------------------------------------------------------------------------------------------
# BatchMPC
# ---------------------------------------------------------------------------------------------
def _batch(name, batch, device, seed=0, vehicle_options=None, **kw):
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    pr = getattr(sc, name)()
    pr.vehicles[0].set_options(vehicle_options or {})
    return BatchMPC(pr, batch=batch, update_time=kw.pop('update_time', 0.1), device=device, seed=seed, **kw)


def _record_solves(bat):
    calls = []
    solve = bat.solver.solve_batch_device

    def rec(X0, P, *a, **kw):
        calls.append((X0.cpu().numpy().copy(), P.cpu().numpy().copy()))
        return solve(X0, P, *a, **kw)
    bat.solver.solve_batch_device = rec
    return calls


GOLDEN_RUNS = [('config1', 1), ('config1', 3), ('config5', 1), ('config5', 3), ('config4', 1), ('config4', 3),
               ('config_disturbances', 1), ('config_disturbances', 3)]
# (x0, p, plant state): the reference integrates with odeint at its default tolerances, the kernel
# with RK4 on the same interpolated input; measured at most 4.8e-6 in x0, 1.9e-6 in p and
# 1.9e-6 in the plant state (config 1), 4.7e-6 / 1.7e-6 / 1.7e-6 (config 5), 1.8e-7 / 6.6e-7 /
# 1.8e-6 (config 4)
GOLDEN_TOL = (1e-5, 5e-6, 5e-6)


def _check_golden(name, batch, device):
    import torch
    G = np.load(GOLDEN)
    dt = float(G[name + '_dt'])
    n_steps = len(G[name + '_status']) if name != 'config4' else 2      # config 4: up to the knot crossing
    bat = _batch(name, batch, torch.device(device), update_time=dt,
                 vehicle_options={'ideal_prediction': False, 'ideal_update': False})
    calls = _record_solves(bat)
    bat.run(n_steps)
    tx, tp, ts = GOLDEN_TOL
    # the golden's noise is instance 0's: with the disturbance only instance 0 repeats it
    b = slice(0, 1) if name == 'config_disturbances' else slice(None)
    for k in range(n_steps):
        X0, P = calls[k]
        h = lambda key: bat.history[key][k + 1][b]
        assert np.abs(X0[b] - G[name + '_x0'][k][None]).max() < tx, (name, k)
        assert np.abs(P[b] - G[name + '_p'][k][None]).max() < tp, (name, k)
        assert np.all(bat.history['status'][k][b] == G[name + '_status'][k])
        assert np.all(bat.history['iters'][k][b] == G[name + '_iters'][k]), (k, bat.history['iters'][k])
        assert np.abs(h('plant') - G[name + '_plant_state'][k + 1][None]).max() < ts, (name, k)
        assert np.abs(h('plant_input') - G[name + '_plant_input'][k + 1][None]).max() < ts, (name, k)
    return bat


@pytest.mark.parametrize('name, batch', GOLDEN_RUNS)
def test_batch_mpc_follows_the_references_closed_loop(emu, name, batch):
    """golden/closed_loop_golden.npz: the reference's predict / solve / store / simulate loop at
    its own (non-ideal) vehicle defaults, and p2p_holonomic_disturbances.py with the lag and the
    disturbance (the reference's add_disturbance, filtfilt, interp1d and odeint on the white
    noise of the device generator, instance 0).  BatchMPC hands the solver the same x0 and p at
    every step, every instance of a batch of identical copies (instance 0 with the
    disturbance: the others draw their own noise), to GOLDEN_TOL (odeint's tolerance);
    statuses and iteration counts are equal and the plant state and applied input follow the
    reference's simulated signals."""
    import torch
    _check_golden(name, batch, 'cpu')


def test_ideal_flags_run_the_existing_path(emu, monkeypatch):
    """Both flags on (this repository's defaults): no plant step is launched, the history has
    the keys it always had, and it is bit-identical to the history recorded from the commit
    before the closed loop was added (golden/make_ideal_history_golden.py: config 5, jittered
    batch of 2, 12 steps through the knot crossing)."""
    import torch
    sys.path.insert(0, os.path.join(HERE, 'golden'))
    import make_ideal_history_golden as ig

    def refuse(*a, **kw):
        raise AssertionError('closed_loop_step called on the ideal path')
    monkeypatch.setattr(b200, 'closed_loop_step', refuse)
    bat = _batch('config5', ig.BATCH, torch.device('cpu'), seed=ig.SEED, jitter=ig.JITTER)
    assert not bat.closed_loop
    bat.run(ig.STEPS)
    assert sorted(bat.history) == ['iters', 'state', 'status']
    G = np.load(ig.OUT)
    for key in ('state', 'iters', 'status'):
        assert np.array_equal(np.array(bat.history[key]), G[key]), key
    assert np.array_equal(bat.X.numpy(), G['X'])


def test_mixed_flags(emu):
    """Exactly one flag off.  ideal_update on: the plant is the spline (lag and disturbance do
    not apply, as in the reference's simulate) and the prediction integrates the planned inputs
    from it.  ideal_prediction
    on: the prediction is the spline value, the plant integrates the lagged input.  (With
    ideal_update on the prediction integrates the new plan from the plant state of the previous
    boundary, as the reference's predict does, so it is not the new spline's value.)"""
    import torch
    from omg_tools_b200.execution.batch_mpc import plant_rows
    dev = torch.device('cpu')
    ideal = _batch('config5', 2, dev, jitter=0.05)
    upd = _batch('config5', 2, dev, jitter=0.05,
                 vehicle_options={'ideal_prediction': False, '1storder_delay': True, 'input_disturbance': DIST})
    pred = _batch('config5', 2, dev, jitter=0.05, vehicle_options={'ideal_update': False, '1storder_delay': True})
    assert upd.time_constant is None and upd.disturbance is None and pred.time_constant == 0.1
    L = len(pred.vehicle.basis)
    for k in range(4):
        px, pu = pred.plant_x.numpy().copy(), pred.plant_u.numpy().copy()
        ux = upd.plant_x.numpy().copy()
        t_rel = np.round(pred.time, 6) % pred.knot_time
        for bat in (ideal, upd, pred):
            bat.step()
        R0, R1 = plant_rows(pred.vehicle.basis, pred.T, t_rel, 0.01, 10)
        spline = lambda X: np.array([[R0[-1].dot(X[b, c * L:(c + 1) * L]) for c in range(2)] for b in range(2)])
        assert np.abs(upd.history['plant'][-1] - spline(upd.X.numpy())).max() < 1e-12, k
        ref = tw.plant_step(0, upd.X.numpy(), L, R0, R1, 0.01, ux, np.zeros((2, 2)), k)
        assert np.abs(upd.state - ref[2]).max() < 1e-13, k
        assert np.array_equal(upd.history['status'][-1], ideal.history['status'][-1])
        X = pred.X.numpy()
        assert np.abs(pred.state - spline(X)).max() < 1e-12, k
        ref = tw.plant_step(0, X, L, R0, R1, 0.01, px, pu, k, time_constant=0.1)
        assert np.abs(pred.history['plant'][-1] - ref[0]).max() < 1e-13, k
        assert np.abs(pred.history['plant_input'][-1] - ref[1]).max() < 1e-13, k


def _disturbed(seed, batch=2, steps=3):
    import torch
    bat = _batch('config5', batch, torch.device('cpu'), seed=seed,
                 vehicle_options={'ideal_prediction': False, 'ideal_update': False, '1storder_delay': True,
                                  'time_constant': 0.1, 'input_disturbance': DIST})
    bat.run(steps)
    return bat


def test_same_seed_same_history_and_schedules_agree(emu, monkeypatch):
    """Config 5 with lag and disturbance: the same seed gives a bit-identical history, another
    seed another plant path, and the reversed and random thread schedules of the emulation give
    bit-identical plant states."""
    a, b = _disturbed(5), _disturbed(5)
    for key in a.history:
        assert all(np.array_equal(x, y) for x, y in zip(a.history[key], b.history[key])), key
    c = _disturbed(6)
    assert not np.array_equal(a.history['plant'][-1], c.history['plant'][-1])
    for sched in ('reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        d = _disturbed(5)
        assert all(np.array_equal(x, y) for x, y in zip(a.history['plant'], d.history['plant'])), sched


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 1024, 4096])
def test_gpu_kernel_matches_the_twin(B):
    """The device kernel against the twin with lag and disturbance on a spread of instances of
    each batch.  1e-12 for Quadrotor3D as on the CPU; 5e-13 for the integrator model (CPU: 1e-13):
    nvcc fuses the multiply-adds of the filter recursion, whose poles at fc = 0.01 lie close to 1
    and carry the rounding differences along (measured 1.7e-13 on an H100)."""
    rng = np.random.default_rng(B)
    for model, case, ns, ni, tol in ((0, _holonomic_case, 2, 2, 5e-13), (1, _quadrotor_case, 8, 3, 1e-12)):
        veh, T, L, X, R0, R1 = case(rng, B=B)
        px = 0.1 * rng.standard_normal((B, ns))
        pu = tw.planned_inputs(model, X[0], L, R0, R1, ni)[0] + 0.05 * rng.standard_normal((B, ni))
        spec = (0.01, 0.02 * np.ones(ni), 0.05 * np.ones(ni), 901)
        out = _call(model, X, L, R0, R1, px, pu, 3, seed=12, tau=0.1,
                    dist=(b200.disturbance_filter(0.01),) + spec[1:], device='cuda')
        idx = np.unique(np.r_[0, B - 1, rng.integers(0, B, 6)])
        ref = tw.plant_step(model, X[idx], L, R0, R1, 0.01, px[idx], pu[idx], 3, seed=12, time_constant=0.1,
                            disturbance_spec=spec, instances=idx)
        for o, r in zip(out, ref):
            assert np.abs(o[idx] - r).max() < tol * max(1., np.abs(r).max()), (model, B)


@pytest.mark.gpu
def test_gpu_batch_mpc_follows_the_references_closed_loop():
    for name in ('config1', 'config5', 'config4', 'config_disturbances'):
        _check_golden(name, 1, 'cuda')


@pytest.mark.gpu
def test_gpu_config5_batch_256_closed_loop():
    """Config 5, batch 256 x 50 steps with lag and disturbance.  Every step's plant step equals
    the twin fed the device's own spline coefficients; instance 0 equals the batch-1 run bit
    for bit (the noise is keyed by instance, not by batch position in a launch)."""
    import torch
    from omg_tools_b200.execution.batch_mpc import plant_rows
    opts = {'ideal_prediction': False, 'ideal_update': False, '1storder_delay': True, 'time_constant': 0.1,
            'input_disturbance': DIST}
    bat = _batch('config5', 256, torch.device('cuda'), seed=3, vehicle_options=opts)
    one = _batch('config5', 1, torch.device('cuda'), seed=3, vehicle_options=opts)
    filt = (0.01, np.zeros(2), DIST['stdev'])
    idx = np.array([0, 1, 77, 255])
    for k in range(50):
        px, pu = bat.plant_x.cpu().numpy().copy(), bat.plant_u.cpu().numpy().copy()
        t_rel = np.round(bat.time, 6) % bat.knot_time
        bat.step()
        one.step()
        X = bat.X.cpu().numpy()
        R0, R1 = plant_rows(bat.vehicle.basis, bat.T, t_rel, 0.01, 10)
        n_traj = int(np.round((bat.T - t_rel) / 0.01, 6)) + 1
        ref = tw.plant_step(0, X[idx], len(bat.vehicle.basis), R0, R1, 0.01, px[idx], pu[idx], k, seed=3,
                            time_constant=0.1, disturbance_spec=filt + (n_traj,), instances=idx)
        assert np.abs(bat.history['plant'][-1][idx] - ref[0]).max() < 1e-13, k
        assert np.abs(bat.state[idx] - ref[2]).max() < 1e-13, k
        assert np.array_equal(bat.history['plant'][-1][0], one.history['plant'][-1][0]), k
        assert np.array_equal(bat.history['iters'][-1][0], one.history['iters'][-1][0]), k


@pytest.mark.gpu
def test_gpu_config4_batch_64_closed_loop_fails_no_more_than_the_ideal_loop():
    import torch
    closed = _batch('config4', 64, torch.device('cuda'), jitter=0.05, update_time=0.4,
                    vehicle_options={'ideal_prediction': False, 'ideal_update': False})
    ideal = _batch('config4', 64, torch.device('cuda'), jitter=0.05, update_time=0.4)
    closed.run(5)
    ideal.run(5)
    for k in range(5):
        bad_closed = closed.history['status'][k] != 0
        bad_ideal = ideal.history['status'][k] != 0
        assert not np.any(bad_closed & ~bad_ideal), (k, closed.history['status'][k], ideal.history['status'][k])
