"""Device-resident receding-horizon update (include/omg_b200.h omg_mpc_*, execution/device_mpc.py):
the batched Point2Point::update() of the reference's export for one Holonomic / Holonomic3D
vehicle.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu) against the reference's
recorded loops (golden/loop_golden.npz, golden/closed_loop_golden.npz), the host evaluation of the
returned plans and BatchMPC; the ones marked gpu run on the device."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
from test_closed_loop import GOLDEN_TOL  # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

LOOP_GOLDEN = os.path.join(HERE, 'golden', 'loop_golden.npz')
CLOSED_GOLDEN = os.path.join(HERE, 'golden', 'closed_loop_golden.npz')


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _t(a, device):
    import torch
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=device)


def _mpc(pr, batch, device, **kw):
    from omg_tools_b200.execution.device_mpc import DeviceMPC
    import torch
    return DeviceMPC(pr, batch, device=torch.device(device), **kw)


def _obstacles_from_p(desc, p):
    """[B, n_obs, 3 n_dim + 1] obstacle records read back from parameter rows p [B, n_par]."""
    nd, off = desc['n_dim'], desc['obs_off'].reshape(-1, 4)
    out = np.zeros((p.shape[0], desc['n_obs'], 3 * nd + 1))
    for k, (ox, ov, oa, oth) in enumerate(off):
        out[:, k, :nd], out[:, k, nd:2 * nd], out[:, k, 2 * nd:3 * nd] = p[:, ox:ox + nd], p[:, ov:ov + nd], p[:, oa:oa + nd]
        if desc['obs_kind'][k]:
            out[:, k, 3 * nd] = p[:, oth]
    return out


def _batch_obstacles(bat):
    """BatchMPC's current obstacle state as update() takes it."""
    nd = bat.vehicle.n_dim
    out = np.zeros((bat.B, len(bat.obs), 3 * nd + 1))
    for k, d in enumerate(bat.obs):
        out[:, k, :nd], out[:, k, nd:2 * nd], out[:, k, 2 * nd:3 * nd] = d['x'], d['v'], d['a']
        if 'theta' in d:
            out[:, k, 3 * nd] = d['theta'][:, 0]
    return out


def _host_eval(desc, x, tau, T):
    """Value and first derivative / T of the vehicle's columns of the rows x [B, n] at tau: [B, nd] each."""
    from omg_tools_b200.basics.spline import BSplineBasis
    basis = BSplineBasis(desc['knots'], desc['degree'])
    Bd, P1 = basis.derivative(1)
    r0, r1 = basis.eval_basis([tau])[0], Bd.eval_basis([tau]).dot(P1)[0] / T
    L, o = desc['L'], desc['spl_offset']
    cols = [x[:, o + c * L:o + (c + 1) * L] for c in range(desc['n_dim'])]
    return np.stack([c.dot(r0) for c in cols], 1), np.stack([c.dot(r1) for c in cols], 1)


# ---------------------------------------------------------------------------------------------
# the reference's loops
# ---------------------------------------------------------------------------------------------
def _check_loop_golden(name, batch, device, tol=1e-6):
    """golden/loop_golden.npz (the reference's ideal loop): the caller feeds the goal and the obstacles'
    x/v/a/theta from the golden's p; every instance hands the solver the golden's x0 and p."""
    G = np.load(LOOP_GOLDEN)
    pr = getattr(sc, name)()
    desc = b200.mpc_desc(pr, float(G[name + '_dt']))
    mpc = _mpc(pr, batch, device, update_time=float(G[name + '_dt']), trajectory_length=11)
    nd, ps, p0 = desc['n_dim'], desc['p_poseT'], desc['p_state0']
    st0 = _t(np.repeat(G[name + '_p'][0][None, p0:p0 + nd], batch, 0), device)      # (the start)
    for k in range(len(G[name + '_status'])):
        p = np.repeat(G[name + '_p'][k][None], batch, 0)
        _, _, status, _ = mpc.update(st0, _t(p[:, ps:ps + nd], device), _t(_obstacles_from_p(desc, p), device))
        X0, P = (a.cpu().numpy() for a in mpc.last_problem())
        assert np.abs(X0 - G[name + '_x0'][k][None]).max() < tol, (name, k)
        assert np.abs(P - G[name + '_p'][k][None]).max() < tol, (name, k)
        assert np.all(status.cpu().numpy() == G[name + '_status'][k]), (name, k)
    return mpc


def _check_closed_golden(name, batch, device):
    """golden/closed_loop_golden.npz (the reference's loop at its non-ideal defaults) with the
    'integrate' prediction: state0 of update k is the golden's plant state at the start of the previous
    plan (Vehicle.predict's signals['state'][:, -n_samp-1])."""
    G = np.load(CLOSED_GOLDEN)
    dt = float(G[name + '_dt'])
    pr = getattr(sc, name)()
    desc = b200.mpc_desc(pr, dt)
    mpc = _mpc(pr, batch, device, update_time=dt, trajectory_length=11, prediction='integrate')
    nd, ps = desc['n_dim'], desc['p_poseT']
    tx, tp, _ = GOLDEN_TOL
    for k in range(len(G[name + '_status'])):
        p = np.repeat(G[name + '_p'][k][None], batch, 0)
        st0 = np.repeat(G[name + '_plant_state'][max(k - 1, 0)][None], batch, 0)
        _, _, status, iters = mpc.update(_t(st0, device), _t(p[:, ps:ps + nd], device),
                                         _t(_obstacles_from_p(desc, p), device))
        X0, P = (a.cpu().numpy() for a in mpc.last_problem())
        assert np.abs(X0 - G[name + '_x0'][k][None]).max() < tx, (name, k)
        assert np.abs(P - G[name + '_p'][k][None]).max() < tp, (name, k)
        assert np.all(status.cpu().numpy() == G[name + '_status'][k]), (name, k)
        assert np.all(iters.cpu().numpy() == G[name + '_iters'][k]), (name, k)


@pytest.mark.parametrize('name, batch', [('config1', 1), ('config1', 3), ('config5', 1), ('config5', 3)])
def test_follows_the_references_ideal_loop(emu, name, batch):
    """12 updates through the knot crossing at t = 1: x0 and p of every solve within 1e-6 of the
    reference's (the bound the emulated BatchMPC config-5 loop meets against the sequential loop,
    DESIGN.md section 5a), equal statuses."""
    _check_loop_golden(name, batch, 'cpu')


@pytest.mark.parametrize('name', ['config1', 'config5'])
def test_follows_the_references_closed_loop(emu, name):
    """The 'integrate' prediction fed the reference's plant state: x0 and p within GOLDEN_TOL (the
    reference's odeint against RK4 on the same interpolated input), equal statuses and iterations."""
    _check_closed_golden(name, 1, 'cpu')


# ---------------------------------------------------------------------------------------------
# outputs, BatchMPC, per-instance semantics
# ---------------------------------------------------------------------------------------------
# the Holonomic3D example with start and goal off the room's limits (test_gpu_parity.py), so that
# jittered copies stay inside
SCENES = {'config1': sc.config1,
          'config_holonomic3d': lambda: sc.config_holonomic3d(start=(-1.7, -1.7, -1.7), goal=(1.7, 1.7, -1.7))}


def _jittered(name, batch, seed=1, jitter=0.2, device='cpu', **kw):
    """A BatchMPC and a DeviceMPC on the same jittered instances."""
    import torch
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(SCENES[name](), batch=batch, update_time=0.1, jitter=jitter, seed=seed,
                   device=torch.device(device))
    mpc = _mpc(SCENES[name](), batch, device, **kw)
    return bat, mpc


def test_trajectory_outputs_are_the_returned_plans(emu):
    """state_traj / input_traj are the plan's values and derivatives / T at t_rel + k * sample_time,
    to 1e-12 of the host evaluation of the solution (which the next update hands the solver as its
    warm start while no knot is crossed)."""
    bat, mpc = _jittered('config1', 2, trajectory_length=30)
    desc = b200.mpc_desc(bat.problem)
    st0, stT = _t(bat.state, 'cpu'), _t(bat.poseT, 'cpu')
    obs = _t(_batch_obstacles(bat), 'cpu')
    outs = []
    for k in range(4):
        xs, us, status, _ = mpc.update(st0, stT, obs)
        assert np.all(status.numpy() == 0)
        outs.append((xs.numpy().copy(), us.numpy().copy(), mpc.last_problem()[0].numpy()))
    T = desc['horizon']
    for k in range(3):
        xs, us, _ = outs[k]
        X = outs[k + 1][2]                    # the solution of update k
        t_rel = np.round(0.1 * k, 6) % desc['knot_time']
        for j in range(30):
            v, d = _host_eval(desc, X, (t_rel + j * 0.01) / T, T)
            assert np.abs(xs[:, j] - v).max() < 1e-12 and np.abs(us[:, j] - d).max() < 1e-12, (k, j)


@pytest.mark.parametrize('name', ['config1', 'config_holonomic3d'])
def test_agrees_with_batch_mpc(emu, name):
    """A jittered batch of 4, 10 ideal updates: the statuses and iteration counts of BatchMPC, and its
    predicted states (the plan at t + update_time, sample 10 of the trajectory) within 1e-8."""
    bat, mpc = _jittered(name, 4, seed=3, trajectory_length=11)
    st0, stT = _t(bat.state, 'cpu'), _t(bat.poseT, 'cpu')
    for k in range(10):
        obs = _t(_batch_obstacles(bat), 'cpu')
        bat.step()
        xs, us, status, iters = mpc.update(st0, stT, obs)
        assert np.array_equal(status.numpy(), bat.history['status'][-1]), k
        assert np.array_equal(iters.numpy(), bat.history['iters'][-1]), k
        assert np.abs(xs.numpy()[:, 10] - bat.state).max() < 1e-8, k
        assert np.abs(us.numpy()[:, 10] - bat.veh.inp).max() < 1e-8, k
    assert np.allclose(mpc.time, 1.0)


def test_a_failed_solve_keeps_its_instance(emu):
    """Batch of 3; at update 3 an obstacle sits on instance 1's position and its solve fails (max_iter
    30 keeps it cheap).  Its time, warm start and output rows stay as they were and the next update
    does not shift again, while the other instances advance; after recover() its next warm start is
    the cold-start rule (the template with linspace(state0, stateT) in the vehicle's columns)."""
    import torch
    pr = sc.config1()
    pr.problem.set_options({'max_iter': 30, 'feas_steps': 0})
    desc = b200.mpc_desc(pr)
    mpc = _mpc(pr, 3, 'cpu', trajectory_length=5)
    st0 = np.array([[-1.5, -1.5], [-1.4, -1.6], [-1.6, -1.4]])
    stT = np.array([[2., 2.], [2.1, 1.9], [1.9, 2.1]])
    obs0 = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], 3, 0))
    for k in range(3):
        xs, us, status, _ = mpc.update(_t(st0, 'cpu'), _t(stT, 'cpu'), _t(obs0, 'cpu'))
        assert np.all(status.numpy() == 0)
    before = (mpc.time, xs.numpy().copy(), us.numpy().copy())
    obs = obs0.copy()
    obs[1, 0, :2] = xs.numpy()[1, 0]          # (the plan's position at this update's time)
    obs[1, 0, 2:6] = 0.
    xs, us, status, _ = mpc.update(_t(st0, 'cpu'), _t(stT, 'cpu'), _t(obs, 'cpu'))
    st = status.numpy().copy()
    assert st[1] != 0 and st[0] == 0 and st[2] == 0, st
    X0_fail, P_fail = (a.numpy() for a in mpc.last_problem())
    t = mpc.time
    assert t[1] == before[0][1] and np.allclose(t[[0, 2]], before[0][[0, 2]] + 0.1)
    assert np.array_equal(xs.numpy()[1], before[1][1]) and np.array_equal(us.numpy()[1], before[2][1])
    assert not np.array_equal(xs.numpy()[0], before[1][0])
    # the next update starts instance 1 from the warm start it failed from, unshifted, at the same t
    mpc.update(_t(st0, 'cpu'), _t(stT, 'cpu'), _t(obs, 'cpu'))
    X0, P = (a.numpy() for a in mpc.last_problem())
    assert np.array_equal(X0[1], X0_fail[1]) and P[1, desc['p_t']] == P_fail[1, desc['p_t']]
    mpc.recover([False, True, False])
    mpc.update(_t(st0, 'cpu'), _t(stT, 'cpu'), _t(obs0, 'cpu'))
    X0, P = (a.numpy() for a in mpc.last_problem())
    cold = desc['x_template'].copy()
    L, o = desc['L'], desc['spl_offset']
    for c in range(2):
        cold[o + c * L:o + (c + 1) * L] = np.linspace(st0[1, c], stT[1, c], L)
    assert np.array_equal(X0[1], cold)
    assert np.array_equal(P[1, desc['p_state0']:desc['p_state0'] + 2], st0[1])
    assert np.array_equal(P[1, desc['p_input0']:desc['p_input0'] + 2], np.zeros(2))
    assert not np.array_equal(X0[0], cold)


def _run(steps=3):
    """A jittered config-1 batch of 3: the outputs, statuses, iterations and solver rows after every
    update."""
    bat, mpc = _jittered('config1', 3, seed=5, trajectory_length=12)
    obs = _batch_obstacles(bat)
    res = []
    for k in range(steps):
        out = mpc.update(_t(bat.state, 'cpu'), _t(bat.poseT, 'cpu'), _t(obs, 'cpu'))
        res.append([o.numpy().copy() for o in out] + [o.numpy().copy() for o in mpc.last_problem()])
    return res


def test_instances_are_independent_and_schedules_agree(emu, monkeypatch):
    """Instance b of a jittered batch of 3 equals a batch-1 run of that instance bit for bit, and the
    reversed and random thread schedules of the emulation give bit-identical results."""
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    import torch
    full = _run()
    bat = BatchMPC(sc.config1(), batch=3, update_time=0.1, jitter=0.2, seed=5, device=torch.device('cpu'))
    obs = _batch_obstacles(bat)
    for b in (1, 2):
        one = _mpc(sc.config1(), 1, 'cpu', trajectory_length=12)
        for k in range(3):
            out = one.update(_t(bat.state[b:b + 1], 'cpu'), _t(bat.poseT[b:b + 1], 'cpu'), _t(obs[b:b + 1], 'cpu'))
            got = [o.numpy()[0] for o in out] + [o.numpy()[0] for o in one.last_problem()]
            assert all(np.array_equal(g, f[b]) for g, f in zip(got, full[k])), (b, k)
    for sched in ('reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        other = _run()
        assert all(np.array_equal(a, c) for ra, rc in zip(full, other) for a, c in zip(ra, rc)), sched


# ---------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------
def _create(lib, pr, desc, B=2, tl=5, mode=0):
    D, keep = b200.pack_mpc_desc(desc)
    h = lib.omg_mpc_create(pr.problem._handle, C.byref(D), B, tl, mode)
    if h:
        lib.omg_mpc_destroy(h)
        return None
    return lib.omg_last_error().decode()


def test_create_rejects(emu):
    pr = sc.config1()
    desc = b200.mpc_desc(pr)
    assert _create(emu, pr, desc) is None
    assert 'the problem has n = 98' in _create(emu, pr, b200.mpc_desc(sc.config5(build_solver=False)))
    assert 'n_par' in _create(emu, pr, dict(desc, n_par=desc['n_par'] + 1))
    assert 'n = 99' in _create(emu, pr, dict(desc, n=99))
    assert 'trajectory_length 0' in _create(emu, pr, desc, tl=0)
    assert _create(emu, pr, desc, tl=1000) is None
    assert 'trajectory_length 1001 outside 1 .. horizon / sample_time = 1000' in _create(emu, pr, desc, tl=1001)
    assert 'not a multiple of sample_time' in _create(emu, pr, dict(desc, update_time=0.105))
    assert 'not a multiple of sample_time' in _create(emu, pr, dict(desc, update_time=0.005))
    assert 'B must be >= 1' in _create(emu, pr, desc, B=0)
    assert 'B must be >= 1' in _create(emu, pr, desc, B=-3)
    assert 'unknown prediction' in _create(emu, pr, desc, mode=2)
    assert 'vehicle splines' in _create(emu, pr, dict(desc, spl_offset=90))
    assert 'obstacle 0 x/v/a' in _create(emu, pr, dict(desc, obs_off=np.array([16, 8, 10, -1], np.int32)))
    assert 'shift block 0' in _create(emu, pr, dict(desc, shift_off=np.array([80, 65, 87], np.int32)))
    D, keep = b200.pack_mpc_desc(desc)
    assert not emu.omg_mpc_create(None, C.byref(D), 2, 5, 0)
    assert 'null argument' in emu.omg_last_error().decode()


def test_update_rejects_null_buffers(emu):
    import torch
    mpc = _mpc(sc.config1(), 2, 'cpu', trajectory_length=5)
    z = torch.zeros((2, 2), dtype=torch.float64)
    obs = torch.zeros((2, 1, 7), dtype=torch.float64)
    xs, us, st, it = mpc.state_traj, mpc.input_traj, mpc.status, mpc.iters
    args = [mpc._handle, z.data_ptr(), z.data_ptr(), obs.data_ptr(), xs.data_ptr(), us.data_ptr(), st.data_ptr(),
            it.data_ptr(), None]
    for i in range(1, 8):
        bad = list(args)
        bad[i] = None
        assert emu.omg_mpc_update(*bad) == -1
        assert 'null argument' in emu.omg_last_error().decode()
        assert emu.omg_mpc_update_host(*bad[:8]) == -1
    assert emu.omg_mpc_update(None, *args[1:]) == -1
    assert emu.omg_mpc_recover(mpc._handle, None) == -1 and emu.omg_mpc_time(mpc._handle, None) == -1
    assert emu.omg_mpc_last_problem(None, None, None, None) == -1


def test_save_mpc_rejects_what_it_does_not_run(tmp_path):
    from omg_tools_b200 import Holonomic, Environment, Obstacle, Circle, Point2point, Rectangle
    path = str(tmp_path / 'x.omgmpc')
    with pytest.raises(NotImplementedError, match='free motion time'):
        b200.save_mpc(sc.config_freeT(build_solver=False), path)
    with pytest.raises(NotImplementedError, match='one vehicle, this problem has 2'):
        b200.save_mpc(sc.config_interveh_offset(build_solver=False), path)
    with pytest.raises(NotImplementedError, match='not Dubins'):
        b200.save_mpc(sc.config_dubins(build_solver=False), path)
    veh = Holonomic()
    veh.set_initial_conditions([-1.5, -1.5])
    veh.set_terminal_conditions([2., 2.])
    env = Environment(room={'shape': Rectangle(width=5., height=5.)})
    env.add_obstacle(Obstacle({'position': [0., 0.]}, shape=Circle(0.4), options={'spline_traj': True}))
    pr = Point2point(veh, env, options={'horizon_time': 10.})
    with pytest.raises(NotImplementedError, match='spline_traj'):
        b200.save_mpc(pr, path)


# ---------------------------------------------------------------------------------------------
# MPC file and native caller
# ---------------------------------------------------------------------------------------------
def _read_desc(lib, path):
    D = lib.omg_mpc_read(path.encode())
    assert D, lib.omg_last_error().decode()
    d = D.contents
    out = {}
    for name, kind in b200.MPC_FIELDS:
        v = getattr(d, name)
        if kind in 'ID':
            size = {'knots': d.L + d.degree + 1, 'obs_kind': d.n_obs, 'obs_off': 4 * d.n_obs, 'shift_off': d.n_shift,
                    'shift_len': d.n_shift, 'shift_ncol': d.n_shift, 'x_template': d.n, 'p_template': d.n_par,
                    'shift_T': int(sum(np.ctypeslib.as_array(d.shift_len, (d.n_shift,)) ** 2))}[name]
            v = np.ctypeslib.as_array(v, (size,)).copy() if size else np.zeros(0)
        out[name] = v
    lib.omg_mpc_free_desc(D)
    return out


@pytest.mark.parametrize('name', ['config5', 'config_holonomic3d'])
def test_mpc_file_round_trip(emu, tmp_path, name):
    pr = getattr(sc, name)(build_solver=False)
    path = str(tmp_path / 'p.omgmpc')
    b200.save_mpc(pr, path, update_time=0.2, sample_time=0.02)
    desc, back = b200.mpc_desc(pr, 0.2, 0.02), _read_desc(emu, path)
    for key, _ in b200.MPC_FIELDS:
        assert np.array_equal(np.asarray(back[key]), np.asarray(desc[key])), key
    assert not emu.omg_mpc_read(str(tmp_path / 'missing').encode())
    with open(str(tmp_path / 'bad'), 'wb') as fp:
        fp.write(b'OMGTBL\0\0')
    assert not emu.omg_mpc_read(str(tmp_path / 'bad').encode())
    assert 'not an omg MPC file' in emu.omg_last_error().decode()


def _native(tmp_path, lib_args, pr, B, N, tl, st0, stT, obs, prediction='ideal'):
    exe = str(tmp_path / 'native_mpc')
    subprocess.check_call(['g++', '-O2', '-I', os.path.join(ROOT, 'include'),
                           os.path.join(ROOT, 'examples', 'native', 'native_mpc.cpp'), '-o', exe] + lib_args)
    b200.save_tables(pr.father.tables, str(tmp_path / 'p.omgtbl'))
    b200.save_mpc(pr, str(tmp_path / 'p.omgmpc'))
    for key, a in (('s0', st0), ('sT', stT), ('obs', obs)):
        np.ascontiguousarray(a, dtype=np.float64).tofile(str(tmp_path / (key + '.f64')))
    out = subprocess.check_output([exe, str(tmp_path / 'p.omgtbl'), str(tmp_path / 'p.omgmpc'), str(B), str(N), str(tl),
                                   prediction] + [str(tmp_path / (k + '.f64')) for k in ('s0', 'sT', 'obs')] +
                                  [str(tmp_path / 'traj.f64')])
    traj = np.fromfile(str(tmp_path / 'traj.f64')).reshape(N, 2, B, tl, -1)
    lines = [l.split() for l in out.decode().strip().splitlines()]
    return traj, np.array([[int(l[5]), int(l[7])] for l in lines]).reshape(N, B, 2)


def _python_loop(pr, B, N, tl, st0, stT, obs, device, prediction='ideal'):
    """DeviceMPC driven as native_mpc.cpp drives the C call."""
    mpc = _mpc(pr, B, device, trajectory_length=tl, prediction=prediction)
    s0, trajs, stat = st0.copy(), [], []
    for k in range(N):
        xs, us, status, iters = mpc.update(_t(s0, device), _t(stT, device), _t(obs, device))
        xs, us, status = xs.cpu().numpy().copy(), us.cpu().numpy().copy(), status.cpu().numpy()
        ok = status == 0
        s0[ok] = xs[ok, 0]
        trajs.append((xs, us))
        stat.append(np.c_[status, iters.cpu().numpy()])
    return np.array(trajs), np.array(stat)


def test_native_mpc_caller(emu, tmp_path):
    """examples/native/native_mpc.cpp (C++ against the C ABI only: a table file and an MPC file in,
    omg_mpc_update_host) linked to the emulation library reproduces DeviceMPC bit for bit, batch 2 over
    3 updates, both predictions."""
    import torch
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(sc.config1(), batch=2, update_time=0.1, jitter=0.2, seed=2, device=torch.device('cpu'))
    obs = _batch_obstacles(bat)
    for prediction in ('ideal', 'integrate'):
        traj, stat = _native(tmp_path, [emu_support.EMU_LIB, '-Wl,-rpath,' + os.path.dirname(emu_support.EMU_LIB)],
                             sc.config1(build_solver=False), 2, 3, 15, bat.state, bat.poseT, obs, prediction)
        ref, ref_stat = _python_loop(sc.config1(), 2, 3, 15, bat.state, bat.poseT, obs, 'cpu', prediction)
        assert np.array_equal(stat, ref_stat) and np.all(stat[:, :, 0] == 0), prediction
        assert np.array_equal(traj, ref), prediction


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_follows_the_references_loops():
    """Items of the CPU golden tests at batch 1 on the device, with the tolerances of the GPU BatchMPC
    golden tests (1e-6 for the ideal loop, GOLDEN_TOL for the closed one), and the trajectory outputs
    against the host evaluation of the returned plans."""
    for name in ('config1', 'config5'):
        _check_loop_golden(name, 1, 'cuda')
        _check_closed_golden(name, 1, 'cuda')
    bat, mpc = _jittered('config1', 2, device='cuda', trajectory_length=30)
    desc = b200.mpc_desc(bat.problem)
    st0, stT, obs = _t(bat.state, 'cuda'), _t(bat.poseT, 'cuda'), _t(_batch_obstacles(bat), 'cuda')
    prev = None
    for k in range(4):
        xs, us, status, _ = mpc.update(st0, stT, obs)
        X = mpc.last_problem()[0].cpu().numpy()
        if prev is not None:
            t_rel = np.round(0.1 * (k - 1), 6)
            for j in range(30):
                v, d = _host_eval(desc, X, (t_rel + j * 0.01) / desc['horizon'], desc['horizon'])
                assert np.abs(prev[0][:, j] - v).max() < 1e-12 and np.abs(prev[1][:, j] - d).max() < 1e-12, (k, j)
        prev = (xs.cpu().numpy().copy(), us.cpu().numpy().copy())


@pytest.mark.gpu
def test_gpu_batch_1024_matches_batch_1_and_batch_mpc():
    """Config 1, jittered batch of 1024, 20 ideal updates: a spread of instances equals batch-1 runs bit
    for bit, and every status equals BatchMPC's on the same instances.  The iteration counts equal
    BatchMPC's but for a few instance-updates: the ideal prediction is the same spline value rounded
    differently (Cox-de Boor and derivative coefficients on the device, numpy's basis rows times the
    derivative matrix in BatchMPC), and a solve whose convergence test is borderline may take one
    iteration more or less (on the CPU, batch 4, they are all equal: test_agrees_with_batch_mpc)."""
    bat, mpc = _jittered('config1', 1024, seed=7, device='cuda', trajectory_length=11)
    idx = np.array([0, 1, 517, 1023])
    st0, stT = _t(bat.state, 'cuda'), _t(bat.poseT, 'cuda')
    ones = [_mpc(sc.config1(), 1, 'cuda', trajectory_length=11) for _ in idx]
    n_diff = 0
    for k in range(20):
        obs = _batch_obstacles(bat)
        bat.step()
        xs, us, status, iters = mpc.update(st0, stT, _t(obs, 'cuda'))
        assert np.array_equal(status.cpu().numpy(), bat.history['status'][-1]), k
        diff = np.abs(iters.cpu().numpy() - bat.history['iters'][-1])
        n_diff += int((diff != 0).sum())
        assert diff.max() <= 2, k
        full = [o.cpu().numpy() for o in (xs, us, status, iters)] + [o.cpu().numpy() for o in mpc.last_problem()]
        for b, one in zip(idx, ones):
            out = one.update(st0[b:b + 1].contiguous(), stT[b:b + 1].contiguous(), _t(obs[b:b + 1], 'cuda'))
            got = [o.cpu().numpy()[0] for o in out] + [o.cpu().numpy()[0] for o in one.last_problem()]
            assert all(np.array_equal(g, f[b]) for g, f in zip(got, full)), (b, k)
    print('iteration counts that differ from BatchMPC: %d of %d' % (n_diff, 20 * 1024))
    assert n_diff <= 0.01 * 20 * 1024


@pytest.mark.gpu
def test_gpu_updates_replay_from_a_cuda_graph():
    """Updates 2 to 11 captured with torch.cuda.graph on a side stream and replayed give bit-identical
    outputs and times to the eager run: an update neither synchronises nor allocates after the first."""
    import torch
    bat, eager = _jittered('config1', 64, seed=3, device='cuda', trajectory_length=20)
    graphed = _mpc(sc.config1(), 64, 'cuda', trajectory_length=20)
    st0, stT, obs = _t(bat.state, 'cuda'), _t(bat.poseT, 'cuda'), _t(_batch_obstacles(bat), 'cuda')
    ref = []
    for k in range(11):
        ref.append([o.clone() for o in eager.update(st0, stT, obs)])
    graphed.update(st0, stT, obs)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    outs = []
    side = torch.cuda.Stream()
    with torch.cuda.graph(g, stream=side):
        for k in range(10):
            outs.append([o.clone() for o in graphed.update(st0, stT, obs)])
    g.replay()
    torch.cuda.synchronize()
    for k in range(10):
        for a, b in zip(outs[k], ref[k + 1]):
            assert torch.equal(a, b), k
    assert np.array_equal(graphed.time, eager.time)


@pytest.mark.gpu
def test_gpu_native_mpc_caller(tmp_path):
    """native_mpc.cpp against libomgb200.so is bit-identical to the Python binding."""
    import torch
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    lib_dir = os.path.join(ROOT, 'omg_tools_b200', 'csrc')
    bat = BatchMPC(sc.config1(), batch=3, update_time=0.1, jitter=0.2, seed=4, device=torch.device('cuda'))
    obs = _batch_obstacles(bat)
    traj, stat = _native(tmp_path, ['-L', lib_dir, '-lomgb200', '-Wl,-rpath,' + lib_dir],
                         sc.config1(build_solver=False), 3, 4, 15, bat.state, bat.poseT, obs)
    ref, ref_stat = _python_loop(sc.config1(), 3, 4, 15, bat.state, bat.poseT, obs, 'cuda')
    assert np.array_equal(stat, ref_stat)
    assert np.array_equal(traj, ref)
