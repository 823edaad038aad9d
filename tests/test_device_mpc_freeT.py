"""Device-resident receding-horizon update with a free motion time (include/omg_b200.h
omg_mpc_create_freet, execution/device_mpc.py): the batched FreeTPoint2point loop for one Holonomic /
Holonomic3D vehicle, and the solve on a row list (omg_solve_batch_rows) that keeps stopped instances
out of it.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu) against BatchMPC's free-T
loop, the reference's recorded loops (golden/freeT_loop_golden.npz,
golden/freeT_closed_loop_golden.npz) and the host evaluation of the returned plans; the ones marked
gpu run on the device."""
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
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

LOOP_GOLDEN = os.path.join(HERE, 'golden', 'freeT_loop_golden.npz')
CLOSED_GOLDEN = os.path.join(HERE, 'golden', 'freeT_closed_loop_golden.npz')
DT = 0.5


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _t(a, device):
    import torch
    return torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=device)


def _holonomic3d_freeT(build_solver=True):
    """config_holonomic3d's vehicle and room with a free motion time: start and goal inside the room's
    limits, so that jittered copies stay inside, and at different heights (with a zero step in one
    column of one instance, numpy's linspace takes another rounding path for every instance of
    BatchMPC's cold start)."""
    from omg_tools_b200 import Holonomic3D, Plate, Cube, Cuboid, RegularPrisma, Rectangle, Environment, Obstacle
    vehicle = Holonomic3D(Plate(Rectangle(0.5, 1.), height=0.1))
    vehicle.set_initial_conditions([-1.7, -1.7, -1.7])
    vehicle.set_terminal_conditions([1.7, 1.7, -1.6])
    environment = Environment(room={'shape': Cube(5.)})
    environment.add_obstacle(Obstacle(
        {'position': [0., 0., -1.5]}, shape=Cuboid(width=0.5, depth=4., height=2.)))
    trajectories = {'velocity': {'time': [4.], 'values': [[0.0, 0.0, 1.]]}}
    environment.add_obstacle(Obstacle(
        {'position': [1., 1., -2.25]}, shape=RegularPrisma(0.25, 0.25, 6),
        simulation={'trajectories': trajectories}))
    return sc._p2p(vehicle, environment, {'hard_term_con': True}, build_solver, freeT=True)


SCENES = {'config_freeT': sc.config_freeT, 'config_freeT_moving': sc.config_freeT_moving,
          'holonomic3d_freeT': _holonomic3d_freeT}


def _mpc(pr, batch, device, **kw):
    from omg_tools_b200.execution.device_mpc import DeviceMPC
    import torch
    kw.setdefault('update_time', DT)
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


def _record_solves(bat):
    """What every BatchMPC solve is handed: (x0, p) of the instances solved."""
    calls = []
    solve = bat.solver.solve_batch_device

    def rec(X0, P, *a, **kw):
        calls.append((X0.cpu().numpy().copy(), P.cpu().numpy().copy()))
        return solve(X0, P, *a, **kw)
    bat.solver.solve_batch_device = rec
    return calls


def _host_eval(desc, x, tau, T):
    """Value and first derivative / T of the vehicle's columns of the rows x [B, n] at tau [B]."""
    from omg_tools_b200.basics.spline import BSplineBasis
    basis = BSplineBasis(desc['knots'], desc['degree'])
    Bd, P1 = basis.derivative(1)
    L, o = desc['L'], desc['spl_offset']
    v, d = np.zeros((len(x), desc['n_dim'])), np.zeros((len(x), desc['n_dim']))
    for b in range(len(x)):
        r0, r1 = basis.eval_basis([tau[b]])[0], Bd.eval_basis([tau[b]]).dot(P1)[0] / T[b]
        for c in range(desc['n_dim']):
            col = x[b, o + c * L:o + (c + 1) * L]
            v[b, c], d[b, c] = col.dot(r0), col.dot(r1)
    return v, d


# ---------------------------------------------------------------------------------------------
# BatchMPC
# ---------------------------------------------------------------------------------------------
def _jittered(name, batch, seed=1, jitter=0.2, device='cpu', **kw):
    """A BatchMPC and a DeviceMPC on the same jittered instances."""
    import torch
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(SCENES[name](), batch=batch, update_time=DT, jitter=jitter, seed=seed, device=torch.device(device))
    return bat, _mpc(SCENES[name](), batch, device, **kw)


def _against_batch_mpc(name, batch, device, seed=1, max_steps=40, finish=True):
    """Runs BatchMPC and DeviceMPC side by side until every instance has stopped; returns the
    per-update comparisons and the stop steps."""
    bat, mpc = _jittered(name, batch, seed=seed, device=device, trajectory_length=20)
    calls = _record_solves(bat)
    desc = b200.mpc_freeT_desc(bat.problem, DT)
    st0, stT = _t(bat.state, device), _t(bat.poseT, device)
    out = []
    for k in range(max_steps):
        if not bat.active.any():
            break
        obs = _t(_batch_obstacles(bat), device)
        act = np.nonzero(bat.active)[0]
        bat.step()
        _, _, status, iters = mpc.update(st0, stT, obs)
        X0, P = (a.cpu().numpy() for a in mpc.last_problem())
        out.append(dict(status=status.cpu().numpy().copy(), iters=iters.cpu().numpy().copy(),
                        T=mpc.motion_time().cpu().numpy(), X0=X0[act], P=P[act], act=act,
                        ref_X0=calls[-1][0], ref_P=calls[-1][1], ref_status=bat.history['status'][-1],
                        ref_iters=bat.history['iters'][-1], ref_T=bat.history['T'][-1]))
    if finish:
        assert not bat.active.any()
        # one more update: every instance is stopped, nothing is solved
        _, _, status, iters = mpc.update(st0, stT, _t(_batch_obstacles(bat), device))
        assert np.all(status.cpu().numpy() == b200.MPC_STOPPED) and np.all(iters.cpu().numpy() == 0)
    return out, desc


@pytest.mark.parametrize('name', ['config_freeT', 'holonomic3d_freeT'])
def test_agrees_with_batch_mpc(emu, name):
    """A jittered batch of 4, ideal, until every instance has stopped: x0 and p of every solve equal
    BatchMPC's bit for bit (the same shift and evaluation arithmetic), and so do the statuses (-1 where
    BatchMPC did not solve), iteration counts, motion times and stop steps.  No solve fails (on a failed
    solve BatchMPC accepts the result and DeviceMPC keeps its warm start)."""
    out, _ = _against_batch_mpc(name, 4, 'cpu')
    for k, o in enumerate(out):
        assert np.array_equal(o['status'], o['ref_status']), (k, o['status'], o['ref_status'])
        assert np.all(o['status'] <= 0), k
        assert np.array_equal(o['iters'], o['ref_iters']), k
        assert np.array_equal(o['T'], o['ref_T']), k
        assert np.array_equal(o['X0'], o['ref_X0']), (k, np.abs(o['X0'] - o['ref_X0']).max())
        assert np.array_equal(o['P'], o['ref_P']), (k, np.abs(o['P'] - o['ref_P']).max())
    print('%s: %d updates, stop steps %s' % (name, len(out), [int((o['status'] == 0).sum()) for o in out]))


# ---------------------------------------------------------------------------------------------
# the reference's loops
# ---------------------------------------------------------------------------------------------
def _check_loop_golden(G, name, batch, device, prediction='ideal', plant=None):
    """The reference's free-T loop: the caller feeds the golden's goal and obstacle states (from its p)
    and, with 'integrate', its plant state at the start of the previous plan.  Statuses and the stop
    step are equal; x0 on the vehicle's columns and T, p and the motion times are returned as errors
    (the solutions cannot be replayed inside the C call, and the hyperplane variables are not unique,
    so the other columns of x0 are not compared)."""
    dt = float(G[name + '_dt'])
    pr = SCENES[name]()
    desc = b200.mpc_freeT_desc(pr, dt)
    mpc = _mpc(pr, batch, device, update_time=dt, trajectory_length=11, prediction=prediction)
    nd, ps, p0, L, o, ti = desc['n_dim'], desc['p_poseT'], desc['p_state0'], desc['L'], desc['spl_offset'], desc['t_index']
    cols = np.r_[o:o + nd * L, ti]
    n_steps = len(G[name + '_status'])
    st0 = np.repeat(G[name + '_p'][0][None, p0:p0 + nd], batch, 0)
    err = np.zeros(3)
    for k in range(n_steps + 1):
        p = np.repeat(G[name + '_p'][min(k, n_steps - 1)][None], batch, 0)
        if plant is not None:
            st0 = np.repeat(G[name + '_plant_state'][max(k - 1, 0)][None], batch, 0)
        _, _, status, _ = mpc.update(_t(st0, device), _t(p[:, ps:ps + nd], device), _t(_obstacles_from_p(desc, p), device))
        status = status.cpu().numpy()
        if k == n_steps:            # the golden's loop has ended: every instance has stopped
            assert np.all(status == b200.MPC_STOPPED), (name, status)
            break
        assert np.all(status == G[name + '_status'][k]), (name, k, status)
        X0, P = (a.cpu().numpy() for a in mpc.last_problem())
        T = mpc.motion_time().cpu().numpy()
        err = np.maximum(err, [np.abs(X0[:, cols] - G[name + '_x0'][k][None, cols]).max(),
                               np.abs(P - G[name + '_p'][k][None]).max(), np.abs(T - G[name + '_T'][k]).max()])
    return err


# T: within 1e-4 of the reference's.  x0 (vehicle columns and T) and p: the minimum-time objective
# fixes T but not the spline coefficients, so without replaying the reference's solutions the plans
# drift apart along the optimum's flat directions, and state0, the prediction from the plan, with
# them (measured: see the tests' docstrings)
GOLDEN_BOUND = (1e-2, 1e-2, 1e-4)


@pytest.mark.parametrize('name, batch', [('config_freeT', 1), ('config_freeT', 3), ('config_freeT_moving', 1),
                                         ('config_freeT_moving', 3)])
def test_follows_the_references_loop(emu, name, batch):
    """golden/freeT_loop_golden.npz: equal statuses and stop step; x0 on the vehicle's columns and T,
    p and the motion time within GOLDEN_BOUND of the reference's.  Measured on the emulation (batch 1
    and 3 alike): config_freeT x0 3.7e-3, p 6.2e-3, T 9.0e-5; config_freeT_moving x0 1.8e-9, p 2.3e-7,
    T 7.4e-5."""
    err = _check_loop_golden(np.load(LOOP_GOLDEN), name, batch, 'cpu')
    print('%s batch %d: x0 %.1e, p %.1e, T %.1e' % ((name, batch) + tuple(err)))
    assert np.all(err < GOLDEN_BOUND), err


def test_follows_the_references_closed_loop(emu):
    """golden/freeT_closed_loop_golden.npz config_freeT_moving with the 'integrate' prediction fed the
    reference's plant states: equal statuses and stop step; x0, p and T within GOLDEN_BOUND (measured:
    x0 3.4e-4, p 1.7e-4, T 8.4e-5)."""
    err = _check_loop_golden(np.load(CLOSED_GOLDEN), 'config_freeT_moving', 1, 'cpu', 'integrate', plant=True)
    print('closed: x0 %.1e, p %.1e, T %.1e' % tuple(err))
    assert np.all(err < GOLDEN_BOUND), err


# ---------------------------------------------------------------------------------------------
# outputs, stop and recover, failed solves, independence
# ---------------------------------------------------------------------------------------------
def test_trajectory_outputs_are_the_returned_plans(emu):
    """state_traj / input_traj row j is the plan's value and derivative / T at min(j st, T) / T, to
    1e-12 of the host evaluation of the solution, rows past the plan's T (which hold its final point)
    included."""
    from omg_tools_b200.basics.spline import BSplineBasis
    bat, mpc = _jittered('config_freeT', 2, trajectory_length=1000)
    desc = b200.mpc_freeT_desc(bat.problem, DT)
    st0, stT, obs = _t(bat.state, 'cpu'), _t(bat.poseT, 'cpu'), _t(_batch_obstacles(bat), 'cpu')
    Xn = []                        # BatchMPC's first solve returns the same plan on the same inputs
    solve = bat.solver.solve_batch_device

    def rec(X0, P, LB, UB, Xo, *a, **kw):
        r = solve(X0, P, LB, UB, Xo, *a, **kw)
        Xn.append(Xo.cpu().numpy().copy())
        return r
    bat.solver.solve_batch_device = rec
    bat.step()
    xs, us, status, _ = mpc.update(st0, stT, obs)
    assert np.all(status.numpy() == 0)
    X = Xn[0]
    T = X[:, desc['t_index']]
    assert np.array_equal(T, mpc.motion_time().numpy())
    basis = BSplineBasis(desc['knots'], desc['degree'])
    Bd, P1 = basis.derivative(1)
    L, o = desc['L'], desc['spl_offset']
    n_past = 0
    for b in range(2):
        tau = np.minimum(np.arange(1000) * 0.01, T[b]) / T[b]
        n_past += int((np.arange(1000) * 0.01 > T[b]).sum())
        R0, R1 = basis.eval_basis(tau), Bd.eval_basis(tau).dot(P1) / T[b]
        for c in range(desc['n_dim']):
            col = X[b, o + c * L:o + (c + 1) * L]
            assert np.abs(xs.numpy()[b, :, c] - R0.dot(col)).max() < 1e-12, (b, c)
            assert np.abs(us.numpy()[b, :, c] - R1.dot(col)).max() < 1e-12, (b, c)
    assert n_past > 0


def _starts():
    """Three instances of config_freeT; instance 1's goal is close to its start, so it stops first."""
    st0 = np.array([[-1.5, -1.5], [-1.4, -1.6], [-1.6, -1.4]])
    stT = np.array([[2., 2.], [-1.1, -1.6], [1.9, 2.1]])
    return st0, stT


def _run_updates(mpc, st0, stT, obs, n, device='cpu'):
    res = []
    for k in range(n):
        out = mpc.update(_t(st0, device), _t(stT, device), _t(obs, device))
        res.append([o.cpu().numpy().copy() for o in out] + [o.cpu().numpy().copy() for o in mpc.last_problem()] +
                   [mpc.motion_time().cpu().numpy().copy(), mpc.time.copy()])
    return res


def test_a_stopped_instance_is_not_solved_and_recovers(emu):
    """Batch of 3 whose instance 1 arrives first: once stopped it is not solved (status -1, 0 iterations)
    and its time, motion time, X0 and output rows stay as they were, while instances 0 and 2 equal
    batch-1 runs bit for bit.  recover() with a new goal cold-starts it and it runs again."""
    pr = sc.config_freeT()
    desc = b200.mpc_freeT_desc(pr, DT)
    st0, stT = _starts()
    obs = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], 3, 0))
    mpc = _mpc(pr, 3, 'cpu', trajectory_length=60)
    full = _run_updates(mpc, st0, stT, obs, 5)
    status = np.array([r[2] for r in full])
    stop = int(np.argmax(status[:, 1] == b200.MPC_STOPPED))
    assert 0 < stop < 4 and np.all(status[:stop] == 0) and np.all(status[stop:, 1] == b200.MPC_STOPPED), status
    assert np.all(status[:, [0, 2]] == 0)
    for k in range(stop, 5):
        xs, us, _, iters, X0, P, T, t = full[k]
        assert iters[1] == 0
        prev = full[stop - 1]
        for a, b in ((xs, prev[0]), (us, prev[1]), (T, prev[6]), (t, prev[7])):
            assert np.array_equal(a[1], b[1]), k
        assert np.array_equal(X0[1], prev[4][1]), k
    for b in (0, 2):
        one = _run_updates(_mpc(sc.config_freeT(), 1, 'cpu', trajectory_length=60), st0[b:b + 1], stT[b:b + 1],
                           obs[b:b + 1], 5)
        for k in range(5):
            assert all(np.array_equal(g[0], f[b]) for g, f in zip(one[k], full[k])), (b, k)
    stT2 = stT.copy()
    stT2[1] = [-1.0, -1.9]
    mpc.recover([False, True, False])
    xs, us, status, iters = mpc.update(_t(st0, 'cpu'), _t(stT2, 'cpu'), _t(obs, 'cpu'))
    assert status.numpy()[1] == 0 and iters.numpy()[1] > 0
    X0, P = (a.numpy() for a in mpc.last_problem())
    cold = desc['x_template'].copy()
    L, o = desc['L'], desc['spl_offset']
    for c in range(2):
        cold[o + c * L:o + (c + 1) * L] = np.linspace(st0[1, c], stT2[1, c], L)
    assert np.array_equal(X0[1], cold)
    assert np.array_equal(P[1, desc['p_input0']:desc['p_input0'] + 2], np.zeros(2))
    assert np.array_equal(P[1, desc['p_poseT']:desc['p_poseT'] + 2], stT2[1])


def test_a_failed_solve_keeps_its_instance(emu):
    """Batch of 2; from update 2 on with max_iter 40 (it keeps the failing solve cheap), and the circle
    put on instance 1's predicted position, where its solve fails.  Its time, motion time and output
    rows stay as they were, and the next update hands the solver the same warm start and parameters
    again: no second shift."""
    pr = sc.config_freeT()
    desc = b200.mpc_freeT_desc(pr, DT)
    st0, stT = _starts()
    st0, stT = st0[[0, 2]], stT[[0, 2]]
    obs0 = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], 2, 0))
    mpc = _mpc(pr, 2, 'cpu', trajectory_length=60)
    ok = _run_updates(mpc, st0, stT, obs0, 2)
    assert all(np.all(r[2] == 0) for r in ok)
    pr.problem.set_options({'max_iter': 40, 'feas_steps': 0})
    obs = obs0.copy()
    obs[1, 2, :2] = ok[-1][0][1, 50]          # (the plan's position at the next update)
    obs[1, 2, 2:6] = 0.
    fail = _run_updates(mpc, st0, stT, obs, 2)
    for r in fail:
        assert r[2][1] > 0 and r[2][0] == 0, r[2]
        for i in (0, 1, 6, 7):
            assert np.array_equal(r[i][1], ok[-1][i][1]), i
    assert np.array_equal(fail[1][4][1], fail[0][4][1]) and np.array_equal(fail[1][5][1], fail[0][5][1])
    assert not np.array_equal(fail[1][4][0], fail[0][4][0])


def _run_three(steps=3):
    bat, mpc = _jittered('config_freeT', 3, seed=5, trajectory_length=12)
    return _run_updates(mpc, bat.state, bat.poseT, _batch_obstacles(bat), steps), bat


def test_instances_are_independent_and_schedules_agree(emu, monkeypatch):
    """Instance b of a jittered batch of 3 equals a batch-1 run of that instance bit for bit, and the
    reversed and random thread schedules of the emulation give bit-identical results."""
    full, bat = _run_three()
    obs = _batch_obstacles(bat)
    for b in (1, 2):
        one = _run_updates(_mpc(sc.config_freeT(), 1, 'cpu', trajectory_length=12), bat.state[b:b + 1],
                           bat.poseT[b:b + 1], obs[b:b + 1], 3)
        for k in range(3):
            assert all(np.array_equal(g[0], f[b]) for g, f in zip(one[k], full[k])), (b, k)
    for sched in ('reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        other, _ = _run_three()
        assert all(np.array_equal(a, c) for ra, rc in zip(full, other) for a, c in zip(ra, rc)), sched


# ---------------------------------------------------------------------------------------------
# the listed solve
# ---------------------------------------------------------------------------------------------
def _solve_rows(lib, pr, X0, P, rows):
    """omg_solve_batch_rows on the listed rows (rows None: omg_solve_batch); unlisted outputs keep NaN / 77."""
    import torch
    B, n, m = X0.shape[0], pr.father.tables.n, pr.father.tables.m
    t = lambda a: torch.tensor(np.ascontiguousarray(a))
    x0, p = t(X0), t(P)
    lb, ub = t(pr.father.tables.lbg), t(pr.father.tables.ubg)
    x, lam, f = t(np.full((B, n), np.nan)), t(np.full((B, m), np.nan)), t(np.full(B, np.nan))
    st, it = t(np.full(B, 77, np.int32)), t(np.full(B, 77, np.int32))
    args = [pr.problem._handle, B, x0.data_ptr(), p.data_ptr(), lb.data_ptr(), ub.data_ptr(), 1, None,
            x.data_ptr(), lam.data_ptr(), f.data_ptr(), st.data_ptr(), it.data_ptr()]
    if rows is None:
        assert lib.omg_solve_batch(*args, None) == 0, lib.omg_last_error()
    else:
        r, nr = t(np.r_[rows, 0].astype(np.int32)), t(np.array([len(rows)], np.int32))
        assert lib.omg_solve_batch_rows(*args, r.data_ptr(), nr.data_ptr(), None) == 0, lib.omg_last_error()
    return [a.numpy() for a in (x, lam, f, st, it)]


@pytest.mark.parametrize('kernel', ['sparse', 'envelope'])
def test_listed_solve_equals_the_full_solve_on_its_rows(emu, monkeypatch, kernel):
    """The solver kernel with a row list equals the full solve on the listed rows bit for bit and leaves
    the other rows' outputs untouched, on the sparse and the envelope kernel."""
    if kernel == 'envelope':
        monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    pr = sc.config1()
    assert ('envelope' in pr.problem.lib.omg_structure_info(pr.problem._handle).decode()) == (kernel == 'envelope')
    X0, P = sc.instance_data(pr, 5, jitter=0.2, seed=3)
    full = _solve_rows(emu, pr, X0, P, None)
    rows = [0, 2, 3]
    part = _solve_rows(emu, pr, X0, P, rows)
    for a, b in zip(full, part):
        assert np.array_equal(a[rows], b[rows])
    assert np.all(np.isnan(part[0][[1, 4]])) and np.all(part[3][[1, 4]] == 77) and np.all(part[4][[1, 4]] == 77)
    none = _solve_rows(emu, pr, X0, P, [])
    assert np.all(np.isnan(none[0])) and np.all(none[3] == 77)


# ---------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------
def _create(lib, pr, desc, B=2, tl=5, mode=0):
    D, keep = b200.pack_mpc_freeT_desc(desc)
    h = lib.omg_mpc_create_freet(pr.problem._handle, C.byref(D), B, tl, mode)
    if h:
        lib.omg_mpc_destroy(h)
        return None
    return lib.omg_last_error().decode()


def test_create_rejects(emu):
    pr = sc.config_freeT()
    desc = b200.mpc_freeT_desc(pr, DT)
    n, T0 = desc['n'], desc['x_template'][desc['t_index']]
    assert T0 == 10. and _create(emu, pr, desc) is None
    f = 'omg_mpc_create_freet: '
    assert f + 'the descriptor is for n = 99' in _create(emu, pr, dict(desc, n=99))
    assert 'n_par' in _create(emu, pr, dict(desc, n_par=desc['n_par'] + 1))
    assert 'B must be >= 1' in _create(emu, pr, desc, B=0)
    assert 'unknown prediction' in _create(emu, pr, desc, mode=2)
    assert 'not a multiple of sample_time' in _create(emu, pr, dict(desc, update_time=0.505))
    assert 'update_time and sample_time must be > 0' in _create(emu, pr, dict(desc, sample_time=0.))
    assert 'vehicle splines' in _create(emu, pr, dict(desc, spl_offset=n - 5))
    assert 'state0 at' in _create(emu, pr, dict(desc, p_state0=desc['n_par'] - 1))
    assert 'obstacle 0 x/v/a' in _create(emu, pr, dict(desc, obs_off=np.r_[desc['n_par'], desc['obs_off'][1:]].astype(np.int32)))
    assert 'knots not non-decreasing' in _create(emu, pr, dict(desc, knots=desc['knots'][::-1].copy()))
    assert 't_index -1 outside [0, %d)' % n in _create(emu, pr, dict(desc, t_index=-1))
    assert 't_index %d outside' % n in _create(emu, pr, dict(desc, t_index=n))
    assert 'block 0: columns outside x' in _create(emu, pr, dict(desc, blk_off=np.r_[n - 3, desc['blk_off'][1:]].astype(np.int32)))
    assert 'block 0: degree 9' in _create(emu, pr, dict(desc, blk_degree=np.r_[9, desc['blk_degree'][1:]].astype(np.int32)))
    assert 'basis length 49' in _create(emu, pr, dict(desc, blk_len=np.r_[49, desc['blk_len'][1:]].astype(np.int32)))
    bad = desc['blk_knots'].copy()
    bad[3], bad[4] = bad[4], bad[3] - 0.01
    assert 'block 0: knots not non-decreasing' in _create(emu, pr, dict(desc, blk_knots=bad))
    assert 'stop_tol must be >= 0' in _create(emu, pr, dict(desc, stop_tol=-1e-3))
    assert 'trajectory_length 0 outside 1 .. (template T) / sample_time = 1000' in _create(emu, pr, desc, tl=0)
    assert _create(emu, pr, desc, tl=1000) is None
    assert 'trajectory_length 1001' in _create(emu, pr, desc, tl=1001)
    D, keep = b200.pack_mpc_freeT_desc(desc)
    assert not emu.omg_mpc_create_freet(None, C.byref(D), 2, 5, 0)
    assert 'null argument' in emu.omg_last_error().decode()
    assert emu.omg_mpc_motion_time(None, None, None) == -1
    assert emu.omg_solve_batch_rows(pr.problem._handle, 1, None, None, None, None, 1, *([None] * 9)) == -1
    assert 'null row list' in emu.omg_last_error().decode()


def test_save_mpc_freeT_rejects_what_it_does_not_run(tmp_path):
    from omg_tools_b200 import Holonomic, Environment, Obstacle, Circle, Point2point, Rectangle, Square
    path = str(tmp_path / 'x.omgmpc')
    fleet = [Holonomic(), Holonomic()]
    for i, v in enumerate(fleet):
        v.set_initial_conditions([-1.5 + i, -1.5])
        v.set_terminal_conditions([2. - i, 2.])
    with pytest.raises(NotImplementedError, match='one vehicle, this problem has 2'):
        b200.save_mpc_freeT(sc._p2p(fleet, Environment(room={'shape': Square(5.)}), {}, False, freeT=True), path)
    with pytest.raises(NotImplementedError, match='not Dubins'):
        b200.save_mpc_freeT(sc.config_dubins_freeT(build_solver=False), path)
    with pytest.raises(NotImplementedError, match='fixed horizon'):
        b200.save_mpc_freeT(sc.config1(build_solver=False), path)
    veh = Holonomic()
    veh.set_initial_conditions([-1.5, -1.5])
    veh.set_terminal_conditions([2., 2.])
    env = Environment(room={'shape': Rectangle(width=5., height=5.)})
    env.add_obstacle(Obstacle({'position': [0., 0.]}, shape=Circle(0.4), options={'spline_traj': True}))
    pr = Point2point(veh, env, freeT=True)
    with pytest.raises(NotImplementedError, match='spline_traj'):
        b200.save_mpc_freeT(pr, path)


# ---------------------------------------------------------------------------------------------
# MPC file and native caller
# ---------------------------------------------------------------------------------------------
def _read_freeT(lib, path):
    D = lib.omg_mpc_freet_read(path.encode())
    assert D, lib.omg_last_error().decode()
    d = D.contents
    out = {}
    for name, kind in b200.MPC_FREET_FIELDS:
        v = getattr(d, name)
        if kind in 'ID':
            lens = np.ctypeslib.as_array(d.blk_len, (d.n_blocks,)) if d.n_blocks else np.zeros(0, int)
            degs = np.ctypeslib.as_array(d.blk_degree, (d.n_blocks,)) if d.n_blocks else np.zeros(0, int)
            size = {'knots': d.L + d.degree + 1, 'obs_kind': d.n_obs, 'obs_off': 4 * d.n_obs, 'x_template': d.n,
                    'p_template': d.n_par, 'blk_knots': int((lens + degs + 1).sum())}.get(name, d.n_blocks)
            v = np.ctypeslib.as_array(v, (size,)).copy() if size else np.zeros(0)
        out[name] = v
    lib.omg_mpc_freet_release(D)
    return out


@pytest.mark.parametrize('name', ['config_freeT_moving', 'holonomic3d_freeT'])
def test_mpc_file_round_trip(emu, tmp_path, name):
    """save_mpc_freeT / omg_mpc_freet_read give back the descriptor, and each reader refuses the other
    kind's file with a message that names the other reader."""
    pr = SCENES[name](build_solver=False)
    path = str(tmp_path / 'p.omgmpc')
    b200.save_mpc_freeT(pr, path, update_time=0.4, sample_time=0.02)
    desc, back = b200.mpc_freeT_desc(pr, 0.4, 0.02), _read_freeT(emu, path)
    for key, _ in b200.MPC_FREET_FIELDS:
        assert np.array_equal(np.asarray(back[key]), np.asarray(desc[key])), key
    assert not emu.omg_mpc_read(path.encode())
    assert 'omg_mpc_freet_read' in emu.omg_last_error().decode()
    fixed = str(tmp_path / 'f.omgmpc')
    b200.save_mpc(sc.config1(build_solver=False), fixed)
    assert not emu.omg_mpc_freet_read(fixed.encode())
    assert 'omg_mpc_read' in emu.omg_last_error().decode()
    assert not emu.omg_mpc_freet_read(str(tmp_path / 'missing').encode())


def _native(tmp_path, lib_args, pr, B, N, tl, st0, stT, obs, prediction='ideal'):
    exe = str(tmp_path / 'native_mpc')
    subprocess.check_call(['g++', '-O2', '-I', os.path.join(ROOT, 'include'),
                           os.path.join(ROOT, 'examples', 'native', 'native_mpc.cpp'), '-o', exe] + lib_args)
    b200.save_tables(pr.father.tables, str(tmp_path / 'p.omgtbl'))
    b200.save_mpc_freeT(pr, str(tmp_path / 'p.omgmpc'), update_time=DT)
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
    """examples/native/native_mpc.cpp on a free-T table file and MPC file, linked to the emulation
    library, reproduces DeviceMPC bit for bit: batch 2 over 3 updates, both predictions."""
    bat, _ = _jittered('config_freeT', 2, seed=2)
    obs = _batch_obstacles(bat)
    for prediction in ('ideal', 'integrate'):
        traj, stat = _native(tmp_path, [emu_support.EMU_LIB, '-Wl,-rpath,' + os.path.dirname(emu_support.EMU_LIB)],
                             sc.config_freeT(build_solver=False), 2, 3, 15, bat.state, bat.poseT, obs, prediction)
        ref, ref_stat = _python_loop(sc.config_freeT(), 2, 3, 15, bat.state, bat.poseT, obs, 'cpu', prediction)
        assert np.array_equal(stat, ref_stat) and np.all(stat[:, :, 0] == 0), prediction
        assert np.array_equal(traj, ref), prediction


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_follows_the_references_loops():
    """The golden checks at batch 1 on the device, with the CPU tests' bound."""
    for name in ('config_freeT', 'config_freeT_moving'):
        err = _check_loop_golden(np.load(LOOP_GOLDEN), name, 1, 'cuda')
        print('%s: x0 %.1e, p %.1e, T %.1e' % ((name,) + tuple(err)))
        assert np.all(err < GOLDEN_BOUND), (name, err)
    err = _check_loop_golden(np.load(CLOSED_GOLDEN), 'config_freeT_moving', 1, 'cuda', 'integrate', plant=True)
    print('closed: x0 %.1e, p %.1e, T %.1e' % tuple(err))
    assert np.all(err < GOLDEN_BOUND), err


@pytest.mark.gpu
def test_gpu_batch_1024_matches_batch_1_and_batch_mpc():
    """Jittered config_freeT, batch 1024, 18 updates (BatchMPC's whole run): a spread of instances equals
    batch-1 runs bit for bit.  Statuses and iteration counts equal BatchMPC's but for a few
    instance-updates: the ideal prediction is the same spline value rounded differently on the device
    and in BatchMPC's evaluation, so a borderline solve (the last solves of a run, T within two updates
    of its end) may take another iteration count or fail in one run and not in the other.  From an
    instance's first failed solve on the two runs differ for it by design (BatchMPC accepts the result,
    DeviceMPC keeps its warm start), and it is left out of the status comparison."""
    import torch
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(sc.config_freeT(), batch=1024, update_time=DT, jitter=0.2, seed=7, device=torch.device('cuda'))
    mpc = _mpc(sc.config_freeT(), 1024, 'cuda', trajectory_length=11)
    idx = np.array([0, 1, 517, 1023])
    st0, stT = _t(bat.state, 'cuda'), _t(bat.poseT, 'cuda')
    ones = [_mpc(sc.config_freeT(), 1, 'cuda', trajectory_length=11) for _ in idx]
    n_sdiff = n_idiff = n_all = 0
    failed = np.zeros(1024, bool)
    for k in range(40):
        if not bat.active.any():
            break
        obs = _batch_obstacles(bat)
        bat.step()
        xs, us, status, iters = mpc.update(st0, stT, _t(obs, 'cuda'))
        s, r = status.cpu().numpy(), bat.history['status'][-1]
        cmp = ~failed & (r != -1)
        n_sdiff += int((s != r)[~failed].sum())
        n_idiff += int((iters.cpu().numpy() != bat.history['iters'][-1])[cmp].sum())
        n_all += int(cmp.sum())
        failed |= (s > 0) | (r > 0)
        full = [o.cpu().numpy() for o in (xs, us, status, iters, mpc.motion_time())] + \
               [o.cpu().numpy() for o in mpc.last_problem()]
        for b, one in zip(idx, ones):
            out = one.update(st0[b:b + 1].contiguous(), stT[b:b + 1].contiguous(), _t(obs[b:b + 1], 'cuda'))
            got = [o.cpu().numpy()[0] for o in out + (one.motion_time(),)] + \
                  [o.cpu().numpy()[0] for o in one.last_problem()]
            assert all(np.array_equal(g, f[b]) for g, f in zip(got, full)), (b, k)
    print('of %d instance-updates, statuses differ from BatchMPC in %d, iteration counts in %d; %d instances '
          'had a failed solve' % (n_all, n_sdiff, n_idiff, int(failed.sum())))
    assert n_sdiff <= 0.002 * n_all and n_idiff <= 0.01 * n_all


@pytest.mark.gpu
def test_gpu_updates_replay_from_a_cuda_graph():
    """Updates 2 to 20 of a jittered batch of 64, captured with torch.cuda.graph on a side stream and
    replayed, give bit-identical outputs, times and motion times to the eager run, through the updates
    at which the instances stop."""
    import torch
    bat, eager = _jittered('config_freeT', 64, seed=3, device='cuda', trajectory_length=20)
    graphed = _mpc(sc.config_freeT(), 64, 'cuda', trajectory_length=20)
    st0, stT, obs = _t(bat.state, 'cuda'), _t(bat.poseT, 'cuda'), _t(_batch_obstacles(bat), 'cuda')
    ref = []
    for k in range(20):
        ref.append([o.clone() for o in eager.update(st0, stT, obs)] + [eager.motion_time()])
    graphed.update(st0, stT, obs)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    outs = []
    side = torch.cuda.Stream()
    with torch.cuda.graph(g, stream=side):
        for k in range(19):
            outs.append([o.clone() for o in graphed.update(st0, stT, obs)] + [graphed.motion_time(stream=side)])
    g.replay()
    torch.cuda.synchronize()
    st = torch.stack([r[2] for r in ref]).cpu().numpy()
    assert np.all(st[1] == 0) and np.mean(st[-1] == b200.MPC_STOPPED) > 0.9, st      # (the window holds the stops)
    for k in range(19):
        for a, b in zip(outs[k], ref[k + 1]):
            assert torch.equal(a, b), k
    assert np.array_equal(graphed.time, eager.time)


@pytest.mark.gpu
def test_gpu_native_mpc_caller(tmp_path):
    """native_mpc.cpp on a free-T MPC file against libomgb200.so is bit-identical to the Python binding."""
    lib_dir = os.path.join(ROOT, 'omg_tools_b200', 'csrc')
    bat, _ = _jittered('config_freeT', 3, seed=4, device='cuda')
    obs = _batch_obstacles(bat)
    traj, stat = _native(tmp_path, ['-L', lib_dir, '-lomgb200', '-Wl,-rpath,' + lib_dir],
                         sc.config_freeT(build_solver=False), 3, 4, 15, bat.state, bat.poseT, obs)
    ref, ref_stat = _python_loop(sc.config_freeT(), 3, 4, 15, bat.state, bat.poseT, obs, 'cuda')
    assert np.array_equal(stat, ref_stat)
    assert np.array_equal(traj, ref)
