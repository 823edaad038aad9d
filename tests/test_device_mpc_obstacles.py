"""Obstacle shapes and avoid flags of the device MPC update (include/omg_b200.h,
omg_mpc_attach_obstacles / omg_mpc_set_obstacles; DeviceMPC.set_obstacles): the checkpoints, radii
and avoid flag of the reference's obstacle_t, per instance.

The obstacle descriptor is checked against the rows and parameters of the reference's own exporter
(golden/update_bounds_golden.npz, tests/golden/make_update_bounds_golden.py).  The tests without a
mark run the kernel source on the CPU (tools/cpu_emu); the ones marked gpu run on the device."""
import ctypes as C
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
from test_device_mpc import _t, _mpc, _obstacles_from_p  # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'update_bounds_golden.npz')
H3D = lambda **kw: sc.config_holonomic3d(start=(-1.7, -1.7, -1.7), goal=(1.7, 1.7, -1.7), **kw)  # noqa: E731
SCENES = {'config1': sc.config1, 'config2': sc.config2, 'config5': sc.config5, 'config_holonomic3d': H3D,
          'config_freeT': sc.config_freeT}


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


@functools.lru_cache(maxsize=None)
def _plain(name):
    """Scenario `name` without a solver, built once: what descriptors and templates are read from."""
    return SCENES[name](build_solver=False)


def _i(a, device):
    import torch
    return torch.tensor(np.ascontiguousarray(a, dtype=np.int32), device=device)


def _desc(pr):
    from omg_tools_b200.problems.point2point import FreeTPoint2point
    return b200.mpc_freeT_desc(pr) if isinstance(pr, FreeTPoint2point) else b200.mpc_desc(pr)


def _template_shapes(pr, B):
    """[B, record] of the problem's own shapes, in the layout set_obstacles takes."""
    od, p = b200.mpc_obstacles_desc(pr), _desc(pr)['p_template']
    rec = np.concatenate([np.r_[p[od['chk_off'][k]:od['chk_off'][k] + od['chk_len'][k]],
                                p[od['rad_off'][k]:od['rad_off'][k] + od['rad_len'][k]]] for k in range(od['n_obs'])])
    return np.repeat(rec[None], B, 0)


def _bounds(pr, avoid):
    """The tables' bounds per instance with the rows of the obstacles not avoided set to -inf / +inf."""
    tb, od = pr.father.tables, b200.mpc_obstacles_desc(pr)
    LB, UB = np.repeat(tb.lbg[None], len(avoid), 0), np.repeat(tb.ubg[None], len(avoid), 0)
    for b, row in enumerate(avoid):
        for k, on in enumerate(row):
            if not on:
                r = slice(od['row_off'][k], od['row_off'][k] + od['row_len'][k])
                LB[b, r], UB[b, r] = -np.inf, np.inf
    return LB, UB


def _starts(name, B, seed):
    """Jittered starts and goals of scenario `name` around its own."""
    rng = np.random.default_rng(seed)
    d = _desc(_plain(name))
    nd, p = d['n_dim'], d['p_template']
    s0, sT = p[d['p_state0']:d['p_state0'] + nd], p[d['p_poseT']:d['p_poseT'] + nd]
    j = 0.05 if name in ('config5', 'config_freeT') else 0.2
    return s0 + rng.uniform(-j, j, (B, len(s0))), sT + rng.uniform(-j, j, (B, len(sT)))


def _outputs(mpc, out):
    return [o.cpu().numpy().copy() for o in out] + [o.cpu().numpy().copy() for o in mpc.last_problem()] + \
        [mpc.motion_time().cpu().numpy().copy(), mpc.time.copy()]


# ---------------------------------------------------------------------------------------------
# the descriptor against the reference's exporter
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['config1', 'config2', 'config5', 'config_holonomic3d'])
def test_descriptor_is_the_references_update_bounds(name):
    """The rows of each obstacle are the rows the reference's updateBounds frees, with the same default
    bounds in the tables, and its checkpoints and radii are the p entries its fillParameterDict writes."""
    G = np.load(GOLDEN)
    pr = getattr(sc, name)(build_solver=False)
    od, tb = b200.mpc_obstacles_desc(pr), pr.father.tables
    assert od['n_obs'] == int(G[name + '_n_obs'])
    for k in range(od['n_obs']):
        rows = np.arange(od['row_off'][k], od['row_off'][k] + od['row_len'][k])
        assert np.array_equal(rows, G['%s_rows_%d' % (name, k)]), k
        assert np.array_equal(tb.lbg[rows], G['%s_lbg_%d' % (name, k)]), k
        assert np.array_equal(tb.ubg[rows], G['%s_ubg_%d' % (name, k)]), k
        assert {'checkpoints', 'rad'} <= set(G['%s_params_%d' % (name, k)].tolist())
        poff = G['%s_poff_%d' % (name, k)]
        assert [od['chk_off'][k], od['chk_len'][k]] == poff[0].tolist(), k
        assert [od['rad_off'][k], od['rad_len'][k]] == poff[1].tolist(), k


# ---------------------------------------------------------------------------------------------
# semantics on the CPU emulation
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['config1', 'config5', 'config_holonomic3d', 'config_freeT'])
def test_attached_with_the_template_is_a_no_op(emu, name):
    """A handle with obstacles attached, every flag set and the template's shapes (through the set
    kernel) gives the statuses, iterations, outputs, solver rows and times of an unattached handle,
    bit for bit."""
    B, n = 2, 3
    s0, sT = _starts(name, B, 11)
    plain, att = (_mpc(SCENES[name](), B, 'cpu', trajectory_length=8) for _ in range(2))
    desc = _desc(_plain(name))
    obs = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], B, 0))
    att.set_obstacles(_t(_template_shapes(_plain(name), B), 'cpu'),
                      _i(np.ones((B, att.n_obs)), 'cpu'))
    for k in range(n):
        a = _outputs(plain, plain.update(_t(s0, 'cpu'), _t(sT, 'cpu'), _t(obs, 'cpu')))
        b = _outputs(att, att.update(_t(s0, 'cpu'), _t(sT, 'cpu'), _t(obs, 'cpu')))
        assert np.all(a[2] == 0), (k, a[2])
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), k


def test_avoid_flags_free_the_obstacles_rows(emu):
    """Config 2, a jittered batch of 4 with random avoid masks that change between updates: each update's
    x, status and iterations equal omg_solve_batch on last_problem()'s x0 and p with per-instance bounds
    built here (the tables' bounds, the golden's rows of the obstacles not avoided set to -inf / +inf)."""
    B = 4
    pr = sc.config2()
    G = np.load(GOLDEN)
    rows = [G['config2_rows_%d' % k] for k in range(3)]
    s0, sT = _starts('config2', B, 3)
    desc = _desc(pr)
    obs = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], B, 0))
    mpc = _mpc(pr, B, 'cpu', trajectory_length=5)
    rng = np.random.default_rng(5)
    for k in range(4):
        avoid = (rng.uniform(size=(B, 3)) < 0.5).astype(np.int32)
        avoid[0] = 1
        avoid[1] = 0
        mpc.set_obstacles(avoid=_i(avoid, 'cpu'))
        _, _, status, iters = mpc.update(_t(s0, 'cpu'), _t(sT, 'cpu'), _t(obs, 'cpu'))
        X0, P = (a.numpy().copy() for a in mpc.last_problem())
        LB, UB = _bounds(pr, avoid)
        for b in range(B):                  # (the bounds built from the reference's rows)
            for j in range(3):
                if not avoid[b, j]:
                    assert np.all(np.isinf(LB[b, rows[j]])) and np.all(np.isinf(UB[b, rows[j]]))
        ref = pr.problem.solve_batch(X0, P, LB, UB, _retry=False)
        assert np.array_equal(status.numpy(), ref['status']) and np.array_equal(iters.numpy(), ref['iters']), k
        # an accepted solution is the next update's warm start (no knot is crossed before t = 1)
        assert k == 0 or np.array_equal(X0[prev_ok], prev_x[prev_ok]), k
        prev_x, prev_ok = ref['x'], ref['status'] == 0
        assert prev_ok[0], k                # (the instance that avoids every obstacle)
    # the flags reach the solve: instance 1 ignores every obstacle, instance 0 avoids every one
    assert not np.array_equal(ref['x'][0], ref['x'][1])


def _min_distance(xs, c):
    return np.sqrt(((xs - np.asarray(c)) ** 2).sum(-1)).min()


def test_avoid_off_goes_through_the_obstacle(emu):
    """Config 1 with its obstacle parked on the straight path: the plan of the instance that avoids it
    keeps the obstacle's radius and the vehicle's clear of its centre; the plan of the instance that does
    not passes through the circle."""
    B = 2
    pr = sc.config1()
    desc = _desc(pr)
    mpc = _mpc(pr, B, 'cpu', trajectory_length=1000)
    obs = np.zeros((B, 1, 7))
    obs[:, 0, :2] = [0.25, 0.25]
    mpc.set_obstacles(avoid=_i([[1], [0]], 'cpu'))
    s0, sT = np.array([[-1.5, -1.5]] * B), np.array([[2., 2.]] * B)
    xs, _, status, _ = mpc.update(_t(s0, 'cpu'), _t(sT, 'cpu'), _t(obs, 'cpu'))
    assert np.all(status.numpy() == 0)
    xs = xs.numpy()
    P = mpc.last_problem()[1].numpy()
    od = b200.mpc_obstacles_desc(pr)
    r_obs = P[0, od['rad_off'][0]]
    r_veh = 0.1                              # Holonomic's Circle(0.1)
    assert r_obs == 0.5 and np.array_equal(P[0, desc['obs_off'][0]:desc['obs_off'][0] + 2], [0.25, 0.25])
    d_avoid, d_free = _min_distance(xs[0], [0.25, 0.25]), _min_distance(xs[1], [0.25, 0.25])
    print('closest approach: avoided %.4f, not avoided %.4f' % (d_avoid, d_free))
    assert d_avoid >= r_obs + r_veh - 1e-6
    assert d_free < r_obs


def _scene(name, shape):
    """Config 2 with Circle(r) obstacles or config 5 with its beams resized, built as the scenario is."""
    from omg_tools_b200 import Holonomic, Environment, Obstacle, Point2point
    from omg_tools_b200.basics.shape import Circle, Beam, Square
    veh = Holonomic()
    if name == 'config2':
        veh.set_options({'safety_distance': 0.1})
        veh.set_initial_conditions([-1.5, -1.5])
        veh.set_terminal_conditions([2., 2.])
        env = Environment(room={'shape': Square(5.)})
        for pos in sc.CONFIG2_OBSTACLES:
            env.add_obstacle(Obstacle({'position': list(pos)}, shape=Circle(shape)))
        opts = {}
    else:
        veh.set_initial_conditions([0., -2.0])
        veh.set_terminal_conditions([0., 2.0])
        env = Environment(room={'shape': Square(5.)})
        w1, w2 = shape
        env.add_obstacle(Obstacle({'position': [-2., 0.]}, shape=Beam(width=w1, height=0.2)))
        env.add_obstacle(Obstacle({'position': [2., 0.]}, shape=Beam(width=w1, height=0.2)))
        omega = 1.5 * (2 * np.pi / 10.)
        env.add_obstacle(Obstacle({'position': [0., 0.], 'velocity': [0., 0.], 'angular_velocity': omega},
                                  shape=Beam(width=w2, height=0.2), simulation={}, options={'horizon_time': 10.}))
        env.add_obstacle(Obstacle({'position': [0., 0.], 'velocity': [0., 0.], 'orientation': 0.5 * np.pi,
                                   'angular_velocity': omega},
                                  shape=Beam(width=w2, height=0.2), simulation={}, options={'horizon_time': 10.}))
        opts = {'horizon_time': 10.}
    return sc._p2p(veh, env, opts, True)


@pytest.mark.parametrize('name, shapes', [('config2', (0.4, 0.3, 0.5)), ('config5', ((2.2, 1.4), (2.0, 1.2)))])
def test_per_instance_shapes_equal_problems_with_those_shapes(emu, name, shapes):
    """Instance b of an attached batch, given through set_obstacles the shapes of a scenario built with
    other radii (config 2's circles) or other beams (config 5), equals bit for bit a batch-1 unattached
    handle on that scenario: the two problems differ in p only."""
    B, n = len(shapes), 3
    base = sc.config2() if name == 'config2' else sc.config5()
    s0, sT = _starts(name, B, 7)
    scenes = [_scene(name, s) for s in shapes]
    recs = np.concatenate([_template_shapes(pr, 1) for pr in scenes])
    for pr in scenes:
        tb, tb0 = pr.father.tables, base.father.tables
        assert (tb.n, tb.m, tb.n_par) == (tb0.n, tb0.m, tb0.n_par)
    mpc = _mpc(base, B, 'cpu', trajectory_length=6)
    mpc.set_obstacles(_t(recs, 'cpu'))
    obs = _obstacles_from_p(_desc(base), np.repeat(_desc(base)['p_template'][None], B, 0))
    ones = [_mpc(pr, 1, 'cpu', trajectory_length=6) for pr in scenes]
    for k in range(n):
        full = _outputs(mpc, mpc.update(_t(s0, 'cpu'), _t(sT, 'cpu'), _t(obs, 'cpu')))
        assert np.all(full[2] == 0), full[2]
        for b, one in enumerate(ones):
            got = _outputs(one, one.update(_t(s0[b:b + 1], 'cpu'), _t(sT[b:b + 1], 'cpu'), _t(obs[b:b + 1], 'cpu')))
            assert all(np.array_equal(g[0], f[b]) for g, f in zip(got, full)), (b, k)
    assert not np.array_equal(full[0][0], full[0][1])


def test_free_T_takes_shapes_and_flags_and_leaves_stopped_instances(emu):
    """Free motion time, batch of 3 whose instance 1 stops first (its goal is close to its start).  Shapes
    and flags set after every update reach the solve: x, status and iterations equal omg_solve_batch on
    the rows that were solved, with bounds built here.  The stopped instance stays stopped: status -1, 0
    iterations, its warm start and parameter rows as they were."""
    pr = sc.config_freeT()
    desc = b200.mpc_freeT_desc(pr, 0.5)
    st0 = np.array([[-1.5, -1.5], [-1.4, -1.6], [-1.6, -1.4]])
    stT = np.array([[2., 2.], [-1.1, -1.6], [1.9, 2.1]])
    obs = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], 3, 0))
    mpc = _mpc(pr, 3, 'cpu', trajectory_length=20, update_time=0.5)
    lay, n_shape = mpc.shape_layout
    od = b200.mpc_obstacles_desc(pr)
    assert n_shape == len(_template_shapes(pr, 1)[0])
    rng = np.random.default_rng(2)
    stopped_at, prev = None, None
    for k in range(5):
        shapes = _template_shapes(pr, 3)
        shapes[:, lay[2][1]] = rng.uniform(0.3, 0.45, (3, 1))   # the circle's radius
        avoid = np.ones((3, 3), np.int32)
        avoid[2, 0] = k % 2                                       # a wall of instance 2, every other update
        mpc.set_obstacles(_t(shapes, 'cpu'), _i(avoid, 'cpu'))
        _, _, status, iters = mpc.update(_t(st0, 'cpu'), _t(stT, 'cpu'), _t(obs, 'cpu'))
        status, iters = status.numpy().copy(), iters.numpy().copy()
        X0, P = (a.numpy().copy() for a in mpc.last_problem())
        live = np.nonzero(status != b200.MPC_STOPPED)[0]
        assert np.array_equal(P[live, od['rad_off'][2]], shapes[live, lay[2][1]][:, 0])
        LB, UB = _bounds(pr, avoid)
        ref = pr.problem.solve_batch(X0[live], P[live], LB[live], UB[live], _retry=False)
        assert np.array_equal(status[live], ref['status']) and np.array_equal(iters[live], ref['iters']), k
        if status[1] == b200.MPC_STOPPED:
            if stopped_at is None:
                stopped_at = k
            assert iters[1] == 0
            assert np.array_equal(X0[1], prev[0][1]) and np.array_equal(P[1], prev[1][1]), k
        prev = (X0, P)
    assert stopped_at is not None and stopped_at < 4


# ---------------------------------------------------------------------------------------------
# rejections and the obstacle file
# ---------------------------------------------------------------------------------------------
def _attach(lib, mpc, od):
    D, keep = b200.pack_mpc_obstacles_desc(od)
    if lib.omg_mpc_attach_obstacles(mpc._handle, C.byref(D)) == 0:
        return None
    return lib.omg_last_error().decode()


def test_attach_and_set_reject(emu):
    pr = sc.config2()
    od = b200.mpc_obstacles_desc(pr)
    mpc = _mpc(pr, 2, 'cpu', trajectory_length=5)
    i32 = lambda *v: np.array(v, np.int32)  # noqa: E731
    assert emu.omg_mpc_set_obstacles(mpc._handle, None, None, None) == -1
    assert 'no obstacles attached' in emu.omg_last_error().decode()
    assert emu.omg_mpc_set_obstacles_host(mpc._handle, None, None) == -1
    assert 'no obstacles attached' in emu.omg_last_error().decode()
    with pytest.raises(RuntimeError, match='no obstacles attached'):
        mpc._check(emu.omg_mpc_set_obstacles(mpc._handle, None, None, None))
    D, keep = b200.pack_mpc_obstacles_desc(od)
    assert emu.omg_mpc_attach_obstacles(None, C.byref(D)) == -1 and 'null argument' in emu.omg_last_error().decode()
    assert emu.omg_mpc_attach_obstacles(mpc._handle, None) == -1 and 'null argument' in emu.omg_last_error().decode()
    assert 'the descriptor has 2 obstacles, the handle 3' in _attach(
        emu, mpc, {k: (v[:2] if k != 'n_obs' else 2) for k, v in od.items()})
    assert 'obstacle 1 checkpoints' in _attach(emu, mpc, dict(od, chk_off=i32(12, 34, 30)))
    assert 'obstacle 0 radii' in _attach(emu, mpc, dict(od, rad_off=i32(-1, 23, 32)))
    assert 'checkpoint coordinates and 2 radii' in _attach(emu, mpc, dict(od, rad_len=i32(2, 1, 1)))
    assert 'checkpoint coordinates and 0 radii' in _attach(emu, mpc, dict(od, rad_len=i32(0, 1, 1),
                                                                          chk_len=i32(0, 2, 2)))
    assert 'obstacle 2 rows' in _attach(emu, mpc, dict(od, row_len=i32(31, 31, 200)))
    assert 'overlap another obstacle' in _attach(emu, mpc, dict(od, row_off=i32(345, 370, 407)))
    eq = int(np.nonzero(pr.father.tables.lbg == pr.father.tables.ubg)[0][0])
    assert 'row %d is an equality' % eq in _attach(emu, mpc, dict(od, row_off=i32(eq, 376, 407)))
    assert _attach(emu, mpc, od) is None
    assert 'already has obstacles attached' in _attach(emu, mpc, od)
    # the binding's own checks
    with pytest.raises(ValueError, match='shapes must be'):
        mpc.set_obstacles(_t(np.zeros((2, 8)), 'cpu'))
    with pytest.raises(ValueError, match='avoid must be'):
        mpc.set_obstacles(avoid=_i(np.zeros((2, 2)), 'cpu'))
    with pytest.raises(ValueError, match='int32'):
        mpc.set_obstacles(avoid=_t(np.zeros((2, 3)), 'cpu'))


def test_save_mpc_obstacles_rejects_what_save_mpc_rejects(tmp_path):
    from omg_tools_b200 import Holonomic, Environment, Obstacle, Circle, Point2point, Rectangle
    path = str(tmp_path / 'x.omgobs')
    with pytest.raises(NotImplementedError, match='one vehicle, this problem has 2'):
        b200.save_mpc_obstacles(sc.config_interveh_offset(build_solver=False), path)
    with pytest.raises(NotImplementedError, match='not Dubins'):
        b200.save_mpc_obstacles(sc.config_dubins(build_solver=False), path)
    veh = Holonomic()
    veh.set_initial_conditions([-1.5, -1.5])
    veh.set_terminal_conditions([2., 2.])
    env = Environment(room={'shape': Rectangle(width=5., height=5.)})
    env.add_obstacle(Obstacle({'position': [0., 0.]}, shape=Circle(0.4), options={'spline_traj': True}))
    with pytest.raises(NotImplementedError, match='spline_traj'):
        b200.save_mpc_obstacles(Point2point(veh, env, options={'horizon_time': 10.}), path)


@pytest.mark.parametrize('name', ['config5', 'config_holonomic3d', 'config_freeT'])
def test_obstacle_file_round_trip(emu, tmp_path, name):
    pr = getattr(sc, name)(build_solver=False)
    path = str(tmp_path / 'p.omgobs')
    b200.save_mpc_obstacles(pr, path)
    od = b200.mpc_obstacles_desc(pr)
    D = emu.omg_mpc_obstacles_read(path.encode())
    assert D, emu.omg_last_error().decode()
    d = D.contents
    assert d.n_obs == od['n_obs']
    for key, kind in b200.MPC_OBSTACLE_FIELDS[1:]:
        assert np.array_equal(np.ctypeslib.as_array(getattr(d, key), (d.n_obs,)), od[key]), key
    emu.omg_mpc_obstacles_release(D)
    b200.save_mpc(sc.config1(build_solver=False), str(tmp_path / 'p.omgmpc'))
    assert not emu.omg_mpc_obstacles_read(str(tmp_path / 'p.omgmpc').encode())
    assert 'not an omg obstacle file' in emu.omg_last_error().decode()
    assert not emu.omg_mpc_obstacles_read(str(tmp_path / 'missing').encode())


# ---------------------------------------------------------------------------------------------
# native caller
# ---------------------------------------------------------------------------------------------
def _inputs(B, seed):
    """Config 2: jittered starts and goals, random radii and avoid flags."""
    pr = _plain('config2')
    s0, sT = _starts('config2', B, seed)
    desc = _desc(pr)
    obs = _obstacles_from_p(desc, np.repeat(desc['p_template'][None], B, 0))
    rng = np.random.default_rng(seed)
    shapes = _template_shapes(pr, B)
    for k in range(3):
        shapes[:, 3 * k + 2] = rng.uniform(0.3, 0.45, B)
    avoid = (rng.uniform(size=(B, 3)) < 0.6).astype(np.int32)
    return s0, sT, obs, shapes, avoid


def _native(tmp_path, lib_args, B, N, tl, s0, sT, obs, shapes, avoid):
    exe = str(tmp_path / 'native_mpc')
    subprocess.check_call(['g++', '-O2', '-I', os.path.join(ROOT, 'include'),
                           os.path.join(ROOT, 'examples', 'native', 'native_mpc.cpp'), '-o', exe] + lib_args)
    pr = _plain('config2')
    b200.save_tables(pr.father.tables, str(tmp_path / 'p.omgtbl'))
    b200.save_mpc(pr, str(tmp_path / 'p.omgmpc'))
    b200.save_mpc_obstacles(pr, str(tmp_path / 'p.omgobs'))
    for key, a in (('s0', s0), ('sT', sT), ('obs', obs), ('shapes', shapes)):
        np.ascontiguousarray(a, dtype=np.float64).tofile(str(tmp_path / (key + '.f64')))
    np.ascontiguousarray(avoid, dtype=np.int32).tofile(str(tmp_path / 'avoid.i32'))
    f = lambda k: str(tmp_path / k)  # noqa: E731
    out = subprocess.check_output([exe, f('p.omgtbl'), f('p.omgmpc'), str(B), str(N), str(tl), 'ideal',
                                   f('s0.f64'), f('sT.f64'), f('obs.f64'), f('traj.f64'), f('p.omgobs'),
                                   f('shapes.f64'), f('avoid.i32')])
    traj = np.fromfile(f('traj.f64')).reshape(N, 2, B, tl, -1)
    lines = [l.split() for l in out.decode().strip().splitlines()]
    return traj, np.array([[int(l[5]), int(l[7])] for l in lines]).reshape(N, B, 2)


def _python_loop(B, N, tl, s0, sT, obs, shapes, avoid, device):
    """DeviceMPC driven as native_mpc.cpp drives the C calls."""
    mpc = _mpc(sc.config2(), B, device, trajectory_length=tl)
    mpc.set_obstacles(_t(shapes, device), _i(avoid, device))
    s0, trajs, stat = s0.copy(), [], []
    for k in range(N):
        if k == N // 2:
            mpc.set_obstacles(avoid=_i(1 - avoid, device))
        xs, us, status, iters = mpc.update(_t(s0, device), _t(sT, device), _t(obs, device))
        xs, us, status = xs.cpu().numpy().copy(), us.cpu().numpy().copy(), status.cpu().numpy()
        ok = status == 0
        s0[ok] = xs[ok, 0]
        trajs.append((xs, us))
        stat.append(np.c_[status, iters.cpu().numpy()])
    return np.array(trajs), np.array(stat)


def test_native_mpc_caller_with_obstacles(emu, tmp_path):
    """native_mpc.cpp with an obstacle file, per-instance radii and avoid flags that it flips at update
    N / 2, linked to the emulation library: bit-identical to DeviceMPC driven the same way."""
    B, N, tl = 2, 4, 10
    args = _inputs(B, 4)
    traj, stat = _native(tmp_path, [emu_support.EMU_LIB, '-Wl,-rpath,' + os.path.dirname(emu_support.EMU_LIB)],
                         B, N, tl, *args)
    ref, ref_stat = _python_loop(B, N, tl, *args, 'cpu')
    assert np.array_equal(stat, ref_stat) and np.all(stat[0, :, 0] == 0)
    assert np.array_equal(traj, ref)


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_batch_1024_with_masks_and_shapes_matches_batch_1():
    """Config 2, jittered batch of 1024, random radii and avoid masks drawn anew at every one of 20 updates:
    a spread of instances equals batch-1 runs given the same shapes and flags, bit for bit."""
    B = 1024
    s0, sT, obs, shapes, avoid = _inputs(B, 9)
    mpc = _mpc(sc.config2(), B, 'cuda', trajectory_length=11)
    idx = np.array([0, 1, 517, 1023])
    ones = [_mpc(sc.config2(), 1, 'cuda', trajectory_length=11) for _ in idx]
    rng = np.random.default_rng(10)
    st0, stT, ob = _t(s0, 'cuda'), _t(sT, 'cuda'), _t(obs, 'cuda')
    n_off = 0
    for k in range(20):
        shapes[:, 2] = rng.uniform(0.3, 0.45, B)
        avoid = (rng.uniform(size=(B, 3)) < 0.7).astype(np.int32)
        n_off += int((avoid == 0).sum())
        mpc.set_obstacles(_t(shapes, 'cuda'), _i(avoid, 'cuda'))
        full = _outputs(mpc, mpc.update(st0, stT, ob))
        for b, one in zip(idx, ones):
            one.set_obstacles(_t(shapes[b:b + 1], 'cuda'), _i(avoid[b:b + 1], 'cuda'))
            got = _outputs(one, one.update(st0[b:b + 1].contiguous(), stT[b:b + 1].contiguous(),
                                           ob[b:b + 1].contiguous()))
            assert all(np.array_equal(g[0], f[b]) for g, f in zip(got, full)), (b, k)
    print('obstacle-instance-updates not avoided: %d of %d' % (n_off, 20 * B * 3))


@pytest.mark.gpu
def test_gpu_updates_and_set_calls_replay_from_a_cuda_graph():
    """Set calls and updates captured together with torch.cuda.graph on a side stream and replayed give
    bit-identical outputs and times to the eager run."""
    import torch
    B = 64
    s0, sT, obs, shapes, avoid = _inputs(B, 3)
    rng = np.random.default_rng(4)
    masks = [_i((rng.uniform(size=(B, 3)) < 0.5), 'cuda') for _ in range(10)]
    radii = []
    for k in range(10):
        s = shapes.copy()
        s[:, 5] = rng.uniform(0.3, 0.45, B)
        radii.append(_t(s, 'cuda'))
    st0, stT, ob = _t(s0, 'cuda'), _t(sT, 'cuda'), _t(obs, 'cuda')
    eager, graphed = (_mpc(sc.config2(), B, 'cuda', trajectory_length=20) for _ in range(2))
    for m in (eager, graphed):
        m.set_obstacles(_t(shapes, 'cuda'), _i(avoid, 'cuda'))
        m.update(st0, stT, ob)
    ref = []
    for k in range(10):
        eager.set_obstacles(radii[k], masks[k])
        ref.append([o.clone() for o in eager.update(st0, stT, ob)])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    outs = []
    side = torch.cuda.Stream()
    with torch.cuda.graph(g, stream=side):
        for k in range(10):
            graphed.set_obstacles(radii[k], masks[k])
            outs.append([o.clone() for o in graphed.update(st0, stT, ob)])
    g.replay()
    torch.cuda.synchronize()
    for k in range(10):
        for a, b in zip(outs[k], ref[k]):
            assert torch.equal(a, b), k
    assert np.array_equal(graphed.time, eager.time)


@pytest.mark.gpu
def test_gpu_native_mpc_caller_with_obstacles(tmp_path):
    """native_mpc.cpp with obstacles against libomgb200.so is bit-identical to the Python binding."""
    lib_dir = os.path.join(ROOT, 'omg_tools_b200', 'csrc')
    B, N, tl = 3, 4, 15
    args = _inputs(B, 6)
    traj, stat = _native(tmp_path, ['-L', lib_dir, '-lomgb200', '-Wl,-rpath,' + lib_dir], B, N, tl, *args)
    ref, ref_stat = _python_loop(B, N, tl, *args, 'cuda')
    assert np.array_equal(stat, ref_stat)
    assert np.array_equal(traj, ref)
