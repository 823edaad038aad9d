"""BatchMPC with a free motion time (FreeTPoint2point) and its two kernels: the per-instance warm
start omg_shift_free_batch (shift_spline from every instance's own T) and the per-instance
evaluation omg_eval_batch.

The tests without a mark run the kernel source on the CPU (tools/cpu_emu) against the host's
shift_spline and basis rows, the reference's own free-T loop (golden/freeT_loop_golden.npz,
make_freeT_loop_golden.py) and this framework's sequential host loop.  The ones marked gpu run the
same checks on the device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import emu_support                       # noqa: E402
from omg_tools_b200 import scenarios as sc          # noqa: E402
from omg_tools_b200.solver import b200              # noqa: E402

GOLDEN = os.path.join(HERE, 'golden', 'freeT_loop_golden.npz')
GOLDEN_TOL = (1e-5, 5e-6)          # x0, p: the ideal-loop tolerances of test_batch_mpc_vehicles.py
DT = 0.5
ITERS_NOT_COMPARED = 2         # final solves of a golden run whose iteration counts are not compared
# motion times over both branches of the reference's rule (T < 2 dt: u = T - dt, target = T), just
# above dt and just above 2 dt, and ones whose tau = u / target is outside (0, 1): left alone
T_SWEEP = [DT + 1e-9, DT + 1e-4, 0.7, 2 * DT - 1e-9, 2 * DT + 1e-9, 2 * DT + 1e-4, 1.6, 3.7, 10., 24.]
T_OUTSIDE = [0.3, DT, 2 * DT]


@pytest.fixture(scope='module')
def emu():
    saved = emu_support.activate()
    yield b200._lib
    emu_support.restore(saved)


def _torch(a, device):
    import torch
    return torch.tensor(np.ascontiguousarray(a), device=device)


def _rule(T):
    u, target = (T - DT, T) if T < 2 * DT else (DT, T - DT)
    return u / target, target


def _product_block(n):
    """A block on the product basis of two degree-2 splines (repeated interior knots, as the
    Dubins substitution's dx, dy of a degree-2 vehicle basis)."""
    from omg_tools_b200.basics.spline import BSplineBasis
    b = BSplineBasis([0., 0., 0., .2, .4, .6, .8, 1., 1., 1.], 2)
    prod = b * b
    assert len(np.unique(prod.knots)) < len(prod.knots) - 2 * prod.degree - 2 + 2
    L = len(prod)
    assert L <= n
    return (0, L, 1, prod.degree, prod.knots)


SHIFT_CASES = ['config_freeT', 'config_warehouse', 'config_dubins_freeT']


def _check_shift(name, B, device, rng):
    """omg_shift_free_batch against shift_spline on every shifted block of the scenario (and the
    product basis with repeated knots, on a copy of x); returns the largest relative error."""
    from omg_tools_b200.basics.spline import BSplineBasis
    from omg_tools_b200.basics.spline_extra import shift_spline
    pr = getattr(sc, name)()
    f = pr.father
    ti = f._var_struct.entries[(pr.label, 'T')][0]
    err = 0.
    for blocks in (b200.spline_blocks(f), [_product_block(f.tables.n)]):
        Ts = np.array(T_SWEEP + T_OUTSIDE)
        Ts = np.resize(Ts, B) if B >= len(Ts) else Ts[rng.integers(0, len(Ts), B)]
        X = rng.standard_normal((B, f.tables.n))
        if blocks[0][0] <= ti < blocks[0][0] + blocks[0][1]:      # (product block over T)
            ti_use = f.tables.n - 1
        else:
            ti_use = ti
        X[:, ti_use] = Ts
        active = (rng.uniform(size=B) < 0.85).astype(np.int32)
        active[:min(B, len(T_SWEEP))] = 1
        Xt = _torch(X, device)
        pr.problem.shift_free_batch_device(Xt, blocks, ti_use, DT, active=_torch(active, device))
        Y = Xt.cpu().numpy()
        check = np.unique(np.r_[np.arange(min(B, len(T_SWEEP) + len(T_OUTSIDE))),
                                rng.integers(0, B, 24), B - 1])
        for b in check:
            tau, target = _rule(Ts[b])
            if not active[b] or not 0. < tau < 1.:
                assert np.array_equal(Y[b], X[b]), (name, b, Ts[b])
                continue
            assert Y[b, ti_use] == target, (name, b)
            for off, L, nc, p, knots in blocks:
                c = X[b, off:off + L * nc].reshape(nc, L).T
                ref = shift_spline(c, tau, BSplineBasis(knots, p))
                got = Y[b, off:off + L * nc].reshape(nc, L).T
                e = np.abs(got - ref).max() / np.abs(c).max()
                err = max(err, e)
                assert e < 1e-12, (name, b, Ts[b], off, e)
    return err


def _check_eval(B, device, rng):
    """omg_eval_batch against _rows (eval_basis and basis.derivative) on the vehicle and an
    environment block of two scenarios: tau at 0, 1, on knots, random, and padding outside the
    span; derivatives 0..3 divided by scale^d."""
    from omg_tools_b200.basics.spline import BSplineBasis
    from omg_tools_b200.execution.batch_mpc import _rows
    err = 0.
    for name in ('config_freeT', 'config_dubins_freeT'):
        pr = getattr(sc, name)(build_solver=False)
        blocks = b200.spline_blocks(pr.father)
        blocks = [blocks[0], blocks[-1]]                           # vehicle (degree 3), environment (degree 1)
        X = rng.standard_normal((B, pr.father.tables.n))
        n_pts = 9
        tau = rng.uniform(0., 1., (B, n_pts))
        tau[:, 0], tau[:, 1], tau[:, 2], tau[:, 3] = 0., 1., 0.2, 0.6
        tau[:, 4], tau[:, 5] = -1., 0.                             # padding
        scale = rng.uniform(0.3, 12., B)
        for n_der in (1, 2, 4):
            use = [b for b in blocks if b[3] + 1 >= n_der]
            out = b200.eval_batch(_torch(X, device), use, _torch(tau, device), _torch(scale, device),
                                  n_der).cpu().numpy()
            check = np.unique(np.r_[0, rng.integers(0, B, 12), B - 1])
            for b in check:
                o = 0
                for off, L, nc, p, knots in use:
                    R = _rows(BSplineBasis(knots, p), tau[b], scale[b], n_der)   # [d, point, L]
                    for c in range(nc):
                        ref = np.einsum('dpl,l->pd', R, X[b, off + c * L:off + (c + 1) * L])
                        got = out[b, o:o + n_pts * n_der].reshape(n_pts, n_der)
                        o += n_pts * n_der
                        e = np.abs(got - ref).max() / max(1., np.abs(ref).max())
                        err = max(err, e)
                        assert e < 1e-12, (name, n_der, b, off, c, e)
                assert o == out.shape[1]
    return err


@pytest.mark.parametrize('name', SHIFT_CASES)
def test_shift_free_matches_shift_spline(emu, name):
    """Every shifted block (degrees 1 and 3; Dubins' dx, dy) and a product basis with repeated
    interior knots, a sweep of T over both branches of the reference's rule: shift_spline to 1e-12
    of the largest coefficient and T written as the target; inactive instances and tau outside
    (0, 1) untouched bit for bit."""
    err = _check_shift(name, 16, 'cpu', np.random.default_rng(1))
    print('%s: %.1e' % (name, err))


def test_eval_matches_the_basis_rows(emu):
    err = _check_eval(5, 'cpu', np.random.default_rng(2))
    print('eval: %.1e' % err)


def _args_shift(h, buf):
    def keep(name, a):
        buf[name] = a
        return a.ctypes.data
    X = np.zeros(40)
    X[30] = 3.
    return [h, 1, keep('x', X), 30, DT, None, 1, keep('o', np.array([0], np.int32)),
            keep('l', np.array([5], np.int32)), keep('c', np.array([2], np.int32)),
            keep('p', np.array([3], np.int32)), keep('k', np.r_[0., 0, 0, 0, .5, 1, 1, 1, 1]), None]


def test_bad_arguments_are_rejected(emu):
    """Both entry points: the valid call passes; each bad argument is rejected with a message."""
    pr = sc.config_freeT()
    h = pr.problem._handle
    n = pr.father.tables.n
    buf = {}
    assert emu.omg_shift_free_batch(*_args_shift(h, buf)) == 0, emu.omg_last_error()
    f = 'omg_shift_free_batch: '
    big = np.r_[np.zeros(10), np.linspace(0, 1, 41), np.ones(10)]
    for index, value, message in (
            (4, 0., 'update_time must be > 0'), (4, -1., 'update_time must be > 0'),
            (3, -1, 't_index -1 outside [0, %d)' % n), (3, n, 't_index %d outside' % n),
            (2, None, 'null argument'), (7, None, 'null argument'), (0, None, 'null argument'),
            (10, np.array([9], np.int32), 'degree 9'), (9, np.array([n], np.int32), 'columns outside x'),
            (8, np.array([3], np.int32), 'basis length 3'), (11, np.r_[0., 0, 0, 0, .5, 1, .9, 1, 1], 'knots'),
            (8, np.array([49], np.int32), 'basis length 49')):
        args = _args_shift(h, buf)
        if isinstance(value, np.ndarray):
            buf[index] = value
            args[index] = value.ctypes.data
            if index == 8 and value[0] == 49:
                buf['big'] = np.r_[np.zeros(3), np.linspace(0, 1, 47), np.ones(3)]
                args[11] = buf['big'].ctypes.data
        else:
            args[index] = value
        assert emu.omg_shift_free_batch(*args) == -1, (index, value)
        err = emu.omg_last_error().decode()
        assert err.startswith(f) and message in err, err
    del big
    # omg_eval_batch
    X, tau, scale, out = np.zeros((1, 40)), np.zeros((1, 3)), np.ones(1), np.zeros(100)
    o, l, c, p = (np.array([v], np.int32) for v in (0, 5, 2, 3))
    k = np.r_[0., 0, 0, 0, .5, 1, 1, 1, 1]
    ok = [1, 40, X.ctypes.data, 1, o.ctypes.data, l.ctypes.data, c.ctypes.data, p.ctypes.data, k.ctypes.data, 3,
          tau.ctypes.data, scale.ctypes.data, 4, out.ctypes.data, None]
    assert emu.omg_eval_batch(*ok) == 0, emu.omg_last_error()
    p1 = np.array([1], np.int32)
    k1 = np.r_[0., 0, .25, .5, .75, 1, 1]
    for index, value, message in ((12, 0, 'n_der 0 outside 1 .. 4'), (12, 5, 'n_der 5 outside 1 .. 4'),
                                  (9, 0, 'n_pts must be >= 1'), (10, None, 'null argument'),
                                  (11, None, 'null argument'), (13, None, 'null argument'),
                                  (7, p1.ctypes.data, 'n_der 4 above degree + 1 = 2'),
                                  (1, 9, 'columns outside x')):
        args = list(ok)
        args[index] = value
        if index == 7:
            args[6] = np.array([2], np.int32).ctypes.data
            args[8] = k1.ctypes.data
            l5 = np.array([5], np.int32)
            args[5] = l5.ctypes.data
        assert emu.omg_eval_batch(*args) == -1, (index, value)
        err = emu.omg_last_error().decode()
        assert err.startswith('omg_eval_batch: ') and message in err, err


# ---------------------------------------------------------------------------------------------
# BatchMPC
# ---------------------------------------------------------------------------------------------
def _batch(name, batch, device, seed=0, jitter=0., **kw):
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    return BatchMPC(getattr(sc, name)(**kw), batch=batch, update_time=DT, device=device, seed=seed,
                    jitter=jitter)


def _record_solves(bat, replay=None):
    """Record what every solve is handed (x0, p of the instances solved); with ``replay`` (solutions
    x [steps, n]) the solution of step k is replaced by replay[k], so the loop around the solver runs
    on those trajectories."""
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


def _check_golden(name, batch, device):
    """BatchMPC against the reference's free-T loop.  The solutions are the reference's (replayed):
    the free-T optima are not unique in the separating hyperplanes, and the rounding of the solver
    builds moves them apart after a few steps; on the reference's own trajectories x0, p, T, the
    statuses, the iteration counts, the stop step and the final state are compared."""
    import torch
    G = np.load(GOLDEN)
    n_steps = len(G[name + '_status'])
    bat = _batch(name, batch, torch.device(device))
    calls = _record_solves(bat, G[name + '_x'])
    bat.run(n_steps + 5)
    assert len(calls) == n_steps and not bat.active.any(), (len(calls), n_steps)
    err = np.zeros(3)
    for k in range(n_steps):
        X0, P = calls[k]
        e = [np.abs(X0 - G[name + '_x0'][k][None]).max(), np.abs(P - G[name + '_p'][k][None]).max(),
             np.abs(bat.history['T'][k] - G[name + '_T'][k]).max()]
        err = np.maximum(err, e)
        assert e[0] < GOLDEN_TOL[0] and e[1] < GOLDEN_TOL[1] and e[2] < GOLDEN_TOL[0], (name, k, e)
        assert np.all(bat.history['status'][k] == G[name + '_status'][k]), (name, k)
    # iteration counts: on the same x0 the kernel and the C oracle round differently, and the last
    # two solves of a run (T within two updates of the end) amplify it by a few iterations: 27 and 93
    # against the oracle's 26 and 62 in the moving-obstacle run on the CPU emulation, 32 against 31
    # in config_freeT's second-to-last solve on an H100.  Those two are not compared.
    n_cmp = n_steps - ITERS_NOT_COMPARED
    its = np.array(bat.history['iters'][:n_cmp])
    assert np.all(its == G[name + '_iters'][:n_cmp, None]), (name, its[:, 0], G[name + '_iters'])
    e_final = np.abs(bat.state - G[name + '_state'][None]).max()
    print('%s batch %d: x0 %.1e, p %.1e, T %.1e, final state %.1e' % ((name, batch) + tuple(err) + (e_final,)))
    assert e_final < 1e-4, e_final


@pytest.mark.parametrize('batch', [1, 3])
@pytest.mark.parametrize('name', ['config_freeT', 'config_freeT_moving'])
def test_batch_mpc_follows_the_references_freeT_loop(emu, name, batch):
    """The reference's predict / solve (init_step with shift_spline, T <- target) / store / simulate
    / stop_criterium loop at 0.5 s updates: every instance of a batch of identical copies gets the
    reference's x0 and p and reaches the reference's T at every step, with equal statuses and
    iteration counts (but for the last two solves), stops at the same step and ends in the same state (within 1e-4: the
    reference's last update moves the vehicle by T rounded to its 0.01 s samples)."""
    _check_golden(name, batch, 'cpu')


def test_dubins_freeT_follows_the_host_loop(emu):
    """config_dubins_freeT (init_v_til = 0.3) against this framework's sequential host loop
    (predict / solve / store / simulate / stop_criterium, init_step inside Problem.solve as the
    reference's Deployer calls it), whose solutions are replayed: x0 without the dx, dy entries
    (which the reference does not shift), p and T at every step, the stop step and the final state
    (its last T is below the sample time: the vehicle does not move in that update)."""
    import torch
    from oracle import ipm_c
    if not ipm_c.available():
        pytest.skip('C oracle not built')
    from test_model import _OracleSolver

    class Recorder(_OracleSolver):
        def __call__(self, x0, p, lbg, ubg, **kw):
            r = _OracleSolver.__call__(self, x0, p, lbg, ubg)
            self.calls.append((np.asarray(x0, float).copy(), np.asarray(p, float).copy(), r['x'].copy()))
            return r
    pr = sc.config_dubins_freeT(build_solver=False, init_v_til=0.3)
    pr.problem = Recorder(pr.father.tables)
    pr.problem.calls = []
    pr.initialize(0.)
    t, Ts = 0., []
    for k in range(30):
        pr.predict(t, DT, 0.01)
        pr.solve(t, DT)
        assert pr.problem.stats()['return_status'] == 'Solve_Succeeded', k
        Ts.append(pr.horizon_time())
        pr.store(t, DT, 0.01)
        pr.simulate(t, DT, 0.01)
        t = np.round(t + DT, 6)
        if pr.stop_criterium(t, DT):
            break
    host = pr.problem.calls
    bat = _batch('config_dubins_freeT', 1, torch.device('cpu'), init_v_til=0.3)
    calls = _record_solves(bat, np.array([c[2] for c in host]))
    bat.run(40)
    assert len(calls) == len(host)
    ent = bat.father._var_struct.entries
    keep = np.ones(bat.tb.n, dtype=bool)
    for nm in ('dx', 'dy'):
        off, size, _ = ent[(bat.vehicle.label, nm)]
        keep[off:off + size] = False
    err = np.zeros(3)
    for k, (x0, p, _) in enumerate(host):
        e = [np.abs(calls[k][0][0] - x0)[keep].max(), np.abs(calls[k][1][0] - p).max(),
             abs(bat.history['T'][k][0] - Ts[k])]
        err = np.maximum(err, e)
        assert e[0] < GOLDEN_TOL[0] and e[1] < GOLDEN_TOL[1] and e[2] < 1e-9, (k, e)
    print('dubins freeT: %d steps, x0 %.1e, p %.1e, T %.1e' % ((len(host),) + tuple(err)))
    assert np.abs(bat.state[0] - pr.vehicles[0].signals["state"][:, -1]).max() < 1e-3


def _instance_alone(bat, b, device):
    """A batch-1 BatchMPC of instance b of ``bat`` before its first step (its start and goal)."""
    one = _batch('config_freeT', 1, device)
    one.veh.state[0], one.veh.poseT[0] = bat.veh.state[b], bat.veh.poseT[b]
    X0 = np.repeat(one.father.get_variables().cat[None], 1, 0)
    one.veh.cold_start(X0)
    one.X.copy_(_torch(X0, device))
    one.history['state'] = [one.state.copy()]
    return one


def _jittered(device, sched=None, B=4, steps=40):
    bat = _batch('config_freeT', B, device, seed=7, jitter=0.6)
    ones = [_instance_alone(bat, b, device) for b in range(B)]
    bat.run(steps)
    return bat, ones


def test_instances_are_independent(emu, monkeypatch):
    """A jittered batch of 4 whose instances stop at different steps: each instance's history is
    the batch-1 run's bit for bit; after it stops its X, state and T do not change; the reversed
    and random thread schedules of the emulation give the same histories."""
    import torch
    dev = torch.device('cpu')
    bat, ones = _jittered(dev)
    act = np.array(bat.history['active'])
    stops = act.sum(axis=0)
    assert not bat.active.any() and len(set(stops.tolist())) > 1, stops
    for b, one in enumerate(ones):
        one.run(40)
        n = len(one.history['status'])
        assert n == stops[b]
        for key in ('status', 'iters', 'T'):
            assert all(np.array_equal(bat.history[key][k][b], one.history[key][k][0]) for k in range(n)), (b, key)
        for k in range(len(bat.history['state'])):
            assert np.array_equal(bat.history['state'][k][b], one.history['state'][min(k, n)][0]), (b, k)
        assert np.array_equal(bat.X[b].numpy(), one.X[0].numpy())
        for k in range(n, len(bat.history['T'])):
            assert bat.history['T'][k][b] == bat.history['T'][n - 1][b] and bat.history['status'][k][b] == -1
    for sched in ('reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        other = _batch('config_freeT', 4, dev, seed=7, jitter=0.6)
        other.run(40)
        for key in ('state', 'T', 'iters', 'status'):
            assert all(np.array_equal(x, y) for x, y in zip(bat.history[key], other.history[key])), (sched, key)
        assert np.array_equal(bat.X.numpy(), other.X.numpy())


def test_unsupported_free_T_settings_raise():
    """Free end time: vehicles without a per-instance prediction and the closed loop raise."""
    import torch
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    with pytest.raises(NotImplementedError, match='free end time'):
        BatchMPC(sc.config_trailer(build_solver=False), 1, device=torch.device('cpu'))
    pr = sc.config_freeT(build_solver=False)
    pr.vehicles[0].set_options({'ideal_update': False})
    with pytest.raises(NotImplementedError, match='ideal_update and ideal_prediction'):
        BatchMPC(pr, 1, device=torch.device('cpu'))


# ---------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('B', [1, 1024, 4096])
def test_gpu_kernels_match_the_host(B):
    """The warm start and the evaluation on the device, beyond the resident blocks at 4096."""
    rng = np.random.default_rng(B)
    for name in SHIFT_CASES:
        print('%s B %d: %.1e' % (name, B, _check_shift(name, B, 'cuda', rng)))
    print('eval B %d: %.1e' % (B, _check_eval(B, 'cuda', rng)))


@pytest.mark.gpu
def test_gpu_batch_mpc_follows_the_references_freeT_loop():
    for name in ('config_freeT', 'config_freeT_moving'):
        _check_golden(name, 1, 'cuda')


@pytest.mark.gpu
def test_gpu_batch_256_freeT():
    """A jittered batch of 256 config_freeT loops at 0.5 s updates: every instance stops within 40
    steps at its goal (1e-2), its T drops by the update time per step (within 0.15, as the host
    test asserts), and instance 0 is a batch-1 run bit for bit."""
    import torch
    dev = torch.device('cuda')
    bat = _batch('config_freeT', 256, dev, seed=3, jitter=0.1)
    one = _batch('config_freeT', 1, dev, seed=3)
    bat.run(40)
    one.run(40)
    assert not bat.active.any()
    assert np.abs(bat.state - bat.poseT).max() < 1e-2
    T, act = np.array(bat.history['T']), np.array(bat.history['active'])
    for b in range(256):
        Tb = T[act[:, b], b]
        assert np.abs(np.diff(Tb) + DT).max() < 0.15, (b, Tb)
    n = len(one.history['status'])
    for key in ('status', 'iters', 'T'):
        assert all(np.array_equal(bat.history[key][k][0], one.history[key][k][0]) for k in range(n)), key
    assert np.array_equal(bat.X[0].cpu().numpy(), one.X[0].cpu().numpy())
    print('batch 256: stopped after %s steps' % np.unique(act.sum(axis=0)))
