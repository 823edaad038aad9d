"""Batched receding-horizon driver: B independent copies of one Point2point
scenario (Holonomic, Holonomic3D, Quadrotor3D, Dubins, HolonomicOrient, planar Quadrotor or
SimpleQuadrotor3D vehicle, or a fleet of Holonomic / Holonomic3D vehicles) advance in lock step,
every MPC step is ONE batched solve on the GPU.

It is the batched counterpart of the reference's ``Simulator.run()`` /
``Deployer.update()`` loop (omgtools/execution/simulator.py:39-99,
deployer.py:43-79).  With the vehicle options ideal_prediction and ideal_update on
(this repository's defaults) the vehicle follows its spline:

    per step:   predict  -> state0/input0 = spline and derivative at t + update_time
                init_step-> knot-crossing shift T.dot(coeffs) of the seg0 variables
                            (point2point.py:187-198)          [omg_shift_batch]
                set_parameters -> t, T, state0, input0, obstacle x/v/a/theta
                            (point2point.py:174-181, obstacle.py:142-155,345-348)
                solve    -> problem(x0, p, lbg, ubg)          [omg_solve_batch]

The decision variables stay resident on the device between steps (warm start);
only the parameter rows (n_par doubles per instance) travel each step.

With either flag off (the reference's defaults) the loop is closed through the vehicle's
own dynamics: after each solve ONE launch (omg_closed_loop_step) integrates the vehicle ODE
from the plant state, once on the planned inputs plus the input disturbance and through the
first-order actuator lag (simulate: the next plant state), once on the clean planned inputs
(predict: state0 of the next solve).  Options read from the vehicle: ideal_update,
ideal_prediction, 1storder_delay, time_constant, input_disturbance {fc, stdev, mean}; the noise
is keyed by ``seed``, the MPC step and the instance, so a realisation does not depend on the
batch size.

Several vehicles in one problem (inter-vehicle avoidance, the central formation) run with a fixed horizon for fleets
of Holonomic or Holonomic3D vehicles that share one spline basis and one set of plant options: one adapter per
vehicle (``vehs``; ``veh`` is vehicle 0) reads its splines at its own column of x, the jitter shifts all starts of an
instance by one vector and all goals by another, the closed loop is ONE launch for the fleet
(omg_closed_loop_step_fleet; vehicle v's noise is signal v * n_input + j of the instance), and ``state``, ``inp``,
``poseT`` and history['state'|'plant'|'plant_input'] are [B, n_veh, ·].  Any other multi-vehicle problem raises
NotImplementedError naming the cause.  history['plant'] and history['plant_input'] hold the plant state and the last
applied input at every update boundary.  ``sample_time`` is the simulation grid of the plant
and of the obstacle motion (the reference simulator's sample_time, 0.01 s by default).

With a FreeTPoint2point (T a decision variable; Holonomic, Holonomic3D, Dubins, HolonomicOrient, the planar
Quadrotor and SimpleQuadrotor3D) every instance
runs the reference's free-T loop on its own motion time (point2point.py:300-374): the warm start
re-expresses the splines with shift_spline from the instance's T [omg_shift_free_batch], only the
instances still running are solved, the prediction samples each plan at its own
tau = min(dt, T) / T [omg_eval_batch], and an instance stops for good when T < dt or at its goal (the
adapter's ``arrived``: the quadrotors compare their position with the target and test the planned
velocity dspl, which the closed loop also reads from the plan at each instance's own tau).
history['T'] and history['active'] hold the motion times and the instances solved at every step.
The free-T loop runs ideal, or closed with ideal_prediction off (ideal_update on or off): one launch
[omg_closed_loop_step_free] on the whole batch samples each moving instance's plan on its own time
axis for min(dt, T) / sample_time samples and filters its disturbance over its own stored trajectory,
T / sample_time + 1 samples; state0 of the next solve is the kernel's prediction, and the stop test
reads the plant, as the reference's check_terminal_conditions reads signals.  A final update with at
most 12 trajectory samples (T < 0.12 s at 0.01 s samples), where the reference's filtfilt would raise,
gets no disturbance.  ideal_update off with ideal_prediction on raises: that prediction never looks at
the plant, while the free-T stop test reads it.
"""
import numpy as np


class _HolonomicAdapter(object):
    """Holonomic / Holonomic3D: state = position spline value, input = its
    derivative / T (holonomic.py:87-105, 153-159)."""

    N_DER = 2       # rows of spline derivatives the plant step reads (value, first derivative)

    def __init__(self, mpc, vehicle, batch, jitter, rng, x_off=0):
        self.mpc, self.v = mpc, vehicle
        self.x_off = x_off      # column of the vehicle's splines in x (several vehicles in one problem)
        self.nd = nd = vehicle.n_dim
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.poseT = rep(vehicle.poseT)
        if jitter > 0:
            self.state[1:] += rng.uniform(-jitter, jitter, (batch - 1, nd))
            self.poseT[1:] += rng.uniform(-jitter, jitter, (batch - 1, nd))

    def cold_start(self, X0):
        L, o = len(self.v.basis), self.x_off
        for k in range(self.nd):
            X0[:, o + k * L:o + (k + 1) * L] = np.linspace(self.state[:, k], self.poseT[:, k], L).T

    def pack(self, P, off):
        v, nd = self.v.label, self.nd
        P[:, off[(v, 'state0')]:off[(v, 'state0')] + nd] = self.state
        P[:, off[(v, 'input0')]:off[(v, 'input0')] + nd] = self.inp
        P[:, off[(v, 'poseT')]:off[(v, 'poseT')] + nd] = self.poseT

    def predict(self, X, t_rel, dt, T, device=True):
        from ..solver.b200 import sample_batch
        basis, nd = self.v.basis, self.nd
        tau = (t_rel + dt) / T
        B0 = basis.eval_basis([tau])
        Bd, P1 = basis.derivative(1)
        B1 = Bd.eval_basis([tau]).dot(P1) / T
        L = len(basis)
        if device:
            out = sample_batch(X, [(self.x_off, L, nd, np.vstack([B0, B1]))]).cpu().numpy()
            # layout: [column][sample] with samples (value, derivative)
            for k in range(nd):
                self.state[:, k], self.inp[:, k] = out[:, 2 * k], out[:, 2 * k + 1]
        else:
            Xh = X.cpu().numpy()
            for k in range(nd):
                c = Xh[:, self.x_off + k * L:self.x_off + (k + 1) * L]
                self.state[:, k] = c.dot(B0[0])
                self.inp[:, k] = c.dot(B1[0])

    def predict_free(self, X, idx, tau1, T, blocks):
        """Free motion time: state and input of the instances idx (X holds their rows) at their
        own tau1 = min(dt, T) / T, value and first derivative / T (omg_eval_batch)."""
        out = _eval(X, blocks, tau1[:, None], T, 2).reshape(-1, self.nd, 2)   # [b][column][derivative]
        self.state[idx], self.inp[idx] = out[:, :, 0], out[:, :, 1]

    def arrived(self, state, inp, idx, tol):
        """Free-T stop test of the instances idx (holonomic.py check_terminal_conditions)."""
        return _at_goal(state, inp, self.poseT[idx], tol)

    def position(self):
        return self.state


class _Quadrotor3DAdapter(object):
    """Quadrotor3D (quadrotor3d.py): the decision splines are the flat outputs
    f~, q_phi, q_theta; position and velocity follow from the double integral of
    the accelerations re-anchored at the previous prediction (splines2signals,
    quadrotor3d.py:253-275).  The integral over one update is taken exactly by
    Gauss-Legendre quadrature per knot piece on device-sampled spline values."""

    NQ = 6      # exact for the degree-9 integrand (tau1 - s) * ddx(s)
    N_DER = 2

    def __init__(self, mpc, vehicle, batch, jitter, rng):
        self.mpc, self.v = mpc, vehicle
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.poseT = rep(vehicle.poseT)
        if jitter > 0:
            self.state[1:, :3] += rng.uniform(-jitter, jitter, (batch - 1, 3))
            self.poseT[1:, :3] += rng.uniform(-jitter, jitter, (batch - 1, 3))

    def cold_start(self, X0):
        L = len(self.v.basis)
        q0 = np.tan(self.state[:, 6:8] / 2.)
        qT = np.tan(self.poseT[:, 3:5] / 2.)
        for k in range(2):
            X0[:, (k + 1) * L:(k + 2) * L] = np.linspace(q0[:, k], qT[:, k], L).T

    def pack(self, P, off):
        v = self.v.label
        st, inp = self.state, self.inp
        qp, qt = np.tan(st[:, 6] / 2.), np.tan(st[:, 7] / 2.)
        def put(name, val):
            val = np.asarray(val, dtype=float)
            val = val[:, None] if val.ndim == 1 else val
            P[:, off[(v, name)]:off[(v, name)] + val.shape[1]] = val

        put('q_phi0', qp), put('q_theta0', qt)
        put('f_til0', inp[:, 0] / ((1 + qp**2) * (1 + qt**2)))
        put('dq_phi0', 0.5 * inp[:, 1] * (1 + qp**2))
        put('dq_theta0', 0.5 * inp[:, 2] * (1 + qt**2))
        put('pos0', st[:, :3]), put('dpos0', st[:, 3:6])
        put('posT', self.poseT[:, :3])
        put('q_phiT', np.tan(self.poseT[:, 3] / 2.)), put('q_thetaT', np.tan(self.poseT[:, 4] / 2.))

    def predict(self, X, t_rel, dt, T, device=True):
        from ..solver.b200 import sample_batch
        basis, g = self.v.basis, self.v.g
        L = len(basis)
        tau0, tau1 = t_rel / T, (t_rel + dt) / T
        # quadrature nodes on [tau0, tau1], split at the knots in between
        brk = [tau0] + [k for k in np.unique(basis.knots) if tau0 + 1e-12 < k < tau1 - 1e-12] + [tau1]
        xg, wg = np.polynomial.legendre.leggauss(self.NQ)
        nodes = np.concatenate([0.5 * (b - a) * xg + 0.5 * (a + b) for a, b in zip(brk[:-1], brk[1:])])
        wts = np.concatenate([0.5 * (b - a) * wg for a, b in zip(brk[:-1], brk[1:])])
        S0 = basis.eval_basis(np.r_[nodes, tau1])
        Bd, P1 = basis.derivative(1)
        S1 = Bd.eval_basis([tau1]).dot(P1)
        ns = len(nodes) + 1
        if device:
            out = sample_batch(X, [(0, L, 3, np.vstack([S0, S1]))]).cpu().numpy()
        else:
            Xh = X.cpu().numpy()
            out = np.concatenate([Xh[:, k * L:(k + 1) * L].dot(np.vstack([S0, S1]).T)
                                  for k in range(3)], axis=1)
        col = lambda k: out[:, k * (ns + 1):(k + 1) * (ns + 1)]
        f, qp, qt = col(0)[:, :ns - 1], col(1)[:, :ns - 1], col(2)[:, :ns - 1]
        acc = np.stack([f * (1 - qp**2) * (2 * qt), -f * (1 + qt**2) * (2 * qp),
                        f * (1 - qp**2) * (1 - qt**2) - g], axis=2)          # [B, nodes, 3]
        I1 = np.einsum('q,bqk->bk', wts, acc)
        I2 = np.einsum('q,bqk->bk', wts * (tau1 - nodes), acc)
        pos, vel = self.state[:, :3], self.state[:, 3:6]
        new_pos = pos + T * vel * (tau1 - tau0) + T * T * I2
        new_vel = vel + T * I1
        f1, qp1, qt1 = col(0)[:, ns - 1], col(1)[:, ns - 1], col(2)[:, ns - 1]
        dqp1, dqt1 = col(1)[:, ns] / T, col(2)[:, ns] / T
        self.state = np.c_[new_pos, new_vel, 2 * np.arctan2(qp1, 1), 2 * np.arctan2(qt1, 1)]
        self.inp = np.c_[f1 * (1 + qp1**2) * (1 + qt1**2), 2 * dqp1 / (1 + qp1**2),
                         2 * dqt1 / (1 + qt1**2)]

    def position(self):
        return self.state[:, :3]


def _rows(basis, tau, T, n_der):
    """Rows of the basis and of its derivatives 1..n_der-1 at tau, derivative d divided by
    T^d: [n_der, len(tau), L]."""
    rows = [basis.eval_basis(tau)]
    for d in range(1, n_der):
        Bd, Pd = basis.derivative(d)
        rows.append(Bd.eval_basis(tau).dot(Pd) / T**d)
    return np.array(rows)


def _eval(X, blocks, tau, T, n_der):
    """Per-instance spline values and derivatives 0..n_der-1 at the abscissae tau [B, n_pts], derivative
    d divided by T^d (omg_eval_batch): numpy [B, columns * n_pts * n_der], column / point / derivative."""
    import torch
    from ..solver.b200 import eval_batch
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=X.device)
    return eval_batch(X, blocks, t(tau), t(T), n_der).cpu().numpy()


def _sample(X, L, n_col, S, device):
    """Spline columns 0..n_col-1 of every instance at the rows S [n_rows, L]: [B, n_col * n_rows]
    laid out column / row (on the device by omg_sample_batch, or on the host)."""
    from ..solver.b200 import sample_batch
    if device:
        return sample_batch(X, [(0, L, n_col, S)]).cpu().numpy()
    Xh = X.cpu().numpy()
    return np.concatenate([Xh[:, k * L:(k + 1) * L].dot(S.T) for k in range(n_col)], axis=1)


def _put(P, off, label, name, val):
    val = np.asarray(val, dtype=float)
    val = val[:, None] if val.ndim == 1 else val
    P[:, off[(label, name)]:off[(label, name)] + val.shape[1]] = val


def _at_goal(state, inp, poseT, tol):
    """check_terminal_conditions of the vehicles whose state is their pose: the state at the target
    and the input at rest (the reference's (a > tol or b) > tol, for stop_tol < 1)."""
    return (np.linalg.norm(state - poseT, axis=1) <= tol) & (np.linalg.norm(inp, axis=1) <= tol)


class _DubinsAdapter(object):
    """Dubins (dubins.py, every formulation): the decision splines are v~ and tg = tan(theta/2);
    the position is the running integral of v~ (1 - tg^2), 2 v~ tg re-anchored at the previous
    prediction (splines2signals, integrate_once).  The integral over one update is taken exactly
    by Gauss-Legendre quadrature per knot piece on device-sampled spline values."""

    N_DER = 2

    def __init__(self, mpc, vehicle, batch, jitter, rng):
        self.mpc, self.v = mpc, vehicle
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.poseT = rep(vehicle.poseT)
        if jitter > 0:
            self.state[1:, :2] += rng.uniform(-jitter, jitter, (batch - 1, 2))
            self.poseT[1:, :2] += rng.uniform(-jitter, jitter, (batch - 1, 2))
        self.nq = (3 * vehicle.degree + 2) // 2     # exact for the degree-3d integrand

    def cold_start(self, X0):
        L = len(self.v.basis)
        X0[:, :L] = self.v.options.get('init_v_til', 0.)
        X0[:, L:2 * L] = np.linspace(np.tan(self.state[:, 2] / 2.), np.tan(self.poseT[:, 2] / 2.), L).T

    def pack(self, P, off):
        v, st, inp = self.v.label, self.state, self.inp
        tg = np.tan(st[:, 2] / 2.)
        _put(P, off, v, 'tg_ha0', tg)
        _put(P, off, v, 'v_til0', inp[:, 0] / (1 + tg**2))
        _put(P, off, v, 'dtg_ha0', 0.5 * inp[:, 1] * (1 + tg**2))
        _put(P, off, v, 'pos0', st[:, :2])
        _put(P, off, v, 'posT', self.poseT[:, :2])
        _put(P, off, v, 'tg_haT', np.tan(self.poseT[:, 2] / 2.))

    def predict(self, X, t_rel, dt, T, device=True):
        basis = self.v.basis
        L = len(basis)
        tau0, tau1 = t_rel / T, (t_rel + dt) / T
        brk = [tau0] + [k for k in np.unique(basis.knots) if tau0 + 1e-12 < k < tau1 - 1e-12] + [tau1]
        xg, wg = np.polynomial.legendre.leggauss(self.nq)
        nodes = np.concatenate([0.5 * (b - a) * xg + 0.5 * (a + b) for a, b in zip(brk[:-1], brk[1:])])
        wts = np.concatenate([0.5 * (b - a) * wg for a, b in zip(brk[:-1], brk[1:])])
        R = _rows(basis, [tau1], T, 2)
        nn = len(nodes)
        out = _sample(X, L, 2, np.vstack([basis.eval_basis(nodes), R[0], R[1]]), device)
        vt, tg = out[:, :nn], out[:, nn + 2:2 * nn + 2]
        vt1, tg1, dtg1 = out[:, nn], out[:, 2 * nn + 2], out[:, 2 * nn + 3]
        q1 = 1 + tg1**2
        self.state = np.c_[self.state[:, 0] + T * (vt * (1 - tg**2)).dot(wts),
                           self.state[:, 1] + T * (vt * (2 * tg)).dot(wts), 2 * np.arctan2(tg1, 1)]
        self.inp = np.c_[vt1 * q1, 2 * dtg1 / q1]

    def predict_free(self, X, idx, tau1, T, blocks):
        """Free motion time: the instances idx (X holds their rows) integrate over their own [0, tau1],
        split at the knots below tau1; the nodes are padded with zero weights to the count of a
        whole horizon so that one omg_eval_batch launch serves the batch (last point: tau1)."""
        knots = np.unique(self.v.basis.knots)
        xg, wg = np.polynomial.legendre.leggauss(self.nq)
        nn = (len(knots) - 1) * self.nq
        pts, wts = np.zeros((len(idx), nn + 1)), np.zeros((len(idx), nn))
        for j, t1 in enumerate(tau1):
            brk = [0.] + [k for k in knots if 1e-12 < k < t1 - 1e-12] + [t1]
            nodes = np.concatenate([0.5 * (b - a) * xg + 0.5 * (a + b) for a, b in zip(brk[:-1], brk[1:])])
            pts[j, :len(nodes)], pts[j, nn] = nodes, t1
            wts[j, :len(nodes)] = np.concatenate([0.5 * (b - a) * wg for a, b in zip(brk[:-1], brk[1:])])
        out = _eval(X, blocks, pts, T, 2).reshape(-1, 2, nn + 1, 2)     # [b][column][point][derivative]
        vt, tg = out[:, 0, :nn, 0], out[:, 1, :nn, 0]
        vt1, tg1, dtg1 = out[:, 0, nn, 0], out[:, 1, nn, 0], out[:, 1, nn, 1]
        q1 = 1 + tg1**2
        st = self.state[idx]
        self.state[idx] = np.c_[st[:, 0] + T * np.einsum('bq,bq->b', vt * (1 - tg**2), wts),
                                st[:, 1] + T * np.einsum('bq,bq->b', vt * (2 * tg), wts), 2 * np.arctan2(tg1, 1)]
        self.inp[idx] = np.c_[vt1 * q1, 2 * dtg1 / q1]

    def arrived(self, state, inp, idx, tol):
        """Free-T stop test of the instances idx (dubins.py check_terminal_conditions)."""
        return _at_goal(state, inp, self.poseT[idx], tol)

    def position(self):
        return self.state[:, :2]


class _HolonomicOrientAdapter(object):
    """HolonomicOrient (holonomicorient.py): x, y and tg = tan(theta/2) are the decision splines;
    state (x, y, theta), input (x', y', theta')."""

    N_DER = 2

    def __init__(self, mpc, vehicle, batch, jitter, rng):
        self.mpc, self.v = mpc, vehicle
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.poseT = rep(vehicle.poseT)
        if jitter > 0:
            self.state[1:, :2] += rng.uniform(-jitter, jitter, (batch - 1, 2))
            self.poseT[1:, :2] += rng.uniform(-jitter, jitter, (batch - 1, 2))

    def cold_start(self, X0):
        L = len(self.v.basis)
        for k in range(2):
            X0[:, k * L:(k + 1) * L] = np.linspace(self.state[:, k], self.poseT[:, k], L).T
        X0[:, 2 * L:3 * L] = 0.

    def pack(self, P, off):
        v, st, inp = self.v.label, self.state, self.inp
        tg = np.tan(st[:, 2] / 2)
        _put(P, off, v, 'pos0', st[:, :2])
        _put(P, off, v, 'tg_ha0', tg)
        _put(P, off, v, 'vel0', inp[:, :2])
        _put(P, off, v, 'dtg_ha0', 0.5 * inp[:, 2] * (1 + tg**2))
        _put(P, off, v, 'posT', self.poseT[:, :2])
        _put(P, off, v, 'tg_haT', np.tan(self.poseT[:, 2] / 2))

    @staticmethod
    def _maps(out):
        """State and input from the values and first derivatives of x, y and tg, out [B, 6] laid out
        column / derivative (splines2signals)."""
        tg, dtg = out[:, 4], out[:, 5]
        return (np.c_[out[:, 0], out[:, 2], 2 * np.arctan2(tg, 1)],
                np.c_[out[:, 1], out[:, 3], 2 * dtg / (1 + tg**2)])

    def predict(self, X, t_rel, dt, T, device=True):
        basis = self.v.basis
        R = _rows(basis, [(t_rel + dt) / T], T, 2)
        out = _sample(X, len(basis), 3, np.vstack([R[0], R[1]]), device)   # column: value, derivative
        self.state, self.inp = self._maps(out)

    def predict_free(self, X, idx, tau1, T, blocks):
        """Free motion time: state and input of the instances idx (X holds their rows) at their own
        tau1 = min(dt, T) / T (omg_eval_batch)."""
        self.state[idx], self.inp[idx] = self._maps(_eval(X, blocks, tau1[:, None], T, 2))

    def arrived(self, state, inp, idx, tol):
        """Free-T stop test of the instances idx (holonomicorient.py check_terminal_conditions)."""
        return _at_goal(state, inp, self.poseT[idx], tol)

    def position(self):
        return self.state[:, :2]


class _QuadrotorAdapter(object):
    """Planar Quadrotor (quadrotor.py): the position splines x, y are the flat outputs; state
    (x, y, x', y', theta), input (thrust, pitch rate) and the spline derivatives dspl, ddspl of
    set_parameters follow from the derivatives up to the third (splines2signals)."""

    N_DER = 4

    def __init__(self, mpc, vehicle, batch, jitter, rng):
        self.mpc, self.v = mpc, vehicle
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.dspl, self.ddspl = rep(vehicle.prediction['dspl']), rep(vehicle.prediction['ddspl'])
        self.poseT = rep(vehicle.poseT)
        if jitter > 0:
            self.state[1:, :2] += rng.uniform(-jitter, jitter, (batch - 1, 2))
            self.poseT[1:, :2] += rng.uniform(-jitter, jitter, (batch - 1, 2))

    def cold_start(self, X0):
        L, d = len(self.v.basis), self.v.degree
        for k in range(2):
            p0, pT = self.state[:, k:k + 1], self.poseT[:, k:k + 1]
            X0[:, k * L:(k + 1) * L] = np.c_[np.repeat(p0, d, 1), np.linspace(p0[:, 0], pT[:, 0], L - 2 * d).T,
                                             np.repeat(pT, d, 1)]

    def pack(self, P, off):
        v = self.v.label
        _put(P, off, v, 'spl0', self.state[:, :2])
        _put(P, off, v, 'dspl0', self.dspl)
        _put(P, off, v, 'ddspl0', self.ddspl)
        _put(P, off, v, 'poseT', self.poseT)

    def _signals(self, X, tau1, T, device):
        """x, y and their derivatives 1..3 at tau1: [B, 2 (column), 4 (derivative)]."""
        basis = self.v.basis
        out = _sample(X, len(basis), 2, _rows(basis, [tau1], T, 4)[:, 0], device)
        return out.reshape(-1, 2, 4)

    def _maps(self, s):
        """State, input, dspl and ddspl from x, y and their derivatives 1..3, s [B, 2, 4]."""
        g = self.v.g
        (x, dx, ddx, dddx), (y, dy, ddy, dddy) = s[:, 0].T, s[:, 1].T
        return (np.c_[x, y, dx, dy, np.arctan2(ddx, ddy + g)],
                np.c_[np.sqrt(ddx**2 + (ddy + g)**2), (dddx * (ddy + g) - ddx * dddy) / ((ddy + g)**2 + ddx**2)],
                s[:, :, 1].copy(), s[:, :, 2].copy())

    def predict(self, X, t_rel, dt, T, device=True):
        self.state, self.inp, self.dspl, self.ddspl = self._maps(self._signals(X, (t_rel + dt) / T, T, device))

    def predict_planned(self, X, t_rel, dt, T, device=True):
        """The signals that the non-ideal prediction still takes from the planned trajectory
        (reference vehicle.py:326-328): dspl and ddspl at t + dt."""
        s = self._signals(X, (t_rel + dt) / T, T, device)
        self.dspl, self.ddspl = s[:, :, 1].copy(), s[:, :, 2].copy()

    def predict_free(self, X, idx, tau1, T, blocks):
        """Free motion time: state, input, dspl and ddspl of the instances idx (X holds their rows) at
        their own tau1 = min(dt, T) / T, derivatives 0..3 in one omg_eval_batch launch."""
        s = _eval(X, blocks, tau1[:, None], T, 4).reshape(-1, 2, 4)          # [b][column][derivative]
        self.state[idx], self.inp[idx], self.dspl[idx], self.ddspl[idx] = self._maps(s)

    def predict_planned_free(self, X, idx, tau1, T, blocks):
        """predict_planned with a free motion time: dspl and ddspl of the instances idx at their own tau1."""
        s = _eval(X, blocks, tau1[:, None], T, 3).reshape(-1, 2, 3)
        self.dspl[idx], self.ddspl[idx] = s[:, :, 1], s[:, :, 2]

    def arrived(self, state, inp, idx, tol):
        """Free-T stop test of the instances idx (quadrotor.py check_terminal_conditions): the position
        part of the state at the target and the planned velocity dspl at rest; the input is not read."""
        return ((np.linalg.norm(state[:, :2] - self.poseT[idx], axis=1) <= tol) &
                (np.linalg.norm(self.dspl[idx], axis=1) <= tol))

    def position(self):
        return self.state[:, :2]


class _SimpleQuadrotor3DAdapter(object):
    """SimpleQuadrotor3D (quadrotor3d_simple.py): the position splines x, y, z are the flat
    outputs; state (position, velocity, roll, pitch) and input (thrust, roll and pitch rates)
    follow from the derivatives up to the third (splines2signals)."""

    N_DER = 4

    def __init__(self, mpc, vehicle, batch, jitter, rng):
        self.mpc, self.v = mpc, vehicle
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.poseT = rep(vehicle.positionT)
        if jitter > 0:
            self.state[1:, :3] += rng.uniform(-jitter, jitter, (batch - 1, 3))
            self.poseT[1:, :3] += rng.uniform(-jitter, jitter, (batch - 1, 3))
        self.vel_plan = self.state[:, 3:6].copy()     # the planned velocity (signals['dspl']) of the free-T stop test

    def cold_start(self, X0):
        L = len(self.v.basis)
        for k in range(3):
            X0[:, k * L:(k + 1) * L] = np.linspace(self.state[:, k], self.poseT[:, k], L).T

    def pack(self, P, off):
        v, st, g = self.v.label, self.state, self.v.g
        f0, phi0, theta0 = self.inp[:, 0], st[:, 6], st[:, 7]
        _put(P, off, v, 'spl0', st[:, :3])
        _put(P, off, v, 'ddspl0', np.c_[f0 * np.cos(phi0) * np.sin(theta0), -f0 * np.sin(phi0),
                                        f0 * np.cos(phi0) * np.cos(theta0) - g])
        _put(P, off, v, 'dspl0', st[:, 3:6])
        _put(P, off, v, 'positionT', self.poseT)

    def predict(self, X, t_rel, dt, T, device=True):
        basis = self.v.basis
        s = _sample(X, len(basis), 3, _rows(basis, [(t_rel + dt) / T], T, 4)[:, 0], device).reshape(-1, 3, 4)
        self.state, self.inp = self._maps(s)

    def _maps(self, s):
        """State and input from x, y, z and their derivatives 1..3, s [B, 3, 4]."""
        g = self.v.g
        pos, vel = s[:, :, 0], s[:, :, 1]
        (ddx, ddy, ddz), (dddx, dddy, dddz) = s[:, :, 2].T, s[:, :, 3].T
        az = ddz + g
        phi = np.arctan2(-ddy, np.sqrt(ddx**2 + az**2))
        theta = np.arctan2(ddx, az)
        u1 = np.sqrt(ddx**2 + ddy**2 + az**2)
        u2 = (-dddy * (ddx**2 + az**2) + ddy * (ddx * dddx + dddz * az)) / \
            ((ddx**2 + ddy**2 + az**2) * np.sqrt(ddx**2 + az**2))
        u3 = (az * dddx - ddx * dddz) / (az**2 + ddx**2)
        return np.c_[pos, vel, phi, theta], np.c_[u1, u2, u3]

    def predict_free(self, X, idx, tau1, T, blocks):
        """Free motion time: state, input and planned velocity of the instances idx (X holds their
        rows) at their own tau1 = min(dt, T) / T, derivatives 0..3 in one omg_eval_batch launch."""
        s = _eval(X, blocks, tau1[:, None], T, 4).reshape(-1, 3, 4)          # [b][column][derivative]
        self.state[idx], self.inp[idx] = self._maps(s)
        self.vel_plan[idx] = s[:, :, 1]

    def predict_planned_free(self, X, idx, tau1, T, blocks):
        """The planned velocity (signals['dspl'], which the closed loop takes from the plan,
        vehicle.py:371-374) of the instances idx at their own tau1."""
        self.vel_plan[idx] = _eval(X, blocks, tau1[:, None], T, 2).reshape(-1, 3, 2)[:, :, 1]

    def arrived(self, state, inp, idx, tol):
        """Free-T stop test of the instances idx (quadrotor3d_simple.py check_terminal_conditions): the
        position part of the state at the target and the planned velocity (signals['dspl']) at rest."""
        return ((np.linalg.norm(state[:, :3] - self.poseT[idx], axis=1) <= tol) &
                (np.linalg.norm(self.vel_plan[idx], axis=1) <= tol))

    def position(self):
        return self.state[:, :3]


def plant_rows(basis, T, t_rel, sample_time, n_samp):
    """Basis rows R0 and derivative rows R1 (divided by T) at t_rel + s * sample_time,
    s = 0..n_samp: the samples of the stored trajectory that one update spans."""
    tau = (t_rel + sample_time * np.arange(n_samp + 1)) / T
    Bd, P1 = basis.derivative(1)
    return basis.eval_basis(tau), Bd.eval_basis(tau).dot(P1) / T


def plant_rows_der(basis, T, t_rel, sample_time, n_samp):
    """plant_rows and the rows of the second and third derivative (divided by T^2, T^3) at the
    same samples: [4, n_samp + 1, L], the layout of omg_closed_loop_step_der."""
    tau = (t_rel + sample_time * np.arange(n_samp + 1)) / T
    return np.concatenate([np.array(plant_rows(basis, T, t_rel, sample_time, n_samp)),
                           _rows(basis, tau, T, 4)[2:]])


# the adapters with a per-instance prediction for a free motion time (predict_free)
_FREE_T = ('Holonomic', 'Holonomic3D', 'Dubins', 'HolonomicOrient', 'Quadrotor', 'SimpleQuadrotor3D')

_ADAPTERS = {'Holonomic': _HolonomicAdapter, 'Holonomic3D': _HolonomicAdapter,
             'Quadrotor3D': _Quadrotor3DAdapter, 'Dubins': _DubinsAdapter,
             'HolonomicOrient': _HolonomicOrientAdapter, 'Quadrotor': _QuadrotorAdapter,
             'SimpleQuadrotor3D': _SimpleQuadrotor3DAdapter}


def _adapter_for(vehicle):
    name = type(vehicle).__name__
    if name not in _ADAPTERS:
        raise NotImplementedError('BatchMPC has no batched prediction for %s' % name)
    return _ADAPTERS[name]


# the vehicle classes BatchMPC runs several of in one problem, and the options they must share
_FLEET = ('Holonomic', 'Holonomic3D')
_FLEET_OPTIONS = ('ideal_update', 'ideal_prediction', '1storder_delay', 'time_constant', 'input_disturbance')


def _check_fleet(problem, free_T):
    """Raise NotImplementedError, naming the cause, for a multi-vehicle problem BatchMPC does not run:
    a free motion time (the Trailer's problem among them), a vehicle that is not simulated, a mixed fleet, a class other than
    Holonomic / Holonomic3D, differing spline bases or differing plant options."""
    vehicles = problem.vehicles
    if free_T:
        raise NotImplementedError('BatchMPC runs a free end time (FreeTPoint2point) for one vehicle only, '
                                  'this problem has %d' % len(vehicles))
    for v in vehicles:
        if not getattr(v, 'to_simulate', True):
            raise NotImplementedError('BatchMPC cannot run %s with several vehicles: it has to_simulate = False'
                                      % type(v).__name__)
    names = sorted(set(type(v).__name__ for v in vehicles))
    if len(names) > 1:
        raise NotImplementedError('BatchMPC runs fleets of one vehicle class only, not a mixed fleet of %s'
                                  % ', '.join(names))
    if names[0] not in _FLEET:
        raise NotImplementedError('BatchMPC runs several vehicles of class Holonomic or Holonomic3D only, not %s'
                                  % names[0])
    b0 = vehicles[0].basis
    for v in vehicles[1:]:
        if v.basis.degree != b0.degree or not np.array_equal(np.asarray(v.basis.knots), np.asarray(b0.knots)):
            raise NotImplementedError('BatchMPC runs fleets with one spline basis only: %s and %s differ in '
                                      'degree or knots' % (vehicles[0].label, v.label))
        for key in _FLEET_OPTIONS:
            a, b = vehicles[0].options.get(key), v.options.get(key)
            if repr(a) != repr(b):
                raise NotImplementedError('BatchMPC runs fleets with equal plant options only: option %r of %s '
                                          'and %s differ' % (key, vehicles[0].label, v.label))


class BatchMPC(object):

    def __init__(self, problem, batch, update_time=0.1, jitter=0.0, seed=0, device_predict=True,
                 device=None, sample_time=0.01):
        import torch
        from ..problems.point2point import FreeTPoint2point
        self.free_T = isinstance(problem, FreeTPoint2point)
        self.vehicles = problem.vehicles
        self.fleet = len(self.vehicles) > 1
        if self.fleet:
            _check_fleet(problem, self.free_T)
        if self.free_T:
            vehicle, opt = problem.vehicles[0], problem.vehicles[0].options
            if type(vehicle).__name__ not in _FREE_T:
                raise NotImplementedError('BatchMPC has no free end time (FreeTPoint2point) for %s'
                                          % type(vehicle).__name__)
            if not opt.get('ideal_update', True) and opt.get('ideal_prediction', True):
                # the ideal prediction never looks at the plant, while the stop test reads it
                raise NotImplementedError('BatchMPC runs a free end time (FreeTPoint2point) only with '
                                          'ideal_update and ideal_prediction on, or with ideal_prediction off')
        self.device_predict = device_predict
        self.torch = torch
        self.problem = problem
        self.solver = problem.problem
        self.father = problem.father
        self.tb = self.father.tables
        self.B = batch
        self.update_time = update_time
        self.vehicle = problem.vehicles[0]
        self.obstacles = problem.environment.obstacles
        if self.free_T:
            self.T = self.knot_time = None       # per instance: the variable T of every solution
        else:
            self.T = problem.options['horizon_time']
            self.knot_time = problem.knot_time
        dev = device if device is not None else torch.device('cuda', self.solver.device)
        self.dev = dev
        rng = np.random.default_rng(seed)
        n, m = self.tb.n, self.tb.m
        # per-instance scenario data (host); the vehicle-specific part lives in the adapters, one per
        # vehicle, each reading its vehicle's splines at their own column of x
        if self.fleet:
            var = self.father._var_struct.entries
            self.vehs = [_adapter_for(v)(self, v, batch, 0., rng, x_off=var[(v.label, 'splines_seg0')][0])
                         for v in self.vehicles]
            if jitter > 0:      # one shift of all starts and one of all goals: the fleet keeps its geometry
                nd = self.vehs[0].nd
                d0, dT = rng.uniform(-jitter, jitter, (batch - 1, nd)), rng.uniform(-jitter, jitter, (batch - 1, nd))
                for a in self.vehs:
                    a.state[1:] += d0
                    a.poseT[1:] += dT
        else:
            self.vehs = [_adapter_for(self.vehicle)(self, self.vehicle, batch, jitter, rng)]
        self.veh = self.vehs[0]
        self.obs = []
        for o in self.obstacles:
            d = {'x': np.repeat(o.signals['position'][:, -1][None], batch, 0).astype(float),
                 'v': np.repeat(o.signals['velocity'][:, -1][None], batch, 0).astype(float),
                 'a': np.repeat(o.signals['acceleration'][:, -1][None], batch, 0).astype(float)}
            if 'theta' in o._parameters:
                d['theta'] = np.repeat(o.signals['orientation'][:, -1][None], batch, 0).astype(float)
                d['omega'] = float(o.signals['angular_velocity'][:, -1][0])
            self.obs.append(d)
        # parameter template and entry offsets
        self.P = np.repeat(self.father.set_parameters(0.).cat[None], batch, 0)
        ent = self.father._par_struct.entries
        self.off = {key: ent[key][0] for key in ent}
        # cold start per instance (holonomic.py:118-127, quadrotor3d.py:189-201)
        X0 = np.repeat(self.father.get_variables().cat[None], batch, 0)
        for a in self.vehs:
            a.cold_start(X0)
        self.X = torch.tensor(X0, device=dev)
        self.Xn = torch.empty_like(self.X)
        self.LAM = torch.empty((batch, m), dtype=torch.float64, device=dev)
        self.F = torch.empty(batch, dtype=torch.float64, device=dev)
        self.ST = torch.empty(batch, dtype=torch.int32, device=dev)
        self.IT = torch.empty(batch, dtype=torch.int32, device=dev)
        self.LB = torch.tensor(self.tb.lbg, device=dev)
        self.UB = torch.tensor(self.tb.ubg, device=dev)
        self.Pd = torch.empty((batch, self.tb.n_par), dtype=torch.float64, device=dev)
        self.blocks = [(off, shape[0], shape[1], T) for (_, _, off, shape, T)
                       in self.father.shifted_entries()]
        self.time = 0.
        self.time_prev = 0.
        self.history = {'state': [self.state.copy()], 'iters': [], 'status': []}
        self.sample_time = sample_time
        opt = self.vehicle.options
        self.ideal_update = opt.get('ideal_update', True)
        self.ideal_prediction = opt.get('ideal_prediction', True)
        self.closed_loop = not (self.ideal_update and self.ideal_prediction)
        if self.closed_loop:
            self._init_plant(opt, seed)
        if self.free_T:
            self._init_free_T()

    def _init_free_T(self):
        """Free motion time: the spline blocks of the warm start and of the prediction, the index of
        T in x, and which instances still run (history['active'][k]: solved at step k)."""
        from ..solver.b200 import spline_blocks
        self.t_index = self.father._var_struct.entries[(self.problem.label, 'T')][0]
        self.shift_blocks = spline_blocks(self.father)
        self.veh_blocks = spline_blocks(self.father, self.vehicle)
        self.active = np.ones(self.B, dtype=bool)
        self.n_solved = 0
        self.history.update({'T': [], 'active': []})

    def _init_plant(self, opt, seed):
        """Plant state and last applied input per instance (device tensors), the lag and the
        disturbance of the vehicle's options, and the filter's scratch.  With ideal_update on the
        plant follows the spline and the reference applies neither (vehicle.py:366-370)."""
        from ..solver.b200 import ODE_MODELS, disturbance_filter
        torch = self.torch
        sample_time = self.sample_time
        self.seed, self.k = seed, 0
        self.model = ODE_MODELS[type(self.vehicle).__name__]
        self.plant_x = torch.tensor(self.state, device=self.dev)      # ([B, n_veh, n] for a fleet)
        self.plant_u = torch.tensor(self.inp, device=self.dev)
        self.pred_x, self.pred_u = torch.empty_like(self.plant_x), torch.empty_like(self.plant_u)
        lag = opt.get('1storder_delay', False) and not self.ideal_update
        self.time_constant = float(opt['time_constant']) if lag else None
        self.disturbance = None
        dist = opt.get('input_disturbance')
        if dist and not self.ideal_update:
            ni = self.plant_u.shape[-1]
            stdev = np.broadcast_to(np.asarray(dist['stdev'], dtype=float), (ni,))
            mean = np.broadcast_to(np.asarray(dist.get('mean', np.zeros(ni)), dtype=float), (ni,))
            # (a free motion time grows the scratch with the longest trajectory of a step)
            n_traj = int(np.round(self.T / sample_time, 6)) + 1 if self.T is not None else 0
            scratch = torch.empty(self.B * len(self.vehs) * ni * (n_traj + 24), dtype=torch.float64,
                                  device=self.dev)
            self.disturbance = (disturbance_filter(dist['fc']), mean, stdev, scratch)
        self.history['plant'] = [self.plant_x.cpu().numpy().copy()]
        self.history['plant_input'] = [self.plant_u.cpu().numpy().copy()]

    # state / input / target of every instance (owned by the vehicle adapters): [B, n] for one
    # vehicle, [B, n_veh, n] for a fleet
    def _stacked(self, key):
        if self.fleet:
            return np.stack([getattr(a, key) for a in self.vehs], axis=1)
        return getattr(self.veh, key)

    state = property(lambda self: self._stacked('state'))
    inp = property(lambda self: self._stacked('inp'))
    poseT = property(lambda self: self._stacked('poseT'))

    # ------------------------------------------------------------------
    def _pack_parameters(self, t):
        P, off = self.P, self.off
        for a in self.vehs:
            a.pack(P, off)
        for o, d in zip(self.obstacles, self.obs):
            nd = o.n_dim
            for key in ('x', 'v', 'a'):
                P[:, off[(o.label, key)]:off[(o.label, key)] + nd] = d[key]
            if 'theta' in d:
                P[:, off[(o.label, 'theta')]] = d['theta'][:, 0]
        if self.free_T:                 # the time axis restarts every update (point2point.py:300-306)
            P[:, off[(self.problem.label, 't')]] = 0.
            return
        P[:, off[(self.problem.label, 't')]] = np.round(t, 6) % self.knot_time
        P[:, off[(self.problem.label, 'T')]] = self.T

    def _advance_obstacles(self, dt, sample_time):
        """Obstacle motion over one update, sample by sample as the reference's
        simulator does it (obstacle.py:229-247): constant-acceleration steps plus the
        increments of the obstacle's 'trajectories' at their switching times."""
        n_samp = int(np.round(dt / sample_time, 6))
        for o, d in zip(self.obstacles, self.obs):
            inc = getattr(o, '_increments', [])
            for _ in range(n_samp):
                t0 = d.setdefault('time', 0.)
                t1 = t0 + sample_time
                d['x'] = d['x'] + sample_time * d['v'] + 0.5 * sample_time**2 * d['a']
                d['v'] = d['v'] + sample_time * d['a']
                for tm, l, val in inc:
                    if t0 + 1e-9 < tm <= t1 + 1e-9:      # (sample times accumulate rounding)
                        key = ('x', 'v', 'a')[l]
                        d[key] = d[key] + val
                d['time'] = t1
            if 'theta' in d:
                d['theta'] = d['theta'] + dt * d['omega']

    # ------------------------------------------------------------------
    def step(self):
        if self.free_T:
            return self._step_free_T()
        torch = self.torch
        t = self.time
        # knot crossing -> shift the warm start on the device
        if int(np.round(self.time_prev / self.knot_time, 6)) < int(np.round(t / self.knot_time, 6)):
            self.solver.shift_batch_device(self.X, self.blocks)
        self.time_prev = t
        self._pack_parameters(t)
        self.Pd.copy_(torch.from_numpy(self.P))
        self.solver.solve_batch_device(self.X, self.Pd, self.LB, self.UB, self.Xn,
                                       self.LAM, self.F, self.ST, self.IT)
        self.X, self.Xn = self.Xn, self.X
        self.history['iters'].append(self.IT.cpu().numpy().copy())
        self.history['status'].append(self.ST.cpu().numpy().copy())
        # ideal update: vehicle and obstacles move over update_time; the prediction at
        # t + update_time comes from spline values sampled on the device
        t_rel = np.round(t, 6) % self.knot_time
        if self.closed_loop:
            self._plant_step(t_rel)
        else:
            for a in self.vehs:
                a.predict(self.X, t_rel, self.update_time, self.T, device=self.device_predict)
        self._advance_obstacles(self.update_time, self.sample_time)
        self.history['state'].append(self.state.copy())
        self.time = np.round(t + self.update_time, 6)

    def _plant_step(self, t_rel):
        """Reference Vehicle.simulate and predict (vehicle.py:302-337, 359-392) of every instance
        in one launch; the ideal half of a mixed setting follows the spline as before."""
        from ..solver.b200 import closed_loop_step, closed_loop_step_fleet
        n_samp = int(np.round(self.update_time / self.sample_time, 6))
        higher = None
        if self.fleet:
            R = plant_rows_der(self.vehicle.basis, self.T, t_rel, self.sample_time, n_samp)[:self.veh.N_DER]
        elif self.veh.N_DER > 2:
            R = plant_rows_der(self.vehicle.basis, self.T, t_rel, self.sample_time, n_samp)
            R0, R1, higher = R[0], R[1], R[2:self.veh.N_DER]
        else:
            R0, R1 = plant_rows(self.vehicle.basis, self.T, t_rel, self.sample_time, n_samp)
        dist = None
        if self.disturbance is not None:
            filt, mean, stdev, scratch = self.disturbance
            n_traj = int(np.round((self.T - t_rel) / self.sample_time, 6)) + 1
            dist = (filt, mean, stdev, n_traj, scratch)
        out = (self.plant_x, self.plant_u, self.pred_x, self.pred_u)
        if self.fleet:          # one launch for every (instance, vehicle)
            closed_loop_step_fleet(self.model, self.X, [a.x_off for a in self.vehs], len(self.vehicle.basis), R,
                                   self.sample_time, self.plant_x, self.plant_u, out, self.k, seed=self.seed,
                                   time_constant=self.time_constant, disturbance=dist)
        else:
            closed_loop_step(self.model, self.X, len(self.vehicle.basis), R0, R1, self.sample_time,
                             self.plant_x, self.plant_u, out, self.k, seed=self.seed,
                             time_constant=self.time_constant, disturbance=dist, higher=higher)
        self.k += 1
        if self.ideal_prediction or self.ideal_update:
            for a in self.vehs:
                a.predict(self.X, t_rel, self.update_time, self.T, device=self.device_predict)
        elif hasattr(self.veh, 'predict_planned'):
            # signals other than state and input come from the planned trajectory (vehicle.py:326-328)
            self.veh.predict_planned(self.X, t_rel, self.update_time, self.T, device=self.device_predict)
        if self.ideal_update:
            self.plant_x.copy_(self.torch.from_numpy(self.state))
            self.plant_u.copy_(self.torch.from_numpy(self.inp))
        if not self.ideal_prediction:
            # (copies: the adapter updates its arrays in place, and on a CPU device .numpy()
            # would share the kernel's output buffers)
            px, pu = self.pred_x.cpu().numpy(), self.pred_u.cpu().numpy()
            if self.fleet:
                for v, a in enumerate(self.vehs):
                    a.state, a.inp = px[:, v].copy(), pu[:, v].copy()
            else:
                self.veh.state, self.veh.inp = px.copy(), pu.copy()
        self.history['plant'].append(self.plant_x.cpu().numpy().copy())
        self.history['plant_input'].append(self.plant_u.cpu().numpy().copy())

    def _step_free_T(self):
        """One update of the reference's free-T loop for every active instance (Simulator.update /
        Deployer.update with FreeTPoint2point, point2point.py:300-374): warm start by shift_spline
        from the instance's own T (omg_shift_free_batch; not on the first step), solve the active
        instances, predict at tau = min(dt, T) / T (omg_eval_batch), move the obstacles, and stop
        the instances with T < dt or at their goal (check_terminal_conditions).  A stopped instance
        is not solved again and its X, state and T stay as they are; status -1 and 0 iterations
        stand for 'not solved' in the history."""
        torch = self.torch
        act = np.nonzero(self.active)[0]
        if len(act) == 0:
            return
        dt = self.update_time
        if self.n_solved > 0:
            mask = torch.tensor(self.active.astype(np.int32), device=self.dev)
            self.solver.shift_free_batch_device(self.X, self.shift_blocks, self.t_index, dt, active=mask)
        self._pack_parameters(0.)
        idx = torch.from_numpy(act).to(self.dev)
        Xa = self.X.index_select(0, idx)
        Pa = torch.from_numpy(self.P[act]).to(self.dev)
        na, m = len(act), self.tb.m
        Xn = torch.empty_like(Xa)
        LAM = torch.empty((na, m), dtype=torch.float64, device=self.dev)
        F = torch.empty(na, dtype=torch.float64, device=self.dev)
        ST = torch.empty(na, dtype=torch.int32, device=self.dev)
        IT = torch.empty(na, dtype=torch.int32, device=self.dev)
        self.solver.solve_batch_device(Xa, Pa, self.LB, self.UB, Xn, LAM, F, ST, IT)
        self.X.index_copy_(0, idx, Xn)
        self.n_solved += 1
        status, iters = np.full(self.B, -1, dtype=np.int32), np.zeros(self.B, dtype=np.int32)
        status[act], iters[act] = ST.cpu().numpy(), IT.cpu().numpy()
        self.history['status'].append(status)
        self.history['iters'].append(iters)
        self.history['active'].append(self.active.copy())
        T = Xn[:, self.t_index].cpu().numpy()
        self.history['T'].append(self.X[:, self.t_index].cpu().numpy().copy())
        # the last update of an instance moves it by min(dt, T), and not at all when T is below the
        # sample time (FreeTPoint2point.simulate, store)
        move = T >= self.sample_time
        if self.closed_loop:
            self._plant_step_free(act, move, T)
        if move.any():
            sel = torch.from_numpy(np.nonzero(move)[0]).to(self.dev)
            args = (Xn.index_select(0, sel) if not move.all() else Xn, act[move],
                    np.minimum(dt, T[move]) / T[move], T[move], self.veh_blocks)
            if not self.closed_loop or self.ideal_update:
                self.veh.predict_free(*args)
            elif hasattr(self.veh, 'predict_planned_free'):
                # signals other than state and input come from the plan (vehicle.py:326-328, 371-374)
                self.veh.predict_planned_free(*args)
        if self.closed_loop:
            moved = act[move]
            if self.ideal_update and len(moved):
                sel = torch.from_numpy(moved).to(self.dev)
                self.plant_x.index_copy_(0, sel, torch.from_numpy(self.state[moved]).to(self.dev))
                self.plant_u.index_copy_(0, sel, torch.from_numpy(self.inp[moved]).to(self.dev))
            # (ideal_prediction is off: state0 of the next solve is the kernel's prediction)
            self.veh.state[moved] = self.pred_x.cpu().numpy()[moved]
            self.veh.inp[moved] = self.pred_u.cpu().numpy()[moved]
            px, pu = self.plant_x.cpu().numpy().copy(), self.plant_u.cpu().numpy().copy()
            self.history['plant'].append(px)
            self.history['plant_input'].append(pu)
            # the reference's check_terminal_conditions reads the plant (signals)
            state, inp = px[act], pu[act]
        else:
            state, inp = self.state[act], self.inp[act]
        self._advance_obstacles(dt, self.sample_time)
        self.history['state'].append(self.state.copy())
        self.time = np.round(self.time + dt, 6)
        arrived = self.veh.arrived(state, inp, act, self.vehicle.options['stop_tol'])
        self.active[act[(T < dt) | arrived]] = False

    def _plant_step_free(self, act, move, T):
        """Reference Vehicle.simulate and predict of every instance that moves in this update
        (FreeTPoint2point.store / simulate) in one launch on the whole batch [omg_closed_loop_step_free]:
        instance b samples its plan on its own time axis for min(dt, T_b) / sample_time samples and
        filters its disturbance over its own stored trajectory, T_b / sample_time + 1 samples.  An
        instance that is stopped or whose T is below the sample time is not touched.  The one
        deviation from the reference: a final update with T_b / sample_time + 1 <= 12 samples (T below
        0.12 s at 0.01 s samples), where the reference's filtfilt would raise, gets no disturbance."""
        from ..solver.b200 import closed_loop_step_free
        st, dt = self.sample_time, self.update_time
        n_samp, n_traj = np.zeros(self.B, dtype=np.int32), np.zeros(self.B, dtype=np.int32)
        Tm, am = T[move], act[move]
        n_samp[am] = np.round(np.minimum(dt, Tm) / st, 6).astype(np.int32)
        n_traj[am] = np.round(Tm / st, 6).astype(np.int32) + 1
        n_traj[n_traj <= 12] = 0
        dist = None
        if self.disturbance is not None:
            filt, mean, stdev, scratch = self.disturbance
            need = self.B * self.plant_u.shape[1] * (int(n_traj.max()) + 24)
            if scratch.numel() < need:
                scratch = self.torch.empty(need, dtype=self.torch.float64, device=self.dev)
                self.disturbance = (filt, mean, stdev, scratch)
            dist = (filt, mean, stdev, n_traj, scratch)
        closed_loop_step_free(self.model, self.X, self.veh_blocks[0], self.t_index, self.veh.N_DER, n_samp, st,
                              self.plant_x, self.plant_u, (self.plant_x, self.plant_u, self.pred_x, self.pred_u),
                              self.k, seed=self.seed, time_constant=self.time_constant, disturbance=dist)
        self.k += 1

    def run(self, n_steps):
        """n_steps MPC updates; with a free end time the run ends early once every instance stopped."""
        for _ in range(n_steps):
            if self.free_T and not self.active.any():
                break
            self.step()
        return self.history
