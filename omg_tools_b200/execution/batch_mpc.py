"""Batched receding-horizon driver: B independent copies of one Point2point
scenario (Holonomic, Holonomic3D or Quadrotor3D vehicle) advance in lock step,
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
batch size.  history['plant'] and history['plant_input'] hold the plant state and the last
applied input at every update boundary.  ``sample_time`` is the simulation grid of the plant
and of the obstacle motion (the reference simulator's sample_time, 0.01 s by default).
"""
import numpy as np


class _HolonomicAdapter(object):
    """Holonomic / Holonomic3D: state = position spline value, input = its
    derivative / T (holonomic.py:87-105, 153-159)."""

    def __init__(self, mpc, vehicle, batch, jitter, rng):
        self.mpc, self.v = mpc, vehicle
        self.nd = nd = vehicle.n_dim
        rep = lambda a: np.repeat(np.asarray(a, float)[None], batch, 0)
        self.state, self.inp = rep(vehicle.prediction['state']), rep(vehicle.prediction['input'])
        self.poseT = rep(vehicle.poseT)
        if jitter > 0:
            self.state[1:] += rng.uniform(-jitter, jitter, (batch - 1, nd))
            self.poseT[1:] += rng.uniform(-jitter, jitter, (batch - 1, nd))

    def cold_start(self, X0):
        L = len(self.v.basis)
        for k in range(self.nd):
            X0[:, k * L:(k + 1) * L] = np.linspace(self.state[:, k], self.poseT[:, k], L).T

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
            out = sample_batch(X, [(0, L, nd, np.vstack([B0, B1]))]).cpu().numpy()
            # layout: [column][sample] with samples (value, derivative)
            for k in range(nd):
                self.state[:, k], self.inp[:, k] = out[:, 2 * k], out[:, 2 * k + 1]
        else:
            Xh = X.cpu().numpy()
            for k in range(nd):
                c = Xh[:, k * L:(k + 1) * L]
                self.state[:, k] = c.dot(B0[0])
                self.inp[:, k] = c.dot(B1[0])

    def position(self):
        return self.state


class _Quadrotor3DAdapter(object):
    """Quadrotor3D (quadrotor3d.py): the decision splines are the flat outputs
    f~, q_phi, q_theta; position and velocity follow from the double integral of
    the accelerations re-anchored at the previous prediction (splines2signals,
    quadrotor3d.py:253-275).  The integral over one update is taken exactly by
    Gauss-Legendre quadrature per knot piece on device-sampled spline values."""

    NQ = 6      # exact for the degree-9 integrand (tau1 - s) * ddx(s)

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


def plant_rows(basis, T, t_rel, sample_time, n_samp):
    """Basis rows R0 and derivative rows R1 (divided by T) at t_rel + s * sample_time,
    s = 0..n_samp: the samples of the stored trajectory that one update spans."""
    tau = (t_rel + sample_time * np.arange(n_samp + 1)) / T
    Bd, P1 = basis.derivative(1)
    return basis.eval_basis(tau), Bd.eval_basis(tau).dot(P1) / T


def _adapter_for(vehicle):
    name = type(vehicle).__name__
    if name in ('Holonomic', 'Holonomic3D'):
        return _HolonomicAdapter
    if name == 'Quadrotor3D':
        return _Quadrotor3DAdapter
    raise NotImplementedError('BatchMPC has no batched prediction for %s' % name)


class BatchMPC(object):

    def __init__(self, problem, batch, update_time=0.1, jitter=0.0, seed=0, device_predict=True,
                 device=None, sample_time=0.01):
        import torch
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
        self.T = problem.options['horizon_time']
        self.knot_time = problem.knot_time
        dev = device if device is not None else torch.device('cuda', self.solver.device)
        self.dev = dev
        rng = np.random.default_rng(seed)
        n, m = self.tb.n, self.tb.m
        # per-instance scenario data (host); the vehicle-specific part lives in the adapter
        self.veh = _adapter_for(self.vehicle)(self, self.vehicle, batch, jitter, rng)
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
        self.veh.cold_start(X0)
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

    def _init_plant(self, opt, seed):
        """Plant state and last applied input per instance (device tensors), the lag and the
        disturbance of the vehicle's options, and the filter's scratch.  With ideal_update on the
        plant follows the spline and the reference applies neither (vehicle.py:366-370)."""
        from ..solver.b200 import ODE_MODELS, disturbance_filter
        torch = self.torch
        sample_time = self.sample_time
        self.seed, self.k = seed, 0
        self.model = ODE_MODELS[type(self.vehicle).__name__]
        self.plant_x = torch.tensor(self.state, device=self.dev)
        self.plant_u = torch.tensor(self.inp, device=self.dev)
        self.pred_x, self.pred_u = torch.empty_like(self.plant_x), torch.empty_like(self.plant_u)
        lag = opt.get('1storder_delay', False) and not self.ideal_update
        self.time_constant = float(opt['time_constant']) if lag else None
        self.disturbance = None
        dist = opt.get('input_disturbance')
        if dist and not self.ideal_update:
            ni = self.plant_u.shape[1]
            stdev = np.broadcast_to(np.asarray(dist['stdev'], dtype=float), (ni,))
            mean = np.broadcast_to(np.asarray(dist.get('mean', np.zeros(ni)), dtype=float), (ni,))
            n_traj = int(np.round(self.T / sample_time, 6)) + 1
            scratch = torch.empty(self.B * ni * (n_traj + 24), dtype=torch.float64, device=self.dev)
            self.disturbance = (disturbance_filter(dist['fc']), mean, stdev, scratch)
        self.history['plant'] = [self.plant_x.cpu().numpy().copy()]
        self.history['plant_input'] = [self.plant_u.cpu().numpy().copy()]

    # state / input / target of every instance (owned by the vehicle adapter)
    state = property(lambda self: self.veh.state)
    inp = property(lambda self: self.veh.inp)
    poseT = property(lambda self: self.veh.poseT)

    # ------------------------------------------------------------------
    def _pack_parameters(self, t):
        P, off = self.P, self.off
        self.veh.pack(P, off)
        for o, d in zip(self.obstacles, self.obs):
            nd = o.n_dim
            for key in ('x', 'v', 'a'):
                P[:, off[(o.label, key)]:off[(o.label, key)] + nd] = d[key]
            if 'theta' in d:
                P[:, off[(o.label, 'theta')]] = d['theta'][:, 0]
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
            self.veh.predict(self.X, t_rel, self.update_time, self.T, device=self.device_predict)
        self._advance_obstacles(self.update_time, self.sample_time)
        self.history['state'].append(self.state.copy())
        self.time = np.round(t + self.update_time, 6)

    def _plant_step(self, t_rel):
        """Reference Vehicle.simulate and predict (vehicle.py:302-337, 359-392) of every instance
        in one launch; the ideal half of a mixed setting follows the spline as before."""
        from ..solver.b200 import closed_loop_step
        n_samp = int(np.round(self.update_time / self.sample_time, 6))
        R0, R1 = plant_rows(self.vehicle.basis, self.T, t_rel, self.sample_time, n_samp)
        dist = None
        if self.disturbance is not None:
            filt, mean, stdev, scratch = self.disturbance
            n_traj = int(np.round((self.T - t_rel) / self.sample_time, 6)) + 1
            dist = (filt, mean, stdev, n_traj, scratch)
        closed_loop_step(self.model, self.X, len(self.vehicle.basis), R0, R1, self.sample_time,
                         self.plant_x, self.plant_u,
                         (self.plant_x, self.plant_u, self.pred_x, self.pred_u), self.k, seed=self.seed,
                         time_constant=self.time_constant, disturbance=dist)
        self.k += 1
        if self.ideal_prediction or self.ideal_update:
            self.veh.predict(self.X, t_rel, self.update_time, self.T, device=self.device_predict)
        if self.ideal_update:
            self.plant_x.copy_(self.torch.from_numpy(self.state))
            self.plant_u.copy_(self.torch.from_numpy(self.inp))
        if not self.ideal_prediction:
            # (copies: the adapter updates its arrays in place, and on a CPU device .numpy()
            # would share the kernel's output buffers)
            self.veh.state = self.pred_x.cpu().numpy().copy()
            self.veh.inp = self.pred_u.cpu().numpy().copy()
        self.history['plant'].append(self.plant_x.cpu().numpy().copy())
        self.history['plant_input'].append(self.plant_u.cpu().numpy().copy())

    def run(self, n_steps):
        for _ in range(n_steps):
            self.step()
        return self.history
