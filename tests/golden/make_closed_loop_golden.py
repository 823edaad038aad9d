"""Generate tests/golden/closed_loop_golden.npz: the REFERENCE's receding-horizon loop with its
own vehicle options, i.e. without forcing ideal_prediction / ideal_update on.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_closed_loop_golden.py

The loop and the stand-ins are make_loop_golden.py's (the solver is this repository's CPU
oracle on the lowered tables).  Left at the reference's defaults (vehicle.py:70-75),
``Vehicle.predict`` integrates the planned inputs of the previous step from the plant state of
that step (odeint, interp1d), and ``Vehicle.simulate`` integrates the vehicle ODE from the
plant state over one update.  Stored per MPC step: x0, p, lbg, ubg, x, status (what the
reference hands to the solver and unpacks), and the plant state and input at every update
boundary (``signals['state'|'input']`` every n_samp samples).

    config1   examples/p2p_holonomic.py as written: ideal_prediction False, ideal_update
              default False; 12 x 0.1 s, through the knot crossing at t = 1
    config5   revolving door, defaults; 12 x 0.1 s
    config4   3-D quadrotor, defaults; 0.4 s steps up to the first knot crossing (the loops
              part there for the slack shift, tests/test_model.py)
    config_disturbances
              examples/p2p_holonomic_disturbances.py as written: first-order lag (tau 0.1),
              input disturbance fc 0.01, stdev 0.05; 12 x 0.1 s.  ``normal`` of the reference's
              vehicle module is replaced by the numpy twin of the device generator
              (tests/plant_twin.py), keyed as instance 0 with seed 0: the reference's own
              butter, filtfilt, interp1d and odeint then run on exactly the white noise the
              kernel draws.  The reference builder of this scenario is written below (same
              values as scenarios.config_disturbances).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_loop_golden as lg                           # noqa: E402
import make_model_golden as mg                          # noqa: E402
import plant_twin as tw                                 # noqa: E402

OUT = os.path.join(HERE, 'closed_loop_golden.npz')


class RecordingSolver(lg.OracleSolver):
    """make_loop_golden's solver object, recording the iteration count of every call too."""

    def __call__(self, x0, p, lbg, ubg, **kw):
        r = lg.OracleSolver.__call__(self, x0, p, lbg, ubg, **kw)
        self.iters = getattr(self, 'iters', []) + [int(self.last['iters'][0])]
        return r


def build_reference_disturbances():
    """examples/p2p_holonomic_disturbances.py against the reference's API."""
    hol, env = mg.ref_import('vehicles.holonomic'), mg.ref_import('environment.environment')
    obs, shp = mg.ref_import('environment.obstacle'), mg.ref_import('basics.shape')
    p2p = mg.ref_import('problems.point2point')
    vehicle = hol.Holonomic()
    vehicle.set_options({'safety_distance': 0.1})
    vehicle.set_options({'1storder_delay': True, 'time_constant': 0.1})
    vehicle.set_options({'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}})
    vehicle.set_options({'stop_tol': 1.e-2})
    vehicle.set_initial_conditions([-1.5, -1.5])
    vehicle.set_terminal_conditions([2., 2.])
    environment = env.Environment(room={'shape': shp.Square(5.)})
    rectangle = shp.Rectangle(width=3., height=0.2)
    environment.add_obstacle(obs.Obstacle({'position': [-2.1, -0.5]}, shape=rectangle))
    environment.add_obstacle(obs.Obstacle({'position': [1.7, -0.5]}, shape=rectangle))
    trajectories = {'velocity': {'time': [3., 4.], 'values': [[-0.15, 0.0], [0., 0.15]]}}
    environment.add_obstacle(obs.Obstacle({'position': [1.5, 0.5]}, shape=shp.Circle(0.4),
                                          simulation={'trajectories': trajectories}))
    problem = p2p.Point2point(vehicle, environment, options={'verbose': 0}, freeT=False)
    problem.father.reset()
    problem.construct()
    return problem


def install_twin_normal(n_sig, seed=0, instance=0):
    """normal(mean, stdev, n) of the reference's vehicle module -> the device generator's draws:
    add_disturbance calls it once per signal and MPC step, in that order."""
    veh = mg.ref_import('vehicles.vehicle')
    calls = [0]

    def normal(mean, stdev, n):
        step, sig = divmod(calls[0], n_sig)
        calls[0] += 1
        return mean + stdev * tw.normals(seed, step, instance, sig, n)
    veh.normal = normal


def run_closed_loop(name, n_steps, update_time, sample_time=0.01, vehicle_options=None):
    from omg_tools_b200 import scenarios as sc
    tables = getattr(sc, name)(build_solver=False).father.tables
    opt = mg.ref_import('basics.optilayer')
    for cls in list(opt.OptiChild.__subclasses__()) + [opt.OptiChild]:
        if hasattr(cls, '_labels'):
            cls._labels = []
    mg.REG = mg.Registry(seed=3)
    if name == 'config_disturbances':
        problem = build_reference_disturbances()
        install_twin_normal(2)
    else:
        problem = mg.build_reference(name)
    vehicle = problem.vehicles[0]
    vehicle.set_options(vehicle_options or {})
    vehicle.problem = problem
    solver = RecordingSolver(tables)
    problem.problem, _ = problem.father.construct_problem(problem.options, problem=solver)
    problem.father.init_transformations(problem.init_primal_transform,
                                        problem.init_dual_transform)
    problem.reinitialize()
    t = 0.
    for k in range(n_steps):
        if k == 0:
            problem.initialize(t)
        problem.predict(t, update_time, sample_time, None, None, None, 0, False, False)
        problem.solve(t, update_time)
        problem.store(t, update_time, sample_time)
        problem.simulate(t, update_time, sample_time)
        t = np.round(t + update_time, 6)
    n_samp = int(np.round(update_time / sample_time, 6))
    calls = solver.calls
    st, inp = (np.asarray(vehicle.signals[key], float) for key in ('state', 'input'))
    return {'x0': np.array([c[0] for c in calls]), 'p': np.array([c[1] for c in calls]),
            'lbg': np.array([c[2] for c in calls]), 'ubg': np.array([c[3] for c in calls]),
            'x': np.array([c[4] for c in calls]), 'status': np.array([c[5] for c in calls]),
            'iters': np.array(solver.iters), 'plant_state': st[:, ::n_samp].T, 'plant_input': inp[:, ::n_samp].T,
            'options': np.array([vehicle.options['ideal_prediction'], vehicle.options['ideal_update']])}


def main():
    mg.install_stubs()
    lg.install_struct_stubs()
    out = {}
    runs = (('config1', 12, 0.1, {'ideal_prediction': False}),
            ('config5', 12, 0.1, None),
            ('config4', 3, 0.4, None),
            ('config_disturbances', 12, 0.1, None))
    for name, n_steps, dt, vopt in runs:
        res = run_closed_loop(name, n_steps, dt, vehicle_options=vopt)
        print(name, 'status', res['status'], 'final plant state', np.round(res['plant_state'][-1], 4))
        for key, val in res.items():
            out['%s_%s' % (name, key)] = val
        out[name + '_dt'] = dt
    np.savez_compressed(OUT, **out)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
