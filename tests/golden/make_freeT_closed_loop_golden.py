"""Generate tests/golden/freeT_closed_loop_golden.npz: the REFERENCE's receding-horizon loop with a free
motion time and its own vehicle options, i.e. closed through the vehicle's dynamics.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_freeT_closed_loop_golden.py

The loop is make_freeT_loop_golden.py's (predict; solve with init_step; store; simulate by
min(update_time, T); stop_criterium) on the same stand-ins and the same solver call (this
repository's CPU oracle, the reference's unset T parameter dropped from p), but the vehicle options
are left at the reference's values (vehicle.py:70-75: ideal_prediction and ideal_update off), so
``Vehicle.predict`` integrates the previous plan from the plant state and ``Vehicle.simulate``
integrates the vehicle ODE over each update.

    config_freeT_moving   the moving-obstacle minimum-time variant of examples/p2p_holonomic.py,
                          which sets ideal_prediction False
    config_dubins_freeT   examples/p2p_dubins.py as written
    config_freeT_disturbed
                          config_freeT with the first-order lag (time constant 0.1) and the input
                          disturbance (fc 0.01, stdev 0.05); ``normal`` of the reference's vehicle
                          module is replaced by the numpy twin of the device generator
                          (make_closed_loop_golden.install_twin_normal, instance 0, seed 0)

The Deployer lowers the update time when less than one update of trajectory is left
(deployer.py:47-55).  With a free motion time that happens only after an update shorter than
update_time, i.e. after an update with T < update_time, after which the loop stops; the script
asserts that it is not reached before the stop.

Stored per configuration and MPC step: x0, p, the solution x, the status, the iteration count and
T; the plant state and input at every update boundary (``signals['state'|'input'][:, -1]`` after
each simulate, the initial ones first); and the update time.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_model_golden as mg                          # noqa: E402
import make_loop_golden as lg                           # noqa: E402
import make_freeT_loop_golden as fg                     # noqa: E402
import make_closed_loop_golden as cg                    # noqa: E402

OUT = os.path.join(HERE, 'freeT_closed_loop_golden.npz')
DISTURBED = {'1storder_delay': True, 'time_constant': 0.1,
             'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}}
RUNS = (('config_freeT_moving', 'config_freeT_moving', {'ideal_prediction': False}),
        ('config_dubins_freeT', 'config_dubins_freeT', None),
        ('config_freeT_disturbed', 'config_freeT', DISTURBED))


def run_reference_freeT_closed_loop(scenario, update_time, vehicle_options=None, max_steps=60, sample_time=0.01):
    from omg_tools_b200 import scenarios as sc
    tables = getattr(sc, scenario)(build_solver=False).father.tables
    opt = mg.ref_import('basics.optilayer')
    for cls in list(opt.OptiChild.__subclasses__()) + [opt.OptiChild]:
        if hasattr(cls, '_labels'):
            cls._labels = []
    mg.REG = mg.Registry(seed=3)
    problem = mg.build_reference(scenario)
    vehicle = problem.vehicles[0]
    vehicle.set_options(vehicle_options or {})
    vehicle.problem = problem
    if (vehicle_options or {}).get('input_disturbance'):
        cg.install_twin_normal(2)
    solver = fg.FreeTOracle(tables, None)
    problem.problem, _ = problem.father.construct_problem(problem.options, problem=solver)
    par = problem.father._par_struct
    solver.t_par = par.locate((problem.label, 'T'))[0]
    problem.father.init_transformations(problem.init_primal_transform, problem.init_dual_transform)
    problem.reinitialize()
    t, Ts, iters = 0., [], []
    plant_x, plant_u = [], []
    for k in range(max_steps):
        if k == 0:
            problem.initialize(t)
        problem.predict(t, update_time, sample_time, None, None, None, 0, False, False)
        problem.solve(t, update_time)
        Ts.append(float(np.asarray(problem.father.get_variables(problem, 'T')).reshape(-1)[0]))
        iters.append(int(solver.last['iters'][0]))
        problem.store(t, update_time, sample_time)
        problem.simulate(t, update_time, sample_time)
        if k == 0:
            plant_x.append(np.asarray(vehicle.signals['state'], float)[:, 0])
            plant_u.append(np.asarray(vehicle.signals['input'], float)[:, 0])
        plant_x.append(np.asarray(vehicle.signals['state'], float)[:, -1])
        plant_u.append(np.asarray(vehicle.signals['input'], float)[:, -1])
        simulated = float(vehicle.signals['time'][0, -1]) - t
        t = np.round(t + update_time, 6)
        if problem.stop_criterium(t, update_time):
            break
        # the Deployer would lower the next update time here (deployer.py:49-50)
        assert round(update_time - simulated, 4) < sample_time, (scenario, k, simulated)
    else:
        raise RuntimeError('%s did not stop within %d steps' % (scenario, max_steps))
    calls = solver.calls
    return {'x0': np.array([c[0] for c in calls]), 'p': np.array([c[1] for c in calls]),
            'x': np.array([c[4] for c in calls]), 'status': np.array([c[5] for c in calls]),
            'iters': np.array(iters), 'T': np.array(Ts),
            'plant_state': np.array(plant_x), 'plant_input': np.array(plant_u),
            'options': np.array([vehicle.options['ideal_prediction'], vehicle.options['ideal_update']])}


def main():
    mg.install_stubs()
    lg.install_struct_stubs()
    out = {}
    for name, scenario, vopt in RUNS:
        res = run_reference_freeT_closed_loop(scenario, 0.5, vopt)
        print(name, 'steps', len(res['status']), 'status', res['status'], 'T', np.round(res['T'], 3),
              'final plant state', np.round(res['plant_state'][-1], 4))
        for key, val in res.items():
            out['%s_%s' % (name, key)] = val
        out[name + '_dt'] = 0.5
    np.savez_compressed(OUT, **out)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
