"""Generate tests/golden/fleet_loop_golden.npz: the REFERENCE's receding-horizon loop for the
problems with several vehicles in one NLP.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_fleet_loop_golden.py

The loop, the stand-ins and the solver are make_closed_loop_golden.py's (the CPU oracle on the
lowered tables, iteration counts recorded).  ``Problem.predict / store / simulate`` loop over
the problem's vehicles (problem.py:187-192), so every vehicle is predicted and simulated.
Stored per run and MPC step: x0, p, lbg, ubg, x, status, iters, and every vehicle's plant state
and input at the update boundaries ([steps + 1, n_veh, n]).

    config_interveh_offset_ideal
              examples/p2p_holonomic_interveh_avoidance.py with vehicle 0 starting 0.1 m off the
              head-on line, both ideal flags on; 12 x 0.1 s (knot crossing at 1.0 s)
    config_interveh_offset
              the same at the reference's non-ideal defaults; 12 x 0.1 s
    config_interveh_offset_disturbed
              the same with the settings of examples/p2p_holonomic_disturbances.py on both
              vehicles: first-order lag (tau 0.1), input disturbance fc 0.01, stdev 0.05.
              ``normal`` of the reference's vehicle module is replaced by the numpy twin of the
              device generator, instance 0, seed 0, signal v * n_input + j for input j of
              vehicle v: the reference draws per step, then per vehicle, then per signal.
    config_formation_central_ideal, config_formation_central
              examples/formation_holonomic_central.py, ideal and at the non-ideal defaults;
              4 x 0.5 s (knot crossing at 1.5 s)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_closed_loop_golden as cg                    # noqa: E402
import make_loop_golden as lg                           # noqa: E402
import make_model_golden as mg                          # noqa: E402

OUT = os.path.join(HERE, 'fleet_loop_golden.npz')

IDEAL = {'ideal_prediction': True, 'ideal_update': True}
DISTURBED = {'1storder_delay': True, 'time_constant': 0.1, 'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}}

# run -> (scenario of this repository, vehicle options, steps, update time)
RUNS = {'config_interveh_offset_ideal': ('config_interveh_offset', IDEAL, 12, 0.1),
        'config_interveh_offset': ('config_interveh_offset', None, 12, 0.1),
        'config_interveh_offset_disturbed': ('config_interveh_offset', DISTURBED, 12, 0.1),
        'config_formation_central_ideal': ('config_formation_central', IDEAL, 4, 0.5),
        'config_formation_central': ('config_formation_central', None, 4, 0.5)}


def build_reference_interveh_offset():
    """examples/p2p_holonomic_interveh_avoidance.py against the reference's API, vehicle 0's
    start moved 0.1 m off the head-on line (same values as scenarios.config_interveh_offset)."""
    hol, env = mg.ref_import('vehicles.holonomic'), mg.ref_import('environment.environment')
    shp, p2p = mg.ref_import('basics.shape'), mg.ref_import('problems.point2point')
    N = 2
    vehicles = [hol.Holonomic() for _ in range(N)]
    for k, vehicle in enumerate(vehicles):
        vehicle.set_initial_conditions([1.5 * np.cos((k * 2. * np.pi) / N),
                                        1.5 * np.sin((k * 2. * np.pi) / N) + (0.1 if k == 0 else 0.)])
        vehicle.set_terminal_conditions([-1.5 * np.cos((k * 2. * np.pi) / N),
                                         -1.5 * np.sin((k * 2. * np.pi) / N)])
    environment = env.Environment(room={'shape': shp.Square(5.)})
    problem = p2p.Point2point(vehicles, environment, options={'verbose': 0}, freeT=False)
    problem.set_options({'inter_vehicle_avoidance': True})
    problem.father.reset()
    problem.construct()
    return problem


def run_fleet_loop(name, vehicle_options, n_steps, update_time, sample_time=0.01):
    from omg_tools_b200 import scenarios as sc
    tables = getattr(sc, name)(build_solver=False).father.tables
    opt = mg.ref_import('basics.optilayer')
    for cls in list(opt.OptiChild.__subclasses__()) + [opt.OptiChild]:
        if hasattr(cls, '_labels'):
            cls._labels = []
    mg.REG = mg.Registry(seed=3)
    problem = build_reference_interveh_offset() if name == 'config_interveh_offset' else mg.build_reference(name)
    for vehicle in problem.vehicles:
        vehicle.set_options(vehicle_options or {})
        vehicle.problem = problem
    if vehicle_options and 'input_disturbance' in vehicle_options:
        cg.install_twin_normal(len(problem.vehicles) * 2)   # two inputs per Holonomic vehicle
    solver = cg.RecordingSolver(tables)
    problem.problem, _ = problem.father.construct_problem(problem.options, problem=solver)
    problem.father.init_transformations(problem.init_primal_transform, problem.init_dual_transform)
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
    plant = {key: np.stack([np.asarray(v.signals[key], float)[:, ::n_samp].T for v in problem.vehicles], axis=1)
             for key in ('state', 'input')}
    return {'x0': np.array([c[0] for c in calls]), 'p': np.array([c[1] for c in calls]),
            'lbg': np.array([c[2] for c in calls]), 'ubg': np.array([c[3] for c in calls]),
            'x': np.array([c[4] for c in calls]), 'status': np.array([c[5] for c in calls]),
            'iters': np.array(solver.iters), 'plant_state': plant['state'], 'plant_input': plant['input'],
            'dt': update_time}


def main():
    mg.install_stubs()
    lg.install_struct_stubs()
    out = {}
    for run, (name, vopt, n_steps, dt) in RUNS.items():
        res = run_fleet_loop(name, vopt, n_steps, dt)
        print(run, 'status', res['status'], 'iters', res['iters'], 'final plant state',
              np.round(res['plant_state'][-1], 4).tolist())
        for key, val in res.items():
            out['%s_%s' % (run, key)] = val
    np.savez_compressed(OUT, **out)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
