"""Generate tests/golden/closed_loop_golden_ext.npz: the REFERENCE's receding-horizon loop for the
vehicles with a heading or an attitude, at the reference's own (non-ideal) vehicle options unless
stated otherwise, each run through its first knot crossing.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_closed_loop_golden_ext.py

The loop, the stand-ins, the solver and the recorded quantities are make_closed_loop_golden.py's
(run_closed_loop); the reference builders are make_model_golden's.

    config_dubins_plain, config_dubins
              Dubins, default formulation and examples/p2p_dubins.py's substitution; reference
              defaults; 6 x 0.5 s
    config_holonomic_orient
              examples/p2p_holonomic_orient.py, reference defaults; 12 x 0.1 s
    config_quadrotor2d
              examples/p2p_quadrotor.py, reference defaults; 7 x 0.1 s (knot at t = 0.5)
    config_quadrotor3d_simple
              SimpleQuadrotor3D, reference defaults; 6 x 0.5 s
    config_holonomic_orient_ideal, config_quadrotor2d_ideal
              the same two with ideal_prediction and ideal_update on
    config_dubins_plain_disturbed
              config_dubins_plain with the first-order lag (tau 0.1) and the input disturbance
              fc 0.01, stdev 0.05 on both inputs; the reference's ``normal`` is replaced by the
              device generator's draws (instance 0, seed 0) as for config_disturbances; 6 x 0.5 s
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_closed_loop_golden as cg                    # noqa: E402

OUT = os.path.join(HERE, 'closed_loop_golden_ext.npz')

DISTURBED = {'1storder_delay': True, 'time_constant': 0.1,
             'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(2)}}
IDEAL = {'ideal_prediction': True, 'ideal_update': True}
# run -> (scenario, MPC steps, update time, vehicle options, device generator's normals)
RUNS = {
    'config_dubins_plain': ('config_dubins_plain', 6, 0.5, None, False),
    'config_dubins': ('config_dubins', 6, 0.5, None, False),
    'config_holonomic_orient': ('config_holonomic_orient', 12, 0.1, None, False),
    'config_quadrotor2d': ('config_quadrotor2d', 7, 0.1, None, False),
    'config_quadrotor3d_simple': ('config_quadrotor3d_simple', 6, 0.5, None, False),
    'config_holonomic_orient_ideal': ('config_holonomic_orient', 12, 0.1, IDEAL, False),
    'config_quadrotor2d_ideal': ('config_quadrotor2d', 7, 0.1, IDEAL, False),
    'config_dubins_plain_disturbed': ('config_dubins_plain', 6, 0.5, DISTURBED, True),
}


def run(name, n_steps, dt, vehicle_options, twin_normal):
    """cg.run_closed_loop; with twin_normal the reference's normal draws the device generator's
    numbers, installed right after the reference problem is built."""
    build = cg.mg.build_reference
    if twin_normal:
        def build_with_twin(scenario):
            problem = build(scenario)
            cg.install_twin_normal(len(problem.vehicles[0].prediction['input']))
            return problem
        cg.mg.build_reference = build_with_twin
    try:
        return cg.run_closed_loop(name, n_steps, dt, vehicle_options=vehicle_options)
    finally:
        cg.mg.build_reference = build


def main():
    cg.mg.install_stubs()
    cg.lg.install_struct_stubs()
    out = {}
    for key, (name, n_steps, dt, vopt, twin) in RUNS.items():
        res = run(name, n_steps, dt, vopt, twin)
        print(key, 'status', res['status'], 'iters', res['iters'],
              'final plant state', np.round(res['plant_state'][-1], 4))
        for k, val in res.items():
            out['%s_%s' % (key, k)] = val
        out[key + '_dt'] = dt
    path = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(path, **out)
    print('wrote', path)


if __name__ == '__main__':
    main()
