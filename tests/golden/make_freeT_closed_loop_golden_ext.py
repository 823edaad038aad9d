"""Generate tests/golden/freeT_closed_loop_golden_ext.npz: the REFERENCE's receding-horizon loop with
a free motion time for HolonomicOrient and the two flat-output quadrotors, closed through the
vehicle's dynamics.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_freeT_closed_loop_golden_ext.py

The loop, the stand-ins, the solver call and the stored quantities are
make_freeT_closed_loop_golden.py's (run_reference_freeT_closed_loop); the reference builders are
make_model_golden_freeT_ext.py's (installed in place of make_model_golden's). Each run uses 0.5 s
updates and goes on until the reference stops (at most 60 steps, the cap of
run_reference_freeT_closed_loop).

    config_holonomic_orient_freeT     examples/p2p_holonomic_orient.py as written, the reference's
                                      vehicle defaults (ideal_prediction and ideal_update off)
    config_quadrotor2d_freeT          the scene of examples/p2p_quadrotor.py with freeT=True,
                                      reference defaults
    config_quadrotor3d_simple_freeT   SimpleQuadrotor3D with freeT=True, reference defaults
    config_holonomic_orient_freeT_ideal_update
                                      the first with ideal_update on and ideal_prediction off
    config_holonomic_orient_freeT_disturbed
                                      the first with the first-order lag (time constant 0.1) and the
                                      input disturbance (fc 0.01, stdev 0.05 on all three inputs);
                                      ``normal`` of the reference's vehicle module is replaced by the
                                      numpy twin of the device generator (instance 0, seed 0)

Stored per run and MPC step: x0, p, the solution x, the status, the iteration count and T; the
plant state and input at every update boundary (the initial ones first); and the update time.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_freeT_closed_loop_golden as fcg             # noqa: E402
import make_model_golden_freeT_ext as mgf              # noqa: E402

OUT = os.path.join(HERE, 'freeT_closed_loop_golden_ext.npz')
DT = 0.5
DISTURBED = {'1storder_delay': True, 'time_constant': 0.1,
             'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(3)}}
RUNS = (('config_holonomic_orient_freeT', 'config_holonomic_orient_freeT', None),
        ('config_quadrotor2d_freeT', 'config_quadrotor2d_freeT', None),
        ('config_quadrotor3d_simple_freeT', 'config_quadrotor3d_simple_freeT', None),
        ('config_holonomic_orient_freeT_ideal_update', 'config_holonomic_orient_freeT',
         {'ideal_update': True, 'ideal_prediction': False}),
        ('config_holonomic_orient_freeT_disturbed', 'config_holonomic_orient_freeT', DISTURBED))


def run(scenario, vehicle_options):
    """fcg.run_reference_freeT_closed_loop with the twin generator installed for the vehicle's three
    inputs (that function installs it for two)."""
    install = fcg.cg.install_twin_normal
    fcg.cg.install_twin_normal = lambda n_sig, **kw: install(3, **kw)
    try:
        return fcg.run_reference_freeT_closed_loop(scenario, DT, vehicle_options)
    finally:
        fcg.cg.install_twin_normal = install


def main():
    fcg.mg.install_stubs()
    mgf.install()
    fcg.lg.install_struct_stubs()
    out = {}
    for name, scenario, vopt in RUNS:
        res = run(scenario, vopt)
        print(name, 'steps', len(res['status']), 'status', res['status'], 'iters', res['iters'],
              'T', np.round(res['T'], 3), 'final plant state', np.round(res['plant_state'][-1], 4), flush=True)
        for key, val in res.items():
            out['%s_%s' % (name, key)] = val
        out[name + '_dt'] = DT
    path = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(path, **out)
    print('wrote', path)


if __name__ == '__main__':
    main()
