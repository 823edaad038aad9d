"""Generate tests/golden/freeT_loop_golden_ext.npz: the REFERENCE's ideal receding-horizon loop with
a free motion time for HolonomicOrient and the two flat-output quadrotors.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_freeT_loop_golden_ext.py

The loop, the stand-ins and the solver call are make_freeT_loop_golden.py's
(run_reference_freeT_loop: ideal_prediction and ideal_update on, the reference's unset T parameter
dropped from p, this repository's CPU oracle behind the solver call); the reference builders are
make_model_golden_freeT_ext.py's (installed in place of make_model_golden's). Each run uses 0.5 s
updates and goes on until the reference stops (at most 60 steps, the cap of
run_reference_freeT_loop).

    config_holonomic_orient_freeT     examples/p2p_holonomic_orient.py as written
    config_quadrotor2d_freeT          the scene of examples/p2p_quadrotor.py with freeT=True
    config_quadrotor3d_simple_freeT   SimpleQuadrotor3D in the scene of examples/p2p_3dquadrotor.py,
                                      freeT=True

Stored per run and MPC step: x0, p, the solution x, the status, the iteration count and T; and
the final state and the update time.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_freeT_loop_golden as fg                     # noqa: E402
import make_model_golden_freeT_ext as mgf              # noqa: E402

OUT = os.path.join(HERE, 'freeT_loop_golden_ext.npz')
RUNS = ('config_holonomic_orient_freeT', 'config_quadrotor2d_freeT', 'config_quadrotor3d_simple_freeT')
DT = 0.5


def main():
    fg.mg.install_stubs()
    mgf.install()
    fg.lg.install_struct_stubs()
    out = {}
    for name in RUNS:
        res = fg.run_reference_freeT_loop(name, DT)
        print(name, 'steps', len(res['status']), 'status', res['status'], 'iters', res['iters'],
              'T', np.round(res['T'], 3), 'final state', np.round(res['state'], 4), flush=True)
        for key, val in res.items():
            out['%s_%s' % (name, key)] = val
        out[name + '_dt'] = DT
    path = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(path, **out)
    print('wrote', path)


if __name__ == '__main__':
    main()
