"""Generate tests/golden/model_golden_freeT_ext.npz from the REFERENCE's own modelling code:
HolonomicOrient, the planar Quadrotor and SimpleQuadrotor3D with a free end time.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_model_golden_freeT_ext.py

The stand-ins, the scenes and the stored quantities are make_model_golden.py's: each problem is the
reference builder's scene of the fixed-T name (FREE_T_SCENES) handed to the reference's
``Point2point`` with freeT=True and no problem options, as scenarios.config_*_freeT build it.  As for
config_freeT there, the reference's T parameter and T variable carry one registry value per sample
(6.3, 8.0, 9.7) and t is 0.  Stored per problem: the flat layouts, x, p, every constraint row g and
the objective f at three random points, the bounds, the trajectory extraction of a perturbed initial
guess, the obstacle motion and the host's parameter vector and initial guess.

``build_reference`` is also the builder of make_freeT_loop_golden_ext.py and
make_freeT_closed_loop_golden_ext.py, which install it in place of make_model_golden's.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_model_golden as mg                          # noqa: E402

OUT = os.path.join(HERE, 'model_golden_freeT_ext.npz')
FREE_T_SCENES = {'config_holonomic_orient_freeT': 'config_holonomic_orient',
                 'config_quadrotor2d_freeT': 'config_quadrotor2d',
                 'config_quadrotor3d_simple_freeT': 'config_quadrotor3d_simple'}
_build_fixed = mg.build_reference


def build_reference(name):
    """make_model_golden.build_reference, and for the names of FREE_T_SCENES the scene of the fixed-T
    name with freeT=True and no problem options."""
    if name not in FREE_T_SCENES:
        return _build_fixed(name)
    p2p = mg.ref_import('problems.point2point')
    fixed = p2p.Point2point
    p2p.Point2point = lambda vehicle, environment, options=None, freeT=False: fixed(
        vehicle, environment, options={'verbose': 0}, freeT=True)
    try:
        return _build_fixed(FREE_T_SCENES[name])
    finally:
        p2p.Point2point = fixed


def install():
    """Route make_model_golden.build_reference (which the loop scripts call) through build_reference."""
    mg.build_reference = build_reference


def main():
    mg.install_stubs()
    out = {}
    for name in FREE_T_SCENES:
        Xs, Ps, Gs, Fs = [], [], [], []
        for k in range(3):
            mg.REG = mg.Registry(seed=1000 * k + 7)
            mg.REG.fixed = {'t': 0., 'T': 6.3 + 1.7 * k}
            # labels restart for every build so that the layout strings are comparable
            opt = mg.ref_import('basics.optilayer')
            for cls in list(opt.OptiChild.__subclasses__()) + [opt.OptiChild]:
                if hasattr(cls, '_labels'):
                    cls._labels = []
            problem = build_reference(name)
            var, par, g, lb, ub, f = mg.flatten(problem)
            Xs.append(np.concatenate([v.column() for _, _, v in var]))
            Ps.append(np.concatenate([v.column() for _, _, v in par]))
            Gs.append(g)
            Fs.append(f)
        C, tax, tr = mg.trajectories(problem, 10., 11)
        out[name + '_traj_C'], out[name + '_traj_time'] = C, tax
        for key, val in tr.items():
            out[name + '_traj_' + key] = val
        out[name + '_traj_keys'] = np.array(sorted(tr))
        out[name + '_host_P'], out[name + '_host_X0'] = mg.host_values(problem, par, var, 0.37)
        out[name + '_obst'] = mg.obstacle_motion(problem, 5.0)
        print(name, 'reference layout: n', len(Xs[0]), 'm', len(Gs[0]), 'n_par', len(Ps[0]))
        out[name + '_X'], out[name + '_P'] = np.array(Xs), np.array(Ps)
        out[name + '_G'], out[name + '_F'] = np.array(Gs), np.array(Fs)
        out[name + '_lb'], out[name + '_ub'] = lb, ub
        out[name + '_var_layout'] = np.array(['%s|%s|%dx%d' % ((lab, nm) + v.a.shape) for lab, nm, v in var])
        out[name + '_par_layout'] = np.array(['%s|%s|%dx%d' % ((lab, nm) + v.a.shape) for lab, nm, v in par])
    path = sys.argv[1] if len(sys.argv) > 1 else OUT
    np.savez_compressed(path, **out)
    print('wrote', path)


if __name__ == '__main__':
    main()
