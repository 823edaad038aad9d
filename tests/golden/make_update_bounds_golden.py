"""Generate tests/golden/update_bounds_golden.npz from the REFERENCE's own exporter.

Needs a checkout of the reference where make_model_golden.REF points:

    python tests/golden/make_update_bounds_golden.py

The reference's C++ export writes, per obstacle, which constraint rows Point2Point::updateBounds
frees when the obstacle's avoid flag is false (export.py _create_updateBounds) and which parameters
fillParameterDict writes from the obstacle_t of every update (_create_fillParameterDict).  Both are
generated as C++ source text from the problem's structure.  This script builds BASELINE configs 1,
2 and 5 and the Holonomic3D example with the reference's modelling code under the stand-in modules
of make_model_golden.py, runs those two generator methods of the reference's Export class and parses
the code they emit.  Per config and obstacle k it stores:

    <name>_rows_<k>       the g rows updateBounds frees (set to -inf / +inf when not avoided)
    <name>_lbg_<k>, _ubg_<k>   the default bounds it restores on those rows when avoided
    <name>_params_<k>     the parameter names fillParameterDict writes for obstacle k
    <name>_poff_<k>       [offset, length] in p of checkpoints and rad, from the reference's layout

tests/test_device_mpc_obstacles.py compares mpc_obstacles_desc with them row for row.
"""
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_model_golden as mg  # noqa: E402

OUT = os.path.join(HERE, 'update_bounds_golden.npz')
NAMES = ('config1', 'config2', 'config5', 'config_holonomic3d')


class _Cat(object):
    """The .cat of the father's bound structs (casadi.tools struct values in the reference)."""

    def __init__(self, cat):
        self.cat = cat


def _size(self, k=None):
    """casadi's MX.size(k): rows for k = 1, columns for k = 2; the shape without an argument."""
    return self.a.shape if k is None else self.a.shape[k - 1]


def build(name):
    mg.REG = mg.Registry(seed=7)
    mg.REG.fixed = {'T': 12. if name == 'config_holonomic3d' else 10., 't': 0.}
    opt = mg.ref_import('basics.optilayer')
    for cls in list(opt.OptiChild.__subclasses__()) + [opt.OptiChild]:
        if hasattr(cls, '_labels'):
            cls._labels = []
    problem = mg.build_reference(name)
    father = problem.father
    # the bounds in children order, as OptiFather.construct_constraints lays them out
    _, par, _, lb, ub, _ = mg.flatten(problem)
    father._lb, father._ub = _Cat(lb), _Cat(ub)
    if not hasattr(father, '_constraint_shutdown'):
        father._constraint_shutdown = {}
    return problem, father, par


def main():
    mg.install_stubs()
    mg.MX.size = _size
    exp = mg.ref_import('export.export')
    out = {}
    for name in NAMES:
        problem, father, par = build(name)
        bounds = exp.Export._create_updateBounds(None, father, problem)['updateBounds']
        fill = exp.Export._create_fillParameterDict(None, father)['fillParameterDict']
        obstacles = problem.environment.obstacles
        blocks = re.split(r'\tif\(!obstacles\[(\d+)\]\.avoid\)\{\n', bounds)[1:]
        assert len(blocks) == 2 * len(obstacles), name
        offsets, o = {}, 0
        for lab, nm, v in par:
            offsets[(lab, nm)] = (o, v.a.size)
            o += v.a.size
        for k, obst in enumerate(obstacles):
            assert int(blocks[2 * k]) == k
            freed, restored = blocks[2 * k + 1].split('\t}else{\n')
            rows = [int(r) for r in re.findall(r'lbg\[(\d+)\] = -inf;', freed)]
            assert rows == [int(r) for r in re.findall(r'ubg\[(\d+)\] = \+inf;', freed)]
            lbg = dict((int(r), float(v)) for r, v in re.findall(r'lbg\[(\d+)\] = ([^;]+);', restored))
            ubg = dict((int(r), float(v)) for r, v in re.findall(r'ubg\[(\d+)\] = ([^;]+);', restored))
            assert sorted(lbg) == rows and sorted(ubg) == rows, (name, k)
            out['%s_rows_%d' % (name, k)] = np.array(rows, dtype=np.int64)
            out['%s_lbg_%d' % (name, k)] = np.array([lbg[r] for r in rows])
            out['%s_ubg_%d' % (name, k)] = np.array([ubg[r] for r in rows])
            params = re.findall(r'par_dict\["%s"\]\["(\w+)"\] = ' % obst.label, fill)
            out['%s_params_%d' % (name, k)] = np.array(params)
            out['%s_poff_%d' % (name, k)] = np.array([offsets[(obst.label, 'checkpoints')],
                                                      offsets[(obst.label, 'rad')]], dtype=np.int64)
            print(name, obst.label, 'rows', rows[0], '..', rows[-1], 'params', params)
        out[name + '_n_obs'] = np.array(len(obstacles))
    np.savez_compressed(OUT, **out)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
