"""Generate tests/golden/freeT_loop_golden.npz: the REFERENCE's receding-horizon loop with a free
motion time.

Run in the authoring container only (needs /root/reference):

    python tests/golden/make_freeT_loop_golden.py

The reference's ``Simulator.update`` / ``Deployer.update`` order with ``FreeTPoint2point``
(predict; solve, whose ``init_step`` re-expresses every shifted spline with ``shift_spline`` from
the solved T and sets T to the target time, point2point.py:354-368; store; simulate by
min(update_time, T); ``stop_criterium``: T < update_time or the vehicle at its goal) runs straight
from /root/reference on the stand-ins of make_model_golden.py and make_loop_golden.py, with this
repository's CPU oracle on the lowered tables behind the solver call, until the reference stops.

The reference's problem has one more parameter than this framework's: it defines T twice under
one name, as a parameter handed to the vehicle and environment rows and as the variable of the
objective (point2point.py:53-62, 281-284), and never sets the parameter.  As in
make_model_golden.py, which gives both the same value, the parameter stands for the variable:
this framework's rows use the variable T wherever the reference's use the parameter.  So the
solver call drops the parameter's entry from the reference's p and solves this framework's
problem, whose rows equal the reference's at T_parameter = T_variable (model_golden.npz).  The
stored p is the vector without that entry.

Stored per configuration and MPC step: x0, p, the solution x, the status, the iteration count
and T; and the final state and the update time.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import make_model_golden as mg                          # noqa: E402
import make_loop_golden as lg                           # noqa: E402

OUT = os.path.join(HERE, 'freeT_loop_golden.npz')


class FreeTOracle(lg.OracleSolver):
    """The oracle behind the reference's solver call, on this framework's parameter vector (the
    reference's p without its unset parameter T at offset ``t_par``)."""

    def __init__(self, tables, t_par):
        lg.OracleSolver.__init__(self, tables)
        self.t_par = t_par

    def __call__(self, x0, p, lbg, ubg, **kw):
        p = np.delete(np.asarray(p, dtype=float).reshape(-1), self.t_par)
        return lg.OracleSolver.__call__(self, x0, p, lbg, ubg, **kw)


def run_reference_freeT_loop(name, update_time, max_steps=60, sample_time=0.01):
    from omg_tools_b200 import scenarios as sc
    tables = getattr(sc, name)(build_solver=False).father.tables
    opt = mg.ref_import('basics.optilayer')
    for cls in list(opt.OptiChild.__subclasses__()) + [opt.OptiChild]:
        if hasattr(cls, '_labels'):
            cls._labels = []
    mg.REG = mg.Registry(seed=3)
    problem = mg.build_reference(name)
    for vehicle in problem.vehicles:            # this framework implements the ideal case
        vehicle.set_options({'ideal_prediction': True, 'ideal_update': True})
        vehicle.problem = problem
    solver = FreeTOracle(tables, None)
    problem.problem, _ = problem.father.construct_problem(problem.options, problem=solver)
    par = problem.father._par_struct
    solver.t_par = t_par = par.locate((problem.label, 'T'))[0]
    assert par.size == tables.n_par + 1, (par.size, tables.n_par)
    problem.father.init_transformations(problem.init_primal_transform, problem.init_dual_transform)
    problem.reinitialize()
    t, Ts, iters = 0., [], []
    for k in range(max_steps):
        if k == 0:
            problem.initialize(t)
        problem.predict(t, update_time, sample_time, None, None, None, 0, False, False)
        problem.solve(t, update_time)
        Ts.append(float(np.asarray(problem.father.get_variables(problem, 'T')).reshape(-1)[0]))
        iters.append(int(solver.last['iters'][0]))
        problem.store(t, update_time, sample_time)
        problem.simulate(t, update_time, sample_time)
        t = np.round(t + update_time, 6)
        if problem.stop_criterium(t, update_time):
            break
    else:
        raise RuntimeError('%s did not stop within %d steps' % (name, max_steps))
    calls = solver.calls
    return {'x0': np.array([c[0] for c in calls]), 'p': np.array([c[1] for c in calls]),
            'x': np.array([c[4] for c in calls]), 'status': np.array([c[5] for c in calls]),
            'iters': np.array(iters), 'T': np.array(Ts),
            'state': np.asarray(problem.vehicles[0].signals['state'], float)[:, -1]}


def main():
    mg.install_stubs()
    lg.install_struct_stubs()
    out = {}
    for name, dt in (('config_freeT', 0.5), ('config_freeT_moving', 0.5)):
        res = run_reference_freeT_loop(name, dt)
        print(name, 'steps', len(res['status']), 'status', res['status'], 'T', np.round(res['T'], 3),
              'final state', np.round(res['state'], 4))
        for key, val in res.items():
            out['%s_%s' % (name, key)] = val
        out[name + '_dt'] = dt
    np.savez_compressed(OUT, **out)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
