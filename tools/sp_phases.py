"""Phase cycle counters of the sparse kernel (omg_ipm_kernel_sp) on config 2, instance 0 of a
full batch: python tools/sp_phases.py [batch] [jitter]

TICK(k) adds the cycles since the previous tick to counter k, so counter 0 (taken at the top of
an iteration) holds the accept pass of the iteration before it (and the setup once).  Counters
8, 15, 9 are the gather / panel / root parts of the factorisation (7); counter 14 is the root of
the backward sweep (10)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from omg_tools_b200 import scenarios as sc
from omg_tools_b200.solver.b200 import B200Solver

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024    # bench.py's config 2 batch
jitter = float(sys.argv[2]) if len(sys.argv) > 2 else 0.0
pr = sc.config2(build_solver=False)
tb = pr.father.tables
if jitter > 0:
    X0, P = sc.instance_data(pr, B, jitter=jitter, seed=100)
else:
    X0, P = sc.instance_data(pr, 1, jitter=0.0)
    X0, P = np.repeat(X0, B, 0), np.repeat(P, B, 0)
slv = B200Solver(tb, {'trace': 1})
print('n', tb.n, 'm', tb.m, slv.info(), slv.structure)
for rep in range(3):
    res = slv.solve_batch(X0, P)
    print('kernel %.3f ms  iters %d status %d' % (slv.last_timing()[0], res['iters'][0], res['status'][0]))
ph = slv.trace(512)[510:512].reshape(-1)
it = max(1, int(res['iters'][0]))
# (counter, name, indent): sub-counters are printed under the phase that contains them
rows = [(1, 'I1 Jacobian + row pass', 0), (2, 'I2 columns + reduce', 0), (3, 'I3 termination + mu', 0),
        (4, 'I4 Sigma pass', 0), (5, 'H gather', 0), (6, 'W + border + rhs + staging', 0),
        (7, 'factorisation', 0), (8, 'gather', 1), (15, 'panel', 1), (9, 'root', 1),
        (10, 'backward sweep', 0), (14, 'root', 1), (11, 'I10 step pass', 0),
        (12, 'I11 line search', 0), (0, 'I12 accept (+ setup)', 0), (13, 'result write', 0)]
top = [k for k, _, ind in rows if ind == 0]
tot = ph[top].sum()
print('phase cycles of instance 0: total %.0f, %d iterations -> %.0f cycles/iter' % (tot, it, tot / it))
print('  %-30s %10s %6s' % ('phase', 'cyc/iter', 'share'))
for k, nme, ind in rows:
    print('  %-30s %10.0f %5.1f%%' % (('  ' * ind + nme), ph[k] / it, 100 * ph[k] / tot))
