"""Phase cycle counters of the envelope (XL) kernel on config 4: python tools/gpu_xl_phases.py [n_obstacles] [batch]"""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from omg_tools_b200 import scenarios as sc
from omg_tools_b200.solver.b200 import B200Solver

nobs = int(sys.argv[1]) if len(sys.argv) > 1 else 2
B = int(sys.argv[2]) if len(sys.argv) > 2 else 132   # one block per SM of an H100
pr = sc.config4(nobs, build_solver=False)
tb = pr.father.tables
X0, P = sc.instance_data(pr, 1, jitter=0.0)
X0, P = np.repeat(X0, B, 0), np.repeat(P, B, 0)
slv = B200Solver(tb, {'trace': 1})
print('n', tb.n, 'm', tb.m, slv.info(), slv.structure)
for rep in range(2):
    res = slv.solve_batch(X0, P)
    print('kernel %.3f ms  iters %d status %d' % (slv.last_timing()[0], res['iters'][0], res['status'][0]))
ph = slv.trace(512)[510:512].reshape(-1)
names = ['setup/accept', 'row pass', 'col pass+reduce', 'barrier logic', 'sigma pass', 'zero+H gather',
         'W+border+rhs', 'factor:diag', 'factor:panel', 'factor:trailing', 'back solve', 'step pass',
         'line search', 'tail', 'slot14', 'slot15']
tot = ph[:14].sum()
print('phase cycles of instance 0 (total %.0f, %d iterations -> %.0f cycles/iter):' % (tot, res['iters'][0], tot / max(1, res['iters'][0])))
for nme, c in zip(names, ph[:16]):
    print('  %-16s %12.0f  %5.1f%%' % (nme, c, 100 * c / tot))
