"""Generate tests/golden/ideal_history_golden.npz: BatchMPC's history on config 5 (revolving
door) with the ideal flags on, recorded from a checkout of the commit before the closed loop
was added, through the CPU emulation of its kernels:

    git worktree add /tmp/before <commit>
    python tests/golden/make_ideal_history_golden.py /tmp/before

tests/test_closed_loop.py runs the same loop in this tree and requires the same history bit
for bit: with both flags on, BatchMPC must run exactly the code it ran before.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'ideal_history_golden.npz')
BATCH, STEPS, JITTER, SEED = 2, 12, 0.05, 4


def main(tree):
    tree = os.path.abspath(tree)
    sys.path.insert(0, os.path.join(tree, 'tests'))
    sys.path.insert(0, tree)
    import torch
    import emu_support
    emu_support.activate()
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(sc.config5(), batch=BATCH, update_time=0.1, jitter=JITTER, seed=SEED,
                   device=torch.device('cpu'))
    bat.run(STEPS)
    h = bat.history
    np.savez_compressed(OUT, state=np.array(h['state']), iters=np.array(h['iters']),
                        status=np.array(h['status']), X=bat.X.numpy())
    print('wrote', OUT, 'from', tree)


if __name__ == '__main__':
    main(sys.argv[1])
