"""Cost of per-instance obstacle shapes and avoid flags in the device MPC update
(DeviceMPC.set_obstacles, include/omg_b200.h omg_mpc_set_obstacles).

    python tools/mpc_obstacles_bench.py [--batch 1024] [--updates 20] [--runs 3] [--out DIR]

Config 2 (BASELINE's batch workload, three static obstacles, m = 563 rows), B instances jittered
by 0.2, N ideal updates of 0.1 s from the cold start, in three cases run one after the other,
`--runs` times in alternation on one card:
  plain    the handle without obstacles attached: every instance solves with the tables' bounds,
           one row shared by all blocks;
  on       obstacles attached with every avoid flag set: the same problem, but each instance reads
           its own bound row (2 m doubles, about 9 MB over a batch of 1024);
  toggle   obstacles attached, and before every update a set call with new random avoid flags
           (each obstacle of each instance avoided with probability 1/2).
Each update is timed with CUDA events on the current stream, the set call of `toggle` separately;
the first update (cold start, first-call allocations) is left out of the medians.  The solve's own
device time (omg_last_timing) is reported too.  The card's name and power limit are read in the
same call.  Needs a CUDA device; prints one JSON line and writes it to
DIR/mpc_obstacles_bench.json when --out is given."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from closed_loop_bench import card          # noqa: E402
from mpc_update_bench import _setup, UPDATE_TIME  # noqa: E402


def run(case, batch, updates, seed):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.device_mpc import DeviceMPC
    dev = torch.device('cuda', 0)
    _, st0, stT, obs = _setup(batch, dev)
    mpc = DeviceMPC(sc.config2(), batch, UPDATE_TIME, 0.01, int(UPDATE_TIME / 0.01) + 1, device=dev)
    if case != 'plain':
        mpc.set_obstacles(avoid=torch.ones((batch, mpc.n_obs), dtype=torch.int32, device=dev))
    rng = np.random.default_rng(seed)
    masks = [torch.tensor(rng.uniform(size=(batch, mpc.n_obs)) < 0.5, dtype=torch.int32, device=dev)
             for _ in range(updates)]
    ms, set_ms, solve_ms, failed = [], [], [], 0
    for k in range(updates):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        if case == 'toggle':
            mpc.set_obstacles(avoid=masks[k])
        ev[1].record()
        mpc.update(st0, stT, obs)
        ev[2].record()
        ev[2].synchronize()
        if k:
            set_ms.append(ev[0].elapsed_time(ev[1]))
            ms.append(ev[1].elapsed_time(ev[2]))
            solve_ms.append(mpc.solver.last_timing()[0])
            failed += int((mpc.status != 0).sum())
    return ms, set_ms, solve_ms, failed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1024)
    ap.add_argument('--updates', type=int, default=20)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('mpc_obstacles_bench needs a CUDA device')
    cases = ('plain', 'on', 'toggle')
    res = {c: {'ms': [], 'set_ms': [], 'solve_ms': [], 'failed': 0} for c in cases}
    run('plain', a.batch, 3, 0)                  # (module load, first-call allocations)
    for r in range(a.runs):
        for c in cases:
            ms, set_ms, solve_ms, failed = run(c, a.batch, a.updates, r)
            res[c]['ms'] += ms
            res[c]['set_ms'] += set_ms
            res[c]['solve_ms'] += solve_ms
            res[c]['failed'] += failed
            res[c].setdefault('run_median_ms', []).append(round(float(np.median(ms)), 3))
    out = {'bench': 'mpc_obstacles', 'config': 'config2', 'batch': a.batch, 'updates': a.updates, 'runs': a.runs}
    out['card'] = card()
    for c in cases:
        d = res[c]
        out[c] = {'median_update_ms': round(float(np.median(d['ms'])), 3),
                  'run_median_ms': d['run_median_ms'],
                  'median_solve_ms': round(float(np.median(d['solve_ms'])), 3),
                  'failed_instance_updates': d['failed']}
    out['toggle']['median_set_ms'] = round(float(np.median(res['toggle']['set_ms'])), 4)
    out['on_vs_plain'] = round(out['on']['median_update_ms'] / out['plain']['median_update_ms'], 4)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'mpc_obstacles_bench.json'), 'w') as fp:
            fp.write(line + '\n')


if __name__ == '__main__':
    main()
