"""Cost of the batched MPC loop with a free motion time (execution/batch_mpc.py, FreeTPoint2point).

    python tools/freet_mpc_bench.py [--steps 40] [--closed] [--scenario NAME [--batch 256]] [--out DIR]

Two workloads at 0.5 s updates: config_freeT with a jittered batch of 1024 (jitter 0.1) and
config_dubins_freeT (init_v_til = 0.3) with a jittered batch of 256; --scenario (repeatable) runs
the named scenarios of omg_tools_b200/scenarios.py instead, each with a jittered batch of --batch
(e.g. config_holonomic_orient_freeT, config_quadrotor2d_freeT, config_quadrotor3d_simple_freeT).
Each runs until every
instance stopped or --steps updates.  Reported per workload and step: the wall time of the MPC
step (closed by a device synchronise), the solve time (CUDA events around the solve launch), the
time of the warm-start (omg_shift_free_batch) and prediction (omg_eval_batch) launches alone (CUDA
events around each call), and the number of active instances.  For comparison, the host path of
the warm start, shift_spline on every shifted block of each active instance (what the sequential
loop does per instance), is timed on the instances and motion times of the second step.  With
--closed the loops run through the vehicle's own dynamics at the reference's vehicle defaults
(ideal_update and ideal_prediction off) with the first-order lag (time constant 0.1) and the input
disturbance (fc 0.01, stdev 0.05 on every input), and the plant step (omg_closed_loop_step_free) is timed like the
other launches; the host's shift_spline is not timed then.  The card's
name and power limit are read in the same call.  Needs a CUDA device; prints one JSON line and
writes it to DIR/freet_mpc_bench.json when --out is given."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [('config_freeT', 1024, {}), ('config_dubins_freeT', 256, {'init_v_til': 0.3})]
DT = 0.5
CLOSED = {'ideal_update': False, 'ideal_prediction': False, '1storder_delay': True, 'time_constant': 0.1,
          'input_disturbance': {'fc': 0.01, 'stdev': 0.05}}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def _timed(events, fn):
    import torch

    def call(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn(*a, **kw)
        e1.record()
        events.append((e0, e1))
        return r
    return call


def host_shift_ms(bat, X, T, n_max=64):
    """shift_spline on every shifted block of up to n_max instances (host), ms per instance."""
    from omg_tools_b200.basics.spline import BSplineBasis
    from omg_tools_b200.basics.spline_extra import shift_spline
    idx = np.arange(min(n_max, X.shape[0]))
    t0 = time.perf_counter()
    for b in idx:
        u, target = (T[b] - DT, T[b]) if T[b] < 2 * DT else (DT, T[b] - DT)
        for off, L, nc, p, knots in bat.shift_blocks:
            shift_spline(X[b, off:off + L * nc].reshape(nc, L).T, u / target, BSplineBasis(knots, p))
    return 1e3 * (time.perf_counter() - t0) / len(idx)


def one_run(name, batch, kw, steps, closed=False):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    from omg_tools_b200.solver import b200
    pr = getattr(sc, name)(**kw)
    if closed:
        pr.vehicles[0].set_options(CLOSED)
    bat = BatchMPC(pr, batch=batch, update_time=DT, seed=1, jitter=0.1)
    ev = {'solve': [], 'shift': [], 'eval': [], 'plant': []}
    bat.solver.solve_batch_device = _timed(ev['solve'], bat.solver.solve_batch_device)
    bat.solver.shift_free_batch_device = _timed(ev['shift'], bat.solver.shift_free_batch_device)
    eval_fn, plant_fn = b200.eval_batch, b200.closed_loop_step_free
    b200.eval_batch = _timed(ev['eval'], eval_fn)
    b200.closed_loop_step_free = _timed(ev['plant'], plant_fn)
    rows = []
    host_ms = None
    try:
        for k in range(steps):
            if not bat.active.any():
                break
            if k == 1 and not closed:
                host_ms = host_shift_ms(bat, bat.X.cpu().numpy(), bat.X[:, bat.t_index].cpu().numpy())
            n_act = int(bat.active.sum())
            for v in ev.values():
                v.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            bat.step()
            torch.cuda.synchronize()
            wall = 1e3 * (time.perf_counter() - t0)
            ms = {key: sum(a.elapsed_time(b) for a, b in v) for key, v in ev.items()}
            rows.append({'active': n_act, 'wall_ms': wall, 'solve_ms': ms['solve'], 'shift_ms': ms['shift'],
                         'eval_ms': ms['eval'], 'plant_ms': ms['plant']})
    finally:
        b200.eval_batch, b200.closed_loop_step_free = eval_fn, plant_fn
    fail = int(sum((s > 0).sum() for s in bat.history['status']))
    med = lambda key: float(np.median([r[key] for r in rows[1:]]))     # (step 0: cold start)
    return {'scenario': name, 'batch': batch, 'closed': closed, 'steps': len(rows), 'stopped': int((~bat.active).sum()),
            'failed_solves': fail, 'active_per_step': [r['active'] for r in rows],
            'wall_ms_median': med('wall_ms'), 'solve_ms_median': med('solve_ms'),
            'shift_ms_median': med('shift_ms'), 'eval_ms_median': med('eval_ms'), 'plant_ms_median': med('plant_ms'),
            'host_shift_spline_ms_per_instance': host_ms,
            'host_shift_spline_ms_per_step_at_batch': host_ms * batch if host_ms else None,
            'per_step': rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--closed', action='store_true', help='closed loop with lag and disturbance')
    ap.add_argument('--scenario', action='append', default=None, help='scenario name (repeatable)')
    ap.add_argument('--batch', type=int, default=256, help='batch of the --scenario workloads')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('freet_mpc_bench.py needs a CUDA device')
    res = {'card': card(), 'device': torch.cuda.get_device_name(0), 'update_time': DT, 'runs': []}
    workloads = [(name, a.batch, {}) for name in a.scenario] if a.scenario else WORKLOADS
    for name, batch, kw in workloads:
        res['runs'].append(one_run(name, batch, kw, a.steps, a.closed))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        fn = 'freet_mpc_bench%s%s.json' % ('_' + '_'.join(a.scenario) if a.scenario else '',
                                           '_closed' if a.closed else '')
        with open(os.path.join(a.out, fn), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
