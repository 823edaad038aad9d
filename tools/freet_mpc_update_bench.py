"""Cost of one device-resident MPC update with a free motion time (execution/device_mpc.py,
omg_mpc_create_freet) against one BatchMPC free-T step on the same instances.

    python tools/freet_mpc_update_bench.py [--batch 1024] [--runs 3] [--out DIR]

config_freeT (the minimum-time Holonomic problem, n=126), B instances jittered by 0.2, ideal updates
of 0.5 s from the cold start until every instance has stopped, in three cases run one after the
other, `--runs` times in alternation:
  eager   DeviceMPC.update called from Python on the current stream;
  graph   one DeviceMPC.update captured in a CUDA graph (torch.cuda.graph on a side stream) after an
          eager first update, then replayed once per update;
  batch   BatchMPC free-T steps (active mask, index_select of the running rows, host packing of the
          parameters, T read back every step).
Each update is timed with CUDA events on the stream it runs on; the first update (cold start,
first-call allocations) is left out.  Reported: the median ms per update over the updates in which
at least half of the batch still runs, the whole run's ms (every update after the first), the eager
solve's own device time (omg_last_timing) and its share, the update after which every instance has
stopped (null when an instance still runs after MAX_UPDATES: a DeviceMPC instance whose solve fails keeps
its warm start and is solved again, where BatchMPC accepts the failed result), and the failed solves.  The card's name and power limit are read in the same call.  Needs
a CUDA device; prints one JSON line and writes it to DIR/freet_mpc_update_bench.json when --out is
given."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from closed_loop_bench import card          # noqa: E402

JITTER, SEED, UPDATE_TIME, MAX_UPDATES = 0.2, 0, 0.5, 80


def _setup(batch, dev):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(sc.config_freeT(), batch=batch, update_time=UPDATE_TIME, jitter=JITTER, seed=SEED, device=dev)
    nd = bat.vehicle.n_dim
    obs = np.zeros((batch, len(bat.obs), 3 * nd + 1))
    for k, d in enumerate(bat.obs):
        obs[:, k, :nd], obs[:, k, nd:2 * nd], obs[:, k, 2 * nd:3 * nd] = d['x'], d['v'], d['a']
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    return bat, t(bat.state), t(bat.poseT), t(obs)


def run_device(batch, graph):
    """ms and running instances of every update after the first, solve ms (eager), failed solves,
    the stop step and the final motion times."""
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.device_mpc import DeviceMPC
    dev = torch.device('cuda', 0)
    _, st0, stT, obs = _setup(batch, dev)
    mpc = DeviceMPC(sc.config_freeT(), batch, UPDATE_TIME, 0.01, int(UPDATE_TIME / 0.01) + 1, device=dev)
    mpc.update(st0, stT, obs)
    torch.cuda.synchronize()
    failed = int((mpc.status.cpu() > 0).sum())
    stream = torch.cuda.current_stream()
    if graph:
        g, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(g, stream=stream):
            mpc.update(st0, stT, obs)
    ms, running, solve_ms, stop = [], [], [], None
    for k in range(1, MAX_UPDATES):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            if graph:
                g.replay()
            else:
                mpc.update(st0, stT, obs)
            e1.record()
        e1.synchronize()
        st = mpc.status.cpu().numpy()
        if not (st != -1).any():
            stop = k
            break
        ms.append(e0.elapsed_time(e1))
        running.append(int((st != -1).sum()))
        if not graph:
            solve_ms.append(mpc.solver.last_timing()[0])
        failed += int((st > 0).sum())
    return ms, running, solve_ms, failed, stop, mpc.motion_time().cpu().numpy(), int((st != -1).sum())


def run_batch(batch):
    import torch
    dev = torch.device('cuda', 0)
    bat, _, _, _ = _setup(batch, dev)
    bat.step()
    ms, running = [], []
    while bat.active.any():
        n_run = int(bat.active.sum())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bat.step()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        running.append(n_run)
    failed = int(sum((s > 0).sum() for s in bat.history['status']))
    return ms, running, failed, len(bat.history['status']), bat.history['T'][-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1024)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('freet_mpc_update_bench needs a CUDA device')
    import __graft_entry__
    __graft_entry__.build()
    half = args.batch / 2.
    res = {k: {'half': [], 'all': []} for k in ('eager', 'graph', 'batch')}
    solve, failed, stop, running_at_end = [], {}, {}, {}
    for _ in range(args.runs):
        for case in ('eager', 'graph'):
            ms, run, sm, f, s, T, left = run_device(args.batch, case == 'graph')
            running_at_end[case] = left
            res[case]['all'] += ms
            res[case]['half'] += [m for m, r in zip(ms, run) if r >= half]
            if case == 'eager':
                solve += [m for m, r in zip(sm, run) if r >= half]
                T_eager = T
            else:
                assert np.array_equal(T, T_eager)
            failed[case], stop[case] = f, s
        ms, run, f, s, T_batch = run_batch(args.batch)
        res['batch']['all'] += ms
        res['batch']['half'] += [m for m, r in zip(ms, run) if r >= half]
        failed['batch'], stop['batch'] = f, s
    med = {k: float(np.median(v['half'])) for k, v in res.items()}
    line = {'workload': 'config_freeT', 'batch': args.batch, 'jitter': JITTER, 'update_time': UPDATE_TIME,
            'runs': args.runs, 'card': card(), 'median_ms_per_update_half_running': med,
            'run_ms': {k: float(np.sum(v['all'])) / args.runs for k, v in res.items()},
            'eager_solve_ms': float(np.median(solve)), 'eager_solve_share': float(np.median(solve)) / med['eager'],
            'stop_step': stop, 'running_after_%d_updates' % MAX_UPDATES: running_at_end,
            'failed_solves_per_run': failed,
            'max_abs_motion_time_diff_vs_batch': float(np.abs(T_eager - T_batch).max())}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'freet_mpc_update_bench.json'), 'w') as fp:
            json.dump(line, fp)


if __name__ == '__main__':
    main()
