"""Cost of one device-resident MPC update (execution/device_mpc.py, omg_mpc_update) against one
BatchMPC step on the same instances.

    python tools/mpc_update_bench.py [--batch 1024] [--updates 20] [--runs 3] [--out DIR]

Config 2 (BASELINE's batch workload, three static obstacles), B instances jittered by 0.2, N ideal
updates of 0.1 s from the cold start, in three cases run one after the other, `--runs` times in
alternation:
  eager   DeviceMPC.update called from Python on the current stream;
  graph   one DeviceMPC.update captured in a CUDA graph (torch.cuda.graph on a side stream) after an
          eager first update, then replayed once per update: the loop state lives on the device, so
          every replay is the next update;
  batch   BatchMPC.step (host packing of the parameters, host prediction maps, H2D of P).
Each update is timed with CUDA events on the stream it runs on; the first update (cold start,
first-call allocations) is left out of the median.  For the eager case the solve's own device
time (omg_last_timing) is reported too, and its share of the update.  The card's name and power
limit are read in the same call.  Needs a CUDA device; prints one JSON line and writes it to
DIR/mpc_update_bench.json when --out is given."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from closed_loop_bench import card          # noqa: E402

JITTER, SEED, UPDATE_TIME = 0.2, 0, 0.1


def _setup(batch, dev):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    bat = BatchMPC(sc.config2(), batch=batch, update_time=UPDATE_TIME, jitter=JITTER, seed=SEED, device=dev)
    nd = bat.vehicle.n_dim
    obs = np.zeros((batch, len(bat.obs), 3 * nd + 1))
    for k, d in enumerate(bat.obs):
        obs[:, k, :nd], obs[:, k, nd:2 * nd], obs[:, k, 2 * nd:3 * nd] = d['x'], d['v'], d['a']
    t = lambda a: torch.tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    return bat, t(bat.state), t(bat.poseT), t(obs)


def run_device(batch, updates, graph):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.device_mpc import DeviceMPC
    dev = torch.device('cuda', 0)
    _, st0, stT, obs = _setup(batch, dev)
    mpc = DeviceMPC(sc.config2(), batch, UPDATE_TIME, 0.01, int(UPDATE_TIME / 0.01) + 1, device=dev)
    mpc.update(st0, stT, obs)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    if graph:
        g, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        with torch.cuda.graph(g, stream=stream):
            mpc.update(st0, stT, obs)
    ms, solve_ms, failed = [], [], 0
    for _ in range(updates - 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record()
            if graph:
                g.replay()
            else:
                mpc.update(st0, stT, obs)
            e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
        if not graph:
            solve_ms.append(mpc.solver.last_timing()[0])
        failed += int((mpc.status != 0).sum())
    return ms, solve_ms, failed, mpc.time


def run_batch(batch, updates):
    import torch
    dev = torch.device('cuda', 0)
    bat, _, _, _ = _setup(batch, dev)
    bat.step()
    ms = []
    for _ in range(updates - 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bat.step()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms, int(sum((s != 0).sum() for s in bat.history['status'][1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1024)
    ap.add_argument('--updates', type=int, default=20)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('mpc_update_bench needs a CUDA device')
    import __graft_entry__
    __graft_entry__.build()
    res = {k: [] for k in ('eager', 'graph', 'batch')}
    solve, failed = [], {}
    for _ in range(args.runs):
        ms, sm, f, t_e = run_device(args.batch, args.updates, False)
        res['eager'] += ms
        solve += sm
        failed['eager'] = f
        ms, _, f, t_g = run_device(args.batch, args.updates, True)
        res['graph'] += ms
        failed['graph'] = f
        assert np.array_equal(t_e, t_g)
        ms, f = run_batch(args.batch, args.updates)
        res['batch'] += ms
        failed['batch'] = f
    med = {k: float(np.median(v)) for k, v in res.items()}
    line = {'workload': 'config2', 'batch': args.batch, 'jitter': JITTER, 'updates': args.updates, 'runs': args.runs,
            'card': card(), 'median_ms_per_update': med,
            'range_ms': {k: [float(np.min(v)), float(np.max(v))] for k, v in res.items()},
            'eager_solve_ms': float(np.median(solve)), 'eager_solve_share': float(np.median(solve)) / med['eager'],
            'failed_solves_per_run': failed}
    print(json.dumps(line))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'mpc_update_bench.json'), 'w') as fp:
            json.dump(line, fp)


if __name__ == '__main__':
    main()
