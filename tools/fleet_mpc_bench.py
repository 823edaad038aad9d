"""Cost of the batched MPC loop for several vehicles in one problem (execution/batch_mpc.py).

    python tools/fleet_mpc_bench.py [--scenario config_formation_central] [--batch 256] [--steps 20]
                                    [--runs 3] [--out DIR]

One multi-vehicle scenario (default the central formation of four Holonomic vehicles, solved
on the XL kernel), B jittered instances x N MPC steps of 0.5 s (0.1 s for the inter-vehicle
avoidance scenarios), in two modes run alternately in one process: the ideal loop (every
vehicle follows its spline) and the closed loop at the reference's non-ideal defaults with the
first-order actuator lag (tau = 0.1 s) and the filtered input disturbance (fc = 0.01,
stdev = 0.05) on every vehicle.  Reported per mode: the wall time per MPC step (a device
synchronise closes every timed step), and in the closed loop the time of the fleet plant-step
launch alone (omg_closed_loop_step_fleet, one block per instance and vehicle) from CUDA events
around each call.  The card's name and power limit are read in the same call.  Needs a CUDA
device; prints one JSON line and writes it to DIR/fleet_mpc_bench.json when --out is given."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from closed_loop_bench import card, closed_options          # noqa: E402

UPDATE_TIME = {'config_interveh': 0.1, 'config_interveh_offset': 0.1}


def one_run(mode, batch, steps, scenario):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    from omg_tools_b200.solver import b200
    pr = getattr(sc, scenario)()
    if mode == 'closed':
        for veh in pr.vehicles:
            veh.set_options(closed_options(len(veh.prediction['input'])))
    bat = BatchMPC(pr, batch=batch, update_time=UPDATE_TIME.get(scenario, 0.5), seed=1, jitter=0.1)
    plant_ms = []
    step_fn = b200.closed_loop_step_fleet

    def timed(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step_fn(*a, **kw)
        e1.record()
        plant_ms.append((e0, e1))
    b200.closed_loop_step_fleet = timed
    try:
        bat.step()                                 # warm-up: module load, first solve from cold start
        torch.cuda.synchronize()
        plant_ms.clear()
        wall = []
        for _ in range(steps - 1):
            t0 = time.perf_counter()
            bat.step()
            torch.cuda.synchronize()
            wall.append(time.perf_counter() - t0)
    finally:
        b200.closed_loop_step_fleet = step_fn
    plant = [a.elapsed_time(b) for a, b in plant_ms]
    fail = int(sum((s != 0).sum() for s in bat.history['status']))
    return {'ms_per_step': 1e3 * float(np.mean(wall)), 'plant_ms_per_step': float(np.mean(plant)) if plant else 0.,
            'failed_solves': fail}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenario', default='config_formation_central', help='a function of omg_tools_b200.scenarios')
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('fleet_mpc_bench.py needs a CUDA device')
    res = {'card': card(), 'device': torch.cuda.get_device_name(0), 'scenario': a.scenario, 'batch': a.batch,
           'steps': a.steps, 'ideal': [], 'closed': []}
    for _ in range(a.runs):
        for mode in ('ideal', 'closed'):
            res[mode].append(one_run(mode, a.batch, a.steps, a.scenario))
    for mode in ('ideal', 'closed'):
        res[mode + '_ms_per_step_median'] = float(np.median([r['ms_per_step'] for r in res[mode]]))
    res['plant_ms_per_step_median'] = float(np.median([r['plant_ms_per_step'] for r in res['closed']]))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'fleet_mpc_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
