"""Cost of closing the MPC loop through the vehicle dynamics (execution/batch_mpc.py).

    python tools/closed_loop_bench.py [--scenario config5] [--batch 256] [--steps 50] [--runs 3] [--out DIR]

One scenario (default config 5, the revolving door), B instances x N MPC steps, in two modes
run alternately in one process: the ideal loop (the vehicle follows its spline) and the closed
loop with the first-order actuator lag (tau = 0.1 s) and the filtered input disturbance
(fc = 0.01, stdev = 0.05 on every input), the settings of the reference's
p2p_holonomic_disturbances example.  The update time is 0.1 s, 0.5 s for the Dubins
scenarios (the steps of their recorded reference loops).  Reported
per mode: the wall time per MPC step (a device synchronise closes every timed step), and in
the closed loop the time of the plant-step launches alone from CUDA events around each call.
The card's name and power limit are read in the same call.  Needs a CUDA device; prints one
JSON line and writes it to DIR/closed_loop_bench.json when --out is given."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UPDATE_TIME = {'config_dubins_plain': 0.5, 'config_dubins': 0.5}


def closed_options(n_input):
    return {'ideal_prediction': False, 'ideal_update': False, '1storder_delay': True, 'time_constant': 0.1,
            'input_disturbance': {'fc': 0.01, 'stdev': 0.05 * np.ones(n_input)}}


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def one_run(mode, batch, steps, scenario='config5'):
    import torch
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    from omg_tools_b200.solver import b200
    pr = getattr(sc, scenario)()
    if mode == 'closed':
        veh = pr.vehicles[0]
        veh.set_options(closed_options(len(veh.prediction['input'])))
    bat = BatchMPC(pr, batch=batch, update_time=UPDATE_TIME.get(scenario, 0.1), seed=1)
    plant_ms = []
    step_fn = b200.closed_loop_step

    def timed(*a, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step_fn(*a, **kw)
        e1.record()
        plant_ms.append((e0, e1))
    b200.closed_loop_step = timed
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
        b200.closed_loop_step = step_fn
    plant = [a.elapsed_time(b) for a, b in plant_ms]
    fail = int(sum((s != 0).sum() for s in bat.history['status']))
    return {'ms_per_step': 1e3 * float(np.mean(wall)), 'plant_ms_per_step': float(np.mean(plant)) if plant else 0.,
            'failed_solves': fail}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--scenario', default='config5', help='a function of omg_tools_b200.scenarios')
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('closed_loop_bench.py needs a CUDA device')
    res = {'card': card(), 'device': torch.cuda.get_device_name(0), 'batch': a.batch, 'steps': a.steps,
           'ideal': [], 'closed': []}
    if a.scenario != 'config5':
        res['scenario'] = a.scenario
    for _ in range(a.runs):
        for mode in ('ideal', 'closed'):
            res[mode].append(one_run(mode, a.batch, a.steps, a.scenario))
    for mode in ('ideal', 'closed'):
        ms = [r['ms_per_step'] for r in res[mode]]
        res[mode + '_ms_per_step_median'] = float(np.median(ms))
    res['plant_ms_per_step_median'] = float(np.median([r['plant_ms_per_step'] for r in res['closed']]))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        fname = 'closed_loop_bench.json' if a.scenario == 'config5' else 'closed_loop_bench_%s.json' % a.scenario
        with open(os.path.join(a.out, fname), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
