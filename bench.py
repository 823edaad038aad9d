"""bench.py -- MPC solves/sec of the batched Point2point hot path on an H100.

  python bench.py --gpus N --steps K --warmup W          (N>1 under torchrun)
  python bench.py --impl reference ...                   (CPU oracle arm)
  python bench.py ... --dump-outputs DIR                 (also write the last step's results)

A "step" is one cold solve of the whole batch (BASELINE config 2: batch 1024
Holonomic Point2point, 10 knot intervals, 3 circular obstacles) from the linear
initial guess.  `value` times the kernel with inputs resident in HBM (CUDA
events on the launching stream); `e2e` times the reference-facing C-ABI call
omg_solve_batch_host with host buffers (H2D + solve + D2H inside).  Per-GPU batch
is fixed (weak scaling): the batch shards across ranks with no collective.
The inputs are a pure function of the arguments, so two builds run with the same
arguments can be compared output for output through --dump-outputs.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

# the source tree may be read-only: no bytecode caches written next to the sources
sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

BATCH = 1024
L2_FLUSH_BYTES = 256 << 20
DUMP_LIMIT_BYTES = 64 << 20


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='b200', choices=['b200', 'reference'])
    ap.add_argument('--batch', type=int, default=0,
                    help='instances (default: the BASELINE size of the workload: 1024; config 4: 512; config 5: 256)')
    ap.add_argument('--jitter', type=float, default=0.0)
    ap.add_argument('--cpu-sample', type=int, default=0)
    ap.add_argument('--workload', default='config2', choices=sorted(WORKLOADS),
                    help='BASELINE configuration (the metric is quoted on config2)')
    ap.add_argument('--scaling', default='weak', choices=['weak', 'strong'],
                    help='weak: --batch instances per GPU; strong: --batch instances in total')
    ap.add_argument('--agents', type=int, default=64, help='config3: agents of the formation')
    ap.add_argument('--formations', type=int, default=1,
                    help='config3: independent formations run side by side in one batch (value counts '
                         'formation-iterations; "limiter" in the output gives the resident blocks per GPU)')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None,
                    help='after the timed steps, write the results of the last timed step as DIR/<name>.npy '
                         '(float64; rank 0 under torchrun; a fixed, seeded sample of instances above 64 MiB)')
    args = ap.parse_args()
    if args.batch <= 0:
        args.batch = {'config4': 512, 'config4_5obs': 512, 'config5': 256}.get(args.workload, BATCH)
    return args


class ClockSampler(object):
    """nvidia-smi clocks / throttle reasons sampled every 50 ms during the timed
    region (one long-running nvidia-smi -lms process, read afterwards)."""
    Q = ('clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,'
         'clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ['nvidia-smi', '-i', str(self.index), '--query-gpu=' + self.Q,
                 '--format=csv,noheader,nounits', '-lms', '50'],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def stop(self):
        if self.proc is None:
            return
        try:
            self.proc.terminate()
            out, _ = self.proc.communicate(timeout=5)
            for line in out.decode().strip().splitlines():
                self.rows.append([c.strip() for c in line.split(',')])
        except Exception:
            try:
                self.proc.kill()
            except Exception:
                pass

    def summary(self):
        def num(x):
            try:
                return float(x)
            except ValueError:
                return None
        sm = [num(r[0]) for r in self.rows if r and num(r[0]) is not None]
        mx = [num(r[1]) for r in self.rows if len(r) > 1 and num(r[1]) is not None]
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown',
                 'sw_power_cap']
        reasons = [n for k, n in enumerate(names)
                   if any(len(r) > 3 + k and r[3 + k].lower().startswith('active')
                          for r in self.rows)]
        return {'sm_mhz': float(np.median(sm)) if sm else None,
                'sm_max_mhz': max(mx) if mx else None, 'reasons': reasons,
                'samples': len(self.rows)}


def roofline_bytes_per_solve(tb, K):
    """SURVEY.md 8(d) staged-KKT model: one write + one read of the packed
    condensed KKT per interior-point iteration + compulsory I/O."""
    n, m, n_par = tb.n, tb.m, tb.n_par
    return K * 2 * 8 * n * (n + 1) / 2 + 8 * (2 * n + n_par + 3 * m)


def flops_per_solve(tb, K):
    n = tb.n
    nnz2 = float(np.sum(np.diff(tb.jrow_ptr).astype(float) ** 2))
    return K * (n ** 3 / 3.0 + 4 * n * n + 2 * nnz2)


def fp64_flops_sparse(slv_info_str, K, tb):
    """Flops the sparse kernel actually executes per solve: gather records of the L D L^T
    factorisation (4 column terms of 3 flops each) x ~1.35 factorisations per iteration + the
    J^T Sigma J gather + the term streams; parsed from the library's structure report
    (OMG_B200_VERBOSE line, "pairs" = record slots)."""
    import re
    m = re.search(r'pairs=(\d+)', slv_info_str or '')
    pairs = float(m.group(1)) if m else 0.0
    nnz2 = float(np.sum(np.diff(tb.jrow_ptr).astype(float) ** 2)) / 2
    per_iter = 1.35 * pairs * 4 * 3 + 2 * 2 * nnz2 + 2 * 3 * (tb.G.n_terms + 2 * tb.J.n_terms + tb.W.n_terms)
    return K * per_iter


def measure_fp64_peak(dev):
    """cuBLAS DGEMM 4096^3 on this GPU, best of 5 (MEASURED_PEAKS.json has no fp64 entry)."""
    import torch
    a = torch.randn(4096, 4096, dtype=torch.float64, device=dev)
    b = torch.randn(4096, 4096, dtype=torch.float64, device=dev)
    torch.matmul(a, b)
    best = 1e9
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); torch.matmul(a, b); e1.record(); torch.cuda.synchronize(dev)
        best = min(best, e0.elapsed_time(e1))
    return 2 * 4096.0 ** 3 / (best * 1e-3) / 1e12


def measured_peaks():
    path = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(path):
        d = json.load(open(path))
        return float(d['hbm_gbs']), 'measured'
    return 3350.0, 'H100 SXM data sheet (HBM3, 700 W card)'


def dump_outputs(path, per_instance, whole=None):
    """Write every array as path/<name>.npy in float64.  `per_instance` arrays have one row per
    instance (or agent); when all arrays together exceed DUMP_LIMIT_BYTES, the same fixed, seeded
    sample of rows is written from each of them, and the sampled row numbers as rows.npy."""
    os.makedirs(path, exist_ok=True)
    per_instance = {k: np.asarray(v, dtype=np.float64) for k, v in per_instance.items()}
    whole = {k: np.asarray(v, dtype=np.float64) for k, v in (whole or {}).items()}
    total = sum(a.nbytes for a in per_instance.values()) + sum(a.nbytes for a in whole.values())
    if total > DUMP_LIMIT_BYTES:
        rows_total = len(next(iter(per_instance.values())))
        row_bytes = sum(a.nbytes for a in per_instance.values()) / float(rows_total)
        keep = max(1, int((DUMP_LIMIT_BYTES - sum(a.nbytes for a in whole.values())) // (row_bytes + 8)))
        rows = np.sort(np.random.default_rng(0).choice(rows_total, min(keep, rows_total), replace=False))
        per_instance = {k: a[rows] for k, a in per_instance.items()}
        whole['rows'] = rows.astype(np.float64)
    for k, a in list(per_instance.items()) + list(whole.items()):
        np.save(os.path.join(path, k + '.npy'), a)


def host_cores():
    """Usable host threads: affinity mask, capped by the cgroup CPU quota."""
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:
        quota, period = open('/sys/fs/cgroup/cpu.max').read().split()[:2]
        if quota != 'max':
            n = max(1, min(n, int(float(quota) / float(period) + 0.5)))
    except (OSError, ValueError):
        pass
    return n


def cpu_baseline(problem, X0, P, sample, threads):
    """Time the CPU oracle (the host restatement of the reference's
    CasADi+IPOPT path) on `sample` instances using `threads` processes."""
    from oracle import cpu_runner
    return cpu_runner.run(problem.father.tables, X0[:sample], P[:sample], threads)


def workload_config(args, tb, world):
    """The `config` object: identical for the GPU arm and the reference arm of one command."""
    B = args.batch if args.scaling == 'weak' else args.batch // world
    return {'workload': '%s, cold solve from the linear initial guess, %s instances' %
            (WORKLOADS[args.workload], 'jittered' if args.jitter > 0 else 'identical'),
            'n': int(tb.n), 'm': int(tb.m), 'n_par': int(tb.n_par),
            'batch_per_gpu': B, 'global_batch': world * B, 'tol': 1e-3,
            'l2': 'GPU arm: flushed between timed iterations (256 MiB fill)',
            'parallelism': 'dp%d (batch sharded, no collective)' % world}


WORKLOADS = {
    'config1': 'config1: Holonomic Point2point (examples/p2p_holonomic.py), 10 knot intervals, '
               '1 moving circular obstacle',
    'config2': 'config2: Holonomic Point2point, 10 knot intervals, 3 circular obstacles',
    'config3': 'config3: FormationPoint2point ADMM (metric: ADMM iterations/s)',
    'config4': 'config4: Quadrotor3D Point2point (examples/p2p_3dquadrotor.py), 10 knot '
               'intervals, 2 plate obstacles',
    'config5': 'config5: Holonomic Point2point through the revolving door '
               '(examples/revolving_door.py), 2 static + 2 rotating beams',
    'config4_5obs': 'config4 at BASELINE size: Quadrotor3D Point2point, 10 knot intervals, '
                    '5 plate obstacles (n=406)',
    # further models (not BASELINE configs; for kernel work on the XL path)
    'config_dubins_plain': 'Dubins Point2point, default formulation (examples/p2p_dubins.py scene, '
                           'fixed end time), cross-Hessian tables',
    'config_holonomic_orient': 'HolonomicOrient Point2point (examples/p2p_holonomic_orient.py scene, '
                               'fixed end time), shared heading products',
    'config_quadrotor3d_simple': 'SimpleQuadrotor3D Point2point, 2 plate obstacles',
}

# bounded CPU sample: about 20 s of single-core work of the C oracle per measurement
CPU_SAMPLE = {'config1': 2048, 'config2': 1024, 'config4': 96, 'config4_5obs': 32, 'config5': 512,
              'config_dubins_plain': 256, 'config_holonomic_orient': 32, 'config_quadrotor3d_simple': 256}


def build_problem(sc, workload, build_solver=True):
    if workload == 'config4_5obs':
        return sc.config4(n_obstacles=5, build_solver=build_solver)
    return getattr(sc, workload)(build_solver=build_solver)


def n_flat(problem):
    """Number of leading entries of x that are the vehicle's spline coefficients."""
    try:
        v = problem.vehicles[0]
        return int(v.n_spl * len(v.basis))
    except Exception:
        return 26


def run_config3(args, rank, world, dev):
    """BASELINE config 3: FormationPoint2point ADMM, --agents agents on a ring sharded over the
    GPUs; a "step" is one ADMM iteration (batched x-update + consensus exchange + z/lambda
    update + residual all-reduce).  Reports ADMM iterations/s and agent x-updates/s."""
    import torch
    import torch.distributed as dist
    from omg_tools_b200 import scenarios as sc
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    pr = sc.config3(args.agents)
    F = max(1, args.formations)
    run = FormationADMMRunner(pr, rank=rank, world=world, formations=F, spread=0.02 if F > 1 else 0.)
    for _ in range(max(args.warmup, 3)):
        run.dual_update(0.)
    torch.cuda.synchronize(dev)
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(args.steps):          # residuals stay on the device until the last iteration
        res = run.dual_update(0., fetch=(k == args.steps - 1))
    e1.record()
    torch.cuda.synchronize(dev)
    tm = torch.tensor([e0.elapsed_time(e1)], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(tm, op=dist.ReduceOp.MAX)
    st, it = run.status()
    per = run.formation_residuals()          # collective: every rank
    if args.dump_outputs and rank == 0:
        tensors = {k: getattr(run, k).cpu().numpy() for k in ('X', 'z_i', 'l_i', 'z_ij', 'l_ij')}
        dump_outputs(args.dump_outputs, dict(tensors, status=st, iters=it),
                     {'residuals': res, 'residuals_per_formation': per})
    if rank == 0:
        ms = float(tm[0])
        tb = pr.tb
        slots = run.solver.info()['ctas_per_sm'] * run.solver.info()['n_sm']
        line = {'metric': 'admm_iterations_per_sec', 'value': F * args.steps / (ms * 1e-3), 'unit': 'iterations/s',
                'n_gpus': world, 'steps': args.steps, 'warmup': max(args.warmup, 3),
                'ms_per_step': ms / args.steps, 'higher_is_better': True, 'scaling': 'strong',
                'vs_baseline': None, 'dtype': 'f64', 'data': 'synthetic',
                'config': {'workload': 'config3: FormationPoint2point ADMM, %d holonomic agents on a ring, '
                           '2 rectangular obstacles, rho = 1' % args.agents, 'n': int(tb.n), 'm': int(tb.m),
                           'n_par': int(tb.n_par), 'agents': args.agents, 'formations': F,
                           'agents_per_gpu': F * args.agents // world,
                           'parallelism': 'agents sharded over %d GPUs; exchange: all-gather of x_i '
                           '(26 doubles/agent), all-reduce of 3 residuals, all-gather of z_ij, l_ij' % world},
                'stats': {'agent_x_updates_per_sec': F * args.agents * args.steps / (ms * 1e-3),
                          'batch_iterations_per_sec': args.steps / (ms * 1e-3),
                          'primal_residual': res[0], 'dual_residual': res[1],
                          'primal_residual_per_formation': [float(v) for v in per[:, 0]],
                          'x_updates_succeeded': bool((st == 0).all()),
                          'mean_ip_iterations': float(it.mean()),
                          'limiter': 'latency of one x-update solve (a block per agent, %d blocks per GPU on '
                                     '%d resident slots) plus three latency-bound collectives per iteration'
                                     % (F * args.agents // world, slots)},
                'gpu_launches': 2 * args.steps}
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def run_reference(args, rank, world):
    """--impl reference: the reference's CPU path (oracle; CasADi+IPOPT is not
    installable in this image) on the host cores, same config and metric."""
    if rank != 0:
        return
    from omg_tools_b200 import scenarios as sc
    problem = build_problem(sc, args.workload, build_solver=False)
    cores = host_cores()
    sample = args.cpu_sample or CPU_SAMPLE[args.workload]
    if args.jitter > 0:
        X0, P = sc.instance_data(problem, sample, jitter=args.jitter, seed=100)
    else:
        X0, P = sc.instance_data(problem, 1, jitter=0.0)
        X0, P = np.repeat(X0, sample, 0), np.repeat(P, sample, 0)
    times = []
    info = None
    for k in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        info = cpu_baseline(problem, X0, P, sample, cores)
        dt = time.perf_counter() - t0
        if k >= args.warmup:
            times.append(dt)
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, {'x': info['x'], 'status': info['status'], 'iters': info['iters']})
    tot = sum(times)
    value = sample * args.steps / tot
    line = {
        'impl': 'reference', 'metric': 'mpc_solves_per_sec', 'value': value,
        'unit': 'solves/s', 'n_gpus': args.gpus, 'steps': args.steps,
        'warmup': args.warmup, 'ms_per_step': 1e3 * tot / args.steps,
        'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
        'dtype': 'f64', 'data': 'synthetic',
        'config': workload_config(args, problem.father.tables, world),
        'stats': {'mean_ip_iterations': float(np.mean(info['iters'])),
                  'succeeded_frac': float(np.mean(info['status'] == 0)), 'sample_per_step': sample},
        'cpu_baseline': {'value': value, 'unit': 'solves/s', 'cores': cores,
                         'kind': info['kind'], 'impl': info.get('impl'),
                         'sample': '%d %s instances of the workload per step' %
                         (sample, 'jittered' if args.jitter > 0 else 'identical')},
        'e2e': {'value': value, 'unit': 'solves/s', 'h2d_bytes_per_step': 0,
                'd2h_bytes_per_step': 0},
        'gpu_launches': 0}
    print(json.dumps(line))


def main():
    args = parse()
    rank = int(os.environ.get('RANK', '0'))
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if args.impl == 'reference':
        run_reference(args, rank, world)
        return
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit('bench.py needs a CUDA device (no CPU fallback)')
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=dev)
    import __graft_entry__ as ge
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    from omg_tools_b200 import scenarios as sc
    os.environ['OMG_B200_DEVICE'] = str(local)
    if args.workload == 'config3':
        return run_config3(args, rank, world, dev)
    os.environ['OMG_B200_VERBOSE'] = '1' if rank == 0 else ''
    problem = build_problem(sc, args.workload)
    slv, tb = problem.problem, problem.father.tables
    B = args.batch if args.scaling == 'weak' else args.batch // world   # per GPU
    if args.jitter > 0:
        X0h, Ph = sc.instance_data(problem, B, jitter=args.jitter, seed=100 + rank)
    else:
        X0h, Ph = sc.instance_data(problem, 1, jitter=0.0)
        X0h, Ph = np.repeat(X0h, B, 0), np.repeat(Ph, B, 0)
    X0 = torch.tensor(X0h, device=dev)
    P = torch.tensor(Ph, device=dev)
    LB, UB = torch.tensor(tb.lbg, device=dev), torch.tensor(tb.ubg, device=dev)
    X = torch.empty_like(X0)
    LAM = torch.empty((B, tb.m), dtype=torch.float64, device=dev)
    F = torch.empty(B, dtype=torch.float64, device=dev)
    ST = torch.empty(B, dtype=torch.int32, device=dev)
    IT = torch.empty(B, dtype=torch.int32, device=dev)
    flush = torch.empty(L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream(dev)

    def barrier():
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    def step():
        slv.solve_batch_device(X0, P, LB, UB, X, LAM, F, ST, IT, stream=stream)

    for _ in range(max(args.warmup, 3)):
        flush.fill_(1)
        step()
    barrier()
    sampler = ClockSampler(local)
    sampler.start()
    # ---- device-timed region: EXACTLY args.steps steps -------------------------
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
           for _ in range(args.steps)]
    barrier()
    for k in range(args.steps):
        flush.fill_(k & 1)              # evict L2 between timed iterations
        evs[k][0].record(stream)
        step()
        evs[k][1].record(stream)
    barrier()
    ms = [a.elapsed_time(b) for a, b in evs]
    tot_ms = float(sum(ms))
    kern_ms = tot_ms / args.steps       # one kernel launch per step
    iters = IT.cpu().numpy()
    status = ST.cpu().numpy()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, {'x': X.cpu().numpy(), 'lam_g': LAM.cpu().numpy(),
                                         'f': F.cpu().numpy(), 'status': status, 'iters': iters})
    # ---- e2e: host buffers through the C-ABI call --------------------------------
    pin = lambda a: torch.from_numpy(a).pin_memory().numpy()
    X0p, Pp = pin(X0h), pin(Ph)
    for _ in range(2):
        slv.solve_batch(X0p, Pp)
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        res = slv.solve_batch(X0p, Pp)
    torch.cuda.synchronize(dev)
    e2e_s = time.perf_counter() - t0
    sampler.stop()
    h2d = X0p.nbytes + Pp.nbytes + 2 * tb.m * 8
    d2h = res['x'].nbytes + res['lam_g'].nbytes + res['f'].nbytes + \
        res['status'].nbytes + res['iters'].nbytes
    # ---- max over ranks ------------------------------------------------------------
    agg = torch.tensor([tot_ms, e2e_s], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(agg, op=dist.ReduceOp.MAX)
    tot_ms, e2e_s = float(agg[0]), float(agg[1])
    if rank == 0:
        K = float(iters.mean())
        value = world * B * args.steps / (tot_ms * 1e-3)
        e2e_v = world * B * args.steps / e2e_s
        peak, how = measured_peaks()
        bps = roofline_bytes_per_solve(tb, K)
        achieved = B * bps / (kern_ms * 1e-3) / 1e9
        info = slv.info()
        fp64_peak = measure_fp64_peak(dev)
        slots = info['ctas_per_sm'] * info['n_sm']
        waves = B / float(slots)
        line = {
            'metric': 'mpc_solves_per_sec', 'value': value, 'unit': 'solves/s',
            'n_gpus': world, 'steps': args.steps, 'warmup': max(args.warmup, 3),
            'ms_per_step': tot_ms / args.steps, 'higher_is_better': True,
            'scaling': args.scaling, 'vs_baseline': None, 'dtype': 'f64',
            'data': 'synthetic',
            'config': workload_config(args, tb, world),
            'stats': {'mean_ip_iterations': K, 'succeeded_frac': float((status == 0).mean()),
                      'resident_slots_per_gpu': slots, 'waves': waves,
                      'wave_efficiency': waves / float(np.ceil(waves))},
            'roofline': {'bound': 'hbm', 'achieved': achieved, 'peak': peak,
                         'unit': 'GB/s', 'frac': achieved / peak,
                         'peak_source': how,
                         'model': 'staged-KKT bytes/solve = K*2*8*n(n+1)/2 + '
                                  '8(2n+n_par+3m) (SURVEY 8d); K=mean iterations',
                         'bytes_per_solve': bps,
                         'fp64_gflops_dense_model': B * flops_per_solve(tb, K) /
                         (kern_ms * 1e-3) / 1e9,
                         'fp64': {'achieved_tflops': B * fp64_flops_sparse(getattr(slv, 'structure', ''), K, tb) /
                                  (kern_ms * 1e-3) / 1e12,
                                  'peak_tflops': fp64_peak,
                                  'peak_source': 'cuBLAS DGEMM 4096^3 measured in this run',
                                  'note': 'flops the sparse kernel executes (L D L^T gather records x 1.35 '
                                          'factorisations/iteration + gathers + term streams)'},
                         'kernel_ms': kern_ms, 'smem_bytes': info['smem_bytes'],
                         'ctas_per_sm': info['ctas_per_sm']},
            'e2e': {'value': e2e_v, 'unit': 'solves/s',
                    'h2d_bytes_per_step': int(h2d), 'd2h_bytes_per_step': int(d2h)},
            'gpu_launches': args.steps,
            'clocks': sampler.summary()}
        cores = host_cores()
        if world == 1:
            sample = min(args.cpu_sample or CPU_SAMPLE[args.workload], len(X0h))
            t0 = time.perf_counter()
            cinfo = cpu_baseline(problem, X0h, Ph, sample, cores)
            dt = time.perf_counter() - t0
            line['cpu_baseline'] = {
                'value': sample / dt, 'unit': 'solves/s', 'cores': cores,
                'kind': cinfo['kind'], 'impl': cinfo.get('impl'),
                'sample': '%d instances of the same workload, %.3f s' % (sample, dt),
                # the two arms solve the same instances: largest difference of the solutions
                # (all variables / the vehicle's spline coefficients, which are unique)
                'max_abs_dx_vs_gpu': float(np.abs(cinfo['x'] - res['x'][:sample]).max()),
                'max_abs_dx_splines_vs_gpu': float(np.abs(cinfo['x'] - res['x'][:sample])[:, :n_flat(problem)].max()),
                'iterations_equal_frac': float(np.mean(cinfo['iters'] == res['iters'][:sample]))}
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
