"""Functional CPU emulation of the CUDA source (tools/cpu_emu): omg_tools_b200/csrc/
omg_b200.cu compiled with g++ against a cuda_runtime.h stand-in, every thread of a block a
fiber, __syncthreads / warp shuffles as barriers.  The emulated kernels -- the same source
lines the GPU runs -- are compared with the CPU oracle.  This is test infrastructure for a
container without a GPU: it checks table decoding, the shared-memory layout chosen for a
H100, barrier placement, the blocked envelope factorisation and the interior-point logic,
not performance and not data races.  The product never loads this library."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from omg_tools_b200 import scenarios as sc
from omg_tools_b200.solver import b200
from oracle import ipm_c

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
import sys
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emu_support                       # noqa: E402
EMU_LIB = emu_support.EMU_LIB
CPU = None


@pytest.fixture(scope='module')
def emu():
    if not ipm_c.available():
        pytest.skip('C oracle not built')
    saved = emu_support.activate()            # B200Solver objects built below bind to it
    yield b200._lib
    emu_support.restore(saved)                # the product library for everything else


def _compare(pr, B, jitter, seed, n_flat, options=None):
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, B, jitter=jitter, seed=seed)
    if options:
        pr.problem.set_options(options)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=4, options=options)
    return res, ref


@pytest.mark.parametrize('kernel, name, B, layout', [
    ('sparse', 'config1', 3, (28368, 7)), ('sparse', 'config2', 2, (54832, 4)), ('sparse', 'config5', 2, None),
    ('envelope', 'config1', 3, (97408, 2)), ('envelope', 'config2', 2, (113552, 2)), ('envelope', 'config5', 2, None)])
def test_standard_kernel_matches_oracle(emu, monkeypatch, kernel, name, B, layout):
    """BASELINE configs 1, 2, 5 through both kernel families: omg_ipm_kernel_sp (sparse
    L D L^T on the minimum-degree structure, thread streams, 128 threads, 4 blocks/SM for
    config 2) and omg_ipm_kernel_2cta (envelope factorisation, 256 threads, 2 blocks/SM):
    same statuses and iteration counts as the C oracle, solutions to rounding."""
    if kernel == 'envelope':
        monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    pr = getattr(sc, name)()
    info = pr.problem.info()
    if layout:
        assert (info['smem_bytes'], info['ctas_per_sm']) == layout   # the H100 layout
    res, ref = _compare(pr, B, 0.1, 1, 26)
    assert np.array_equal(res['status'], ref['status']) and (ref['status'] == 0).all()
    assert np.array_equal(res['iters'], ref['iters'])
    assert np.abs(res['x'] - ref['x'])[:, :26].max() < 1e-4
    assert np.abs(res['f'] - ref['f']).max() < 1e-8
    # tight tolerance: the end point is solver independent for the vehicle splines
    tight = {'tol': 1e-8, 'compl_inf_tol': 1e-8, 'constr_viol_tol': 1e-8}
    res, ref = _compare(pr, 1, 0.1, 2, 26, tight)
    assert res['status'][0] == 0 == ref['status'][0]
    assert np.abs(res['x'] - ref['x'])[:, :26].max() < 1e-7


def test_sparse_structure_of_config2_is_pinned(emu):
    """The host-side symbolic analysis (csrc/omg_sp_host.cuh): constrained minimum degree, dense
    root, supernodes of four columns with at most 8 explicit zeros each -- config 2 has 8
    supernode levels (29 column levels), 3 960 stored entries, a root of 36 columns, every level
    free of equality rows (early inertia rejection on all of them), 4 blocks per SM."""
    info = sc.config2().problem.structure
    for piece in ('N=200', 'nnz(L)=3960', 'levels=8 (early-reject 8)', 'root=36', 'ctas/SM=4', 'smem=54832'):
        assert piece in info, (piece, info)


def test_early_inertia_rejection_does_not_change_the_iterates(emu, monkeypatch):
    """The early rejection stops a factorisation at the first negative pivot among variables that
    no equality row touches (omg_sp.cuh: SP_CHECK) instead of counting the pivots to the end; the
    verdict -- wrong inertia, increase delta_w -- is the same, so every iterate is: bit-identical
    solutions, iteration counts and multipliers with the switch on and off, on jittered cold
    starts (which take the inertia correction in about a third of their iterations)."""
    pr = sc.config2()
    X0, P = sc.instance_data(pr, 6, jitter=0.2, seed=7)
    on = pr.problem.solve_batch(X0, P)
    monkeypatch.setenv('OMG_B200_EARLY_REJECT', '0')
    off = sc.config2().problem.solve_batch(X0, P)
    assert 'early-reject 0' in sc.config2().problem.structure
    for key in ('x', 'lam_g', 'f', 'iters', 'status'):
        assert np.array_equal(on[key], off[key]), key


@pytest.mark.parametrize('snw', ['1', '2', '3'])
def test_narrower_supernodes_give_the_same_iterates(emu, monkeypatch, snw):
    """OMG_B200_SNW limits the supernode width (1 = one column per level step, the kernel before
    the supernodes): other level schedules, records and panel shapes, the same factorisation --
    statuses and iteration counts as the oracle, solutions to rounding."""
    monkeypatch.setenv('OMG_B200_SNW', snw)
    res, ref = _compare(sc.config2(), 2, 0.1, 1, 26)
    assert np.array_equal(res['status'], ref['status']) and (ref['status'] == 0).all()
    assert np.array_equal(res['iters'], ref['iters'])
    assert np.abs(res['x'] - ref['x'])[:, :26].max() < 1e-6


@pytest.mark.parametrize('name, nflat, options', [
    ('config_freeT', 26, None),                 # T as a variable, cubic rows, soft restoration
    ('config_holonomic3d', 39, None),           # 3-D hyperplanes, 1 block/SM layout
    ('config_quadrotor2d', 26, None),           # sign-indefinite pivots (IPOPT's inertia count)
    ('config2', 26, {'inertia_mode': 1}),       # the positional inertia test of the first kernels
])
def test_more_models_and_options(emu, name, nflat, options):
    """Further problem classes through the emulated standard kernel: identical iteration
    counts as the C oracle, solutions to rounding."""
    pr = getattr(sc, name)()
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 2, jitter=0.05, seed=1)
    if options:
        pr.problem.set_options(options)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=2, options=options)
    assert np.array_equal(res['status'], ref['status']) and (res['status'] == 0).all()
    assert np.array_equal(res['iters'], ref['iters'])
    assert np.abs(res['x'] - ref['x'])[:, :nflat].max() < 1e-6
    assert np.abs(res['f'] - ref['f']).max() < 1e-9


def test_one_block_per_sm_variant(emu, monkeypatch):
    """omg_ipm_kernel (envelope, 512 threads, everything in shared memory)."""
    monkeypatch.setenv('OMG_B200_KERNEL', 'envelope')
    monkeypatch.setenv('OMG_B200_CTAS', '1')
    pr = sc.config2()
    assert pr.problem.info()['ctas_per_sm'] == 1
    res, ref = _compare(pr, 1, 0.1, 3, 26)
    assert res['status'][0] == 0 and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x'])[:, :26].max() < 1e-5


def test_xl_kernel_config4(emu):
    """omg_ipm_kernel_xl with intermediates (Quadrotor3D, 236 mids, K in shared memory)."""
    pr = sc.config4()
    res, ref = _compare(pr, 1, 0.0, 0, 36)
    assert res['status'][0] == 0 and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x']).max() < 1e-4
    assert abs(res['f'][0] - ref['f'][0]) < 1e-7


def test_xl_kernel_cross_hessian_dubins_default(emu):
    """The cross-Hessian slots of the XL kernel (Dubins without substitution: hyperplane
    normal times integrated position; include/omg_b200.h xq_*): identical path on the
    nominal instance."""
    pr = sc.config_dubins_plain()
    tb = pr.father.tables
    assert tb.nnz_wx > 0
    res, ref = _compare(pr, 1, 0.0, 0, 26)
    assert res['status'][0] == 0 and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x']).max() < 1e-7
    assert np.abs(res['lam_g'] - ref['lam_g']).max() < 1e-6


def test_xl_kernel_mid_mid_hessian_bicycle(emu):
    """Products of two intermediates (bicycle steering-rate rows): the C^T M C gather of the
    XL kernel, identical path on the nominal instance from a rolling initial guess."""
    pr = sc.config_bicycle()
    tb = pr.father.tables
    assert (tb.xq_b >= 0).any()
    X0, P = sc.instance_data(pr, 1)
    X0[0, :7] = 0.3
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=1)
    assert res['status'][0] == 0 == ref['status'][0] and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x']).max() < 1e-5
    assert np.abs(res['f'] - ref['f']).max() < 1e-7


def test_xl_kernel_k_in_scratch_central_formation(emu):
    """FormationPoint2pointCentral (n = 420, KKT envelope 390 KB): the XL kernel with K in the
    L2-resident scratch, 2 blocks/SM layout."""
    pr = sc.config_formation_central()
    tb, f = pr.father.tables, pr.father
    info = pr.problem.info()
    assert tb.env_size * 8 > 232448 and info['ctas_per_sm'] == 2
    X0, P = f.get_variables().cat[None], f.set_parameters(0.).cat[None]
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=1)
    assert res['status'][0] == 0 and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x']).max() < 1e-6


def test_two_vehicles_with_intervehicle_avoidance(emu):
    """A multi-vehicle NLP (examples/p2p_holonomic_interveh_avoidance.py): two vehicles swap
    places, separated by a hyperplane spline.  The head-on start is symmetric (pass left or
    right is decided by rounding), so the start is perturbed."""
    pr = sc.config_interveh()
    tb, f = pr.father.tables, pr.father
    assert (tb.n, tb.m, tb.n_par) == (111, 619, 14)
    rng = np.random.default_rng(0)
    X0 = f.get_variables().cat[None] + 0.05 * rng.standard_normal((1, tb.n))
    P = f.set_parameters(0.).cat[None]
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=1)
    assert res['status'][0] == 0 and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x']).max() < 1e-8
    x = res['x'][0]                      # the vehicles keep their distance: 2 x radius 0.1
    ent = f._var_struct.entries
    C = [x[ent[(v.label, 'splines_seg0')][0]:][:26].reshape(2, 13) for v in pr.vehicles]
    S = pr.vehicles[0].basis.eval_basis(np.linspace(0., 1., 101))
    d = np.hypot(*(S.dot((C[0] - C[1]).T).T))
    assert d.min() > 0.2 - 1e-3


def test_xl_kernel_trailer_free_end_time(emu):
    """examples/p2p_trailer.py (two vehicles in one problem, free end time, 290 shared
    intermediates, 53 k Jacobian slots): the emulated XL kernel follows the oracle."""
    pr = sc.config_trailer(init_v_til=0.3)
    tb, f = pr.father.tables, pr.father
    X0, P = f.get_variables().cat[None], f.set_parameters(0.).cat[None]
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=1)
    assert res['status'][0] == 0 and res['iters'][0] == ref['iters'][0]
    assert np.abs(res['x'] - ref['x']).max() < 1e-6 and np.abs(res['f'] - ref['f']).max() < 1e-9


def test_feasibility_kernel_and_the_fallback_after_restoration_failed(emu):
    """omg_feas_kernel (Levenberg-Marquardt on the constraint violation; one block per
    instance, normal equations through the CSC view of the Jacobian, dense Cholesky with
    the right-hand side as an extra row) against oracle_feas_batch, on standard tables
    (config 5, two cold starts whose line search fails, and one that succeeds) and on tables
    with intermediates (the Dubins example with a free end time from the reference's
    zero-speed guess) -- and B200Solver.solve_batch's default path around it: solve,
    feasibility phase for the Restoration_Failed instances, one more solve."""
    pr = sc.config5()
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 12, jitter=0.3, seed=5)
    X0, P = X0[[5, 10, 0]], P[[5, 10, 0]]
    xg, vg, kg = pr.problem.feasibility_batch(X0, P)
    xc, vc, kc = ipm_c.feas_batch(tb, X0, P)
    assert np.array_equal(kg, kc) and (kc > 0).all()
    assert np.abs(xg - xc).max() < 1e-9 and np.abs(vg - vc).max() < 1e-9
    x5, v5, k5 = pr.problem.feasibility_batch(X0, P, max_steps=5)      # the step limit
    assert (k5 == 5).all() and (v5 >= vg).all()
    plain = ipm_c.solve_batch_full(tb, X0, P, threads=3, options={'feas_steps': 0})
    assert list(plain['status']) == [2, 2, 0]
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=3)
    # (these two are local infeasibilities of the separation constraints: the second solve
    # wanders for hundreds of iterations and fails again, no iteration-exact comparison)
    assert np.array_equal(res['status'], ref['status'])
    assert (res['iters'][:2] > plain['iters'][:2]).all() and res['iters'][2] == plain['iters'][2] == ref['iters'][2]
    assert np.abs(res['x'] - ref['x'])[2].max() < 1e-6
    pr.problem.set_options({'feas_steps': 0})                           # switched off
    off = pr.problem.solve_batch(X0, P)
    assert np.array_equal(off['status'], plain['status']) and (off['iters'] < res['iters'])[:2].all()

    pr = sc.config_dubins_freeT()
    tb, f = pr.father.tables, pr.father
    assert tb.n_mid > 0
    X0, P = sc.instance_data(pr, 2, jitter=0.05, seed=3)
    res = pr.problem.solve_batch(X0, P)
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=2)
    plain = ipm_c.solve_batch_full(tb, X0, P, threads=2, options={'feas_steps': 0})
    assert (plain['status'] == 2).all()
    assert (res['status'] == 0).all() and np.array_equal(res['iters'], ref['iters'])
    assert np.abs(res['x'] - ref['x']).max() < 1e-4 and np.abs(res['f'] - ref['f']).max() < 1e-7
    assert (res['f'] > 7.0).all() and (res['f'] < 8.0).all()           # the end time


def test_native_cpp_caller_with_the_feasibility_fallback(emu, tmp_path):
    """examples/native/native_solve.cpp (C++ against the C ABI only, table file in, no
    Python) linked to the emulation library: the Dubins example with a free end time from
    the zero-speed guess -- omg_solve_batch_host, omg_feas_batch_host for the
    Restoration_Failed instances, omg_solve_batch_host again -- equals the oracle."""
    pr = sc.config_dubins_freeT(build_solver=False)
    tb = pr.father.tables
    exe = str(tmp_path / 'native_emu')
    subprocess.check_call(['g++', '-O2', '-I', os.path.join(ROOT, 'include'),
                           os.path.join(ROOT, 'examples', 'native', 'native_solve.cpp'), '-o', exe,
                           EMU_LIB, '-Wl,-rpath,' + os.path.dirname(EMU_LIB)])
    X0, P = sc.instance_data(pr, 2, jitter=0.05, seed=3)
    b200.save_tables(tb, str(tmp_path / 'p.omgtbl'))
    X0.tofile(str(tmp_path / 'x0.f64'))
    P.tofile(str(tmp_path / 'p.f64'))
    out = subprocess.check_output([exe, str(tmp_path / 'p.omgtbl'), str(tmp_path / 'x0.f64'),
                                   str(tmp_path / 'p.f64'), '2', str(tmp_path / 'x.f64')])
    ref = ipm_c.solve_batch_full(tb, X0, P, threads=2)
    x = np.fromfile(str(tmp_path / 'x.f64')).reshape(2, tb.n)
    assert (ref['status'] == 0).all() and np.abs(x - ref['x']).max() < 1e-6
    for b, line in enumerate(out.decode().strip().splitlines()):
        tok = line.split()
        assert int(tok[3]) == 0 and int(tok[5]) == ref['iters'][b]


def test_edge_cases_and_dropin(emu):
    """Empty batch, per-instance bounds, NaN parameters, max_iter, warm start with
    multipliers, Problem.solve()."""
    pr = sc.config1()
    tb = pr.father.tables
    out = pr.problem.solve_batch(np.zeros((0, tb.n)), np.zeros((0, tb.n_par)))
    assert out['x'].shape == (0, tb.n)
    X0, P = sc.instance_data(pr, 3, jitter=0.1, seed=0)
    a = pr.problem.solve_batch(X0, P)
    LB, UB = np.repeat(tb.lbg[None], 3, 0), np.repeat(tb.ubg[None], 3, 0)
    b = pr.problem.solve_batch(X0, P, LB, UB)              # per-instance bounds == shared
    assert np.array_equal(a['x'], b['x'])
    Pn = P.copy()
    Pn[1, 0] = np.nan                                      # NaN parameter: reported, isolated
    r = pr.problem.solve_batch(X0, Pn)
    assert r['status'][1] == 4 and r['status'][0] == 0 and np.array_equal(r['x'][0], a['x'][0])
    pr.problem.set_options({'max_iter': 5})
    try:
        r = pr.problem.solve_batch(X0[:2], P[:2])
    finally:
        pr.problem.set_options({'max_iter': 3000})
    assert np.all(r['status'] == 1) and np.all(r['iters'] == 5)
    w = pr.problem.solve_batch(a['x'], P, lam_g0=a['lam_g'])    # warm start incl. multipliers
    ref = ipm_c.solve_batch_full(tb, a['x'], P, threads=2, lam_g0=a['lam_g'])
    assert np.all(w['status'] == 0) and np.all(w['iters'] < a['iters'])
    assert np.array_equal(w['iters'], ref['iters'])
    pr.solve(0., 0.1)
    assert pr.problem.stats()['return_status'] == 'Solve_Succeeded'


def test_shift_and_sampling_kernels(emu):
    """omg_shift_kernel == T.dot(coeffs) of the seg0 variables, omg_sample_kernel == the
    sampled splines (device pointers are host pointers in the emulation)."""
    pr = sc.config1()
    slv = pr.problem
    X0, P = sc.instance_data(pr, 3, jitter=0.1, seed=4)
    X = slv.solve_batch(X0, P)['x']
    blocks = [(off, shape[0], shape[1], T) for (_, _, off, shape, T) in pr.father.shifted_entries()]
    offs = np.array([b[0] for b in blocks], dtype=np.int32)
    lens = np.array([b[1] for b in blocks], dtype=np.int32)
    ncols = np.array([b[2] for b in blocks], dtype=np.int32)
    Tm = np.concatenate([np.asarray(b[3], dtype=np.float64).reshape(-1) for b in blocks])
    Xs = X.copy()
    assert emu.omg_shift_batch(slv._handle, Xs.shape[0], Xs.ctypes.data, len(blocks), offs.ctypes.data,
                               lens.ctypes.data, ncols.ctypes.data, Tm.ctypes.data, None) == 0
    want = X.copy()
    for off, L, nc, T in blocks:
        for c in range(nc):
            seg = slice(off + c * L, off + (c + 1) * L)
            want[:, seg] = X[:, seg] @ np.asarray(T).T
    assert np.abs(Xs - want).max() < 1e-13
    basis = pr.vehicles[0].basis
    tau = np.linspace(0., 1., 51)
    S0 = np.ascontiguousarray(basis.eval_basis(tau), dtype=np.float64)
    out = np.zeros((X.shape[0], 2 * 51))
    o1, l1, c1, s1 = (np.array([v], dtype=np.int32) for v in (0, 13, 2, 51))
    assert emu.omg_sample_batch(X.shape[0], X.shape[1], X.ctypes.data, 1, o1.ctypes.data, l1.ctypes.data,
                                c1.ctypes.data, s1.ctypes.data, S0.ctypes.data, out.ctypes.data, None) == 0
    for c in range(2):
        assert np.abs(out[:, c * 51:(c + 1) * 51] - X[:, c * 13:(c + 1) * 13] @ S0.T).max() < 1e-13


def test_rk4_kernel(emu):
    """omg_rk4_kernel vs numpy RK4 with the vehicle classes' own ode()."""
    from omg_tools_b200 import Holonomic, Quadrotor, Quadrotor3D

    def rk4(veh, x, U, dt):
        for i in range(U.shape[0] - 1):
            k1 = veh.ode(x, U[i])
            k2 = veh.ode(x + 0.5 * dt * k1, U[i])
            k3 = veh.ode(x + 0.5 * dt * k2, U[i])
            k4 = veh.ode(x + dt * k3, U[i + 1])
            x = x + dt / 6. * (k1 + 2 * k2 + 2 * k3 + k4)
        return x

    rng = np.random.default_rng(5)
    B, steps, dt = 131, 20, 0.01              # more instances than one 128-thread block
    for model, veh, ns, ni in ((0, Holonomic(), 2, 2), (1, Quadrotor3D(0.5), 8, 3), (2, Quadrotor(), 5, 2)):
        x0 = 0.3 * rng.standard_normal((B, ns))
        U = 0.5 * rng.standard_normal((B, steps + 1, ni))
        if ni == 3:
            U[:, :, 0] += 9.81
        out = np.zeros_like(x0)
        assert emu.omg_integrate_rk4(model, B, ns, ni, x0.ctypes.data, U.ctypes.data, dt, steps,
                                     out.ctypes.data, None) == 0
        ref = np.array([rk4(veh, x0[b], U[b], dt) for b in range(B)])
        assert np.abs(out - ref).max() < 1e-12


def test_admm_consensus_kernel(emu):
    """omg_admm_zl_kernel (z-update, multiplier update, residuals of one agent per block)
    vs the reference's KKT-solve formulas (admm.py:149-155, 260-266, 296-303) on BASELINE
    config 3's structure, at a time inside the first knot interval (non-trivial first-knot
    transforms)."""
    _check_consensus_kernel(emu, sc.config3(4, build_solver=False), 0.37)
    # RendezVous: shared blocks of length 1 (terminal positions), identity transforms
    _check_consensus_kernel(emu, sc.config_rendezvous(4, build_solver=False), 0.37)


def _check_consensus_kernel(emu, pr, t):
    rng = np.random.default_rng(7)
    N, nsh, nn, L = pr.N, pr.nsh, pr.n_nghb, pr.L
    rho = 1.3
    x_i, l_i, z_i = (rng.standard_normal((N, nsh)) for _ in range(3))
    x_j, l_ij, z_ij = (rng.standard_normal((N, nn, nsh)) for _ in range(3))
    Tf, Tb = pr.first_knot_transforms(t)
    PzT = np.ascontiguousarray(pr.Pz.T)
    c = np.ascontiguousarray(pr.c)
    zi, zij, li, lij = z_i.copy(), z_ij.copy(), l_i.copy(), l_ij.copy()
    res = np.zeros((N, 3))
    Tf, Tb = np.ascontiguousarray(Tf), np.ascontiguousarray(Tb)
    assert emu.omg_admm_zl_update(N, nsh, nn, L, PzT.ctypes.data, c.ctypes.data, Tf.ctypes.data,
                                  Tb.ctypes.data, rho, x_i.ctypes.data, x_j.ctypes.data,
                                  zi.ctypes.data, zij.ctypes.data, li.ctypes.data, lij.ctypes.data,
                                  res.ctypes.data, None) == 0
    nblk = nsh // L * (1 + nn)
    TF, TB = np.kron(np.eye(nblk), Tf), np.kron(np.eye(nblk), Tb)
    for i in range(N):
        x = TF.dot(np.r_[x_i[i], x_j[i].reshape(-1)])
        l = TF.dot(np.r_[l_i[i], l_ij[i].reshape(-1)])
        f = -(l + rho * x)
        G = -(1. / rho) * pr.A.dot(pr.A.T)
        h = pr._b_of(i) + (1. / rho) * pr.A.dot(f)
        z = TB.dot(-(1. / rho) * (pr.A.T.dot(np.linalg.solve(G, h)) + f))
        assert np.abs(np.r_[zi[i], zij[i].reshape(-1)] - z).max() < 1e-9
        l_new = np.r_[l_i[i], l_ij[i].reshape(-1)] + rho * (np.r_[x_i[i], x_j[i].reshape(-1)] - z)
        assert np.abs(np.r_[li[i], lij[i].reshape(-1)] - l_new).max() < 1e-9
        e1 = TF.dot(np.r_[x_i[i], x_j[i].reshape(-1)] - z)
        e2 = TF.dot(z - np.r_[z_i[i], z_ij[i].reshape(-1)])
        pri, dri = e1.dot(e1), rho * e2.dot(e2)
        assert np.allclose(res[i], [pri, dri, rho * pri + dri], rtol=1e-9, atol=1e-12)


def test_results_do_not_depend_on_the_thread_schedule(emu, monkeypatch):
    """Race check without a GPU: the emulator resumes the runnable fibers of a block in
    forward, reverse or random order between barriers (OMG_EMU_SCHED).  A read that no
    barrier separates from another thread's write would change the result with the order;
    the standard kernel, the XL kernel and its cross / mid-mid Hessian gathers give
    bit-identical solutions and multipliers under every schedule.  (compute-sanitizer
    racecheck on the GPU, tools/sanitize.py, covers the kernel paths on the device.)"""
    cases = []
    for name, B in (('config1', 2), ('config2', 1), ('config_dubins_plain', 1), ('config_bicycle', 1)):
        pr = getattr(sc, name)()
        X0, P = sc.instance_data(pr, B, jitter=0.1, seed=1)
        if name == 'config_bicycle':
            X0[:, :7] = 0.3
        cases.append((pr, X0, P))
    results = {}
    for sched in ('forward', 'reverse', 'random:1'):
        monkeypatch.setenv('OMG_EMU_SCHED', sched)
        results[sched] = [pr.problem.solve_batch(X0, P) for pr, X0, P in cases]
    for sched in ('reverse', 'random:1'):
        for a, b in zip(results['forward'], results[sched]):
            assert np.array_equal(a['iters'], b['iters']) and (a['status'] == 0).all()
            assert np.array_equal(a['x'], b['x']) and np.array_equal(a['lam_g'], b['lam_g'])


def test_device_pointer_api_on_cpu_tensors(emu):
    """solve_batch_device / shift_batch_device with CPU tensors are accepted by the emulation
    library only; the runner of the formation ADMM then follows the sequential oracle."""
    import torch
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    from oracle.admm_ref import ADMMOracle
    assert hasattr(emu, 'omg_is_emulation')
    run = FormationADMMRunner(sc.config3(4), device=torch.device('cpu'))
    orc = ADMMOracle(sc.config3(4, build_solver=False))
    for it in range(4):
        rg, ro = run.dual_update(0.), orc.dual_update(0.)
        st, _ = run.status()
        assert np.all(st == 0) and np.all(orc.status == 0)
        assert np.abs(run.x_i.numpy() - orc.x_i).max() < 1e-4, it
        assert np.abs(run.z_i.numpy() - orc.z_i).max() < 1e-4
        assert abs(rg[0] - ro[0]) < 1e-3 * max(1., ro[0])


def test_side_by_side_formations_equal_the_single_formation(emu):
    """FormationADMMRunner(formations=F): F copies of the formation advance in ONE x-update
    launch / consensus kernel / exchange per iteration.  Without spread every copy repeats the
    single formation bit for bit (the neighbour offsets keep the copies apart); with spread the
    copies start from different guesses and each still converges on its own residuals."""
    import torch
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    single = FormationADMMRunner(sc.config3(4), device=torch.device('cpu'))
    multi = FormationADMMRunner(sc.config3(4), device=torch.device('cpu'), formations=3)
    for it in range(3):
        rs, rm = single.dual_update(0.), multi.dual_update(0.)
    for key in ('x_i', 'z_i', 'l_i', 'z_ji'):
        a, b = getattr(single, key), getattr(multi, key)
        for f in range(3):
            assert torch.equal(a, b[4 * f:4 * f + 4]), (key, f)
    per = multi.formation_residuals()
    assert per.shape == (3, 3) and np.allclose(per, np.array(rs)[None, :], rtol=1e-12)
    assert np.isclose(rm[0] ** 2, 3 * rs[0] ** 2, rtol=1e-12)      # the global sum covers all copies
    spread = FormationADMMRunner(sc.config3(4), device=torch.device('cpu'), formations=2, spread=0.05)
    for it in range(3):
        spread.dual_update(0.)
    assert (spread.status()[0] == 0).all()
    assert not torch.equal(spread.x_i[:4], spread.x_i[4:])


def test_dual_decomposition_runner_follows_the_oracle(emu):
    """problems/dualdecomposition.py through FormationDDRunner (one batched xz-update, device-side
    multiplier update, the two exchanges) against the sequential DDOracle (reference
    dualdecomposition.py:279-314), iteration by iteration and across a knot crossing."""
    import torch
    from omg_tools_b200.problems.admm_gpu import FormationDDRunner
    from oracle.admm_ref import DDOracle
    run = FormationDDRunner(sc.config_formation_dd(4, options={'rho': 0.02}), device=torch.device('cpu'))
    orc = DDOracle(sc.config_formation_dd(4, build_solver=False, options={'rho': 0.02}))
    for it, t in enumerate([0., 0., 0.5, 1.0, 1.0]):          # knot_time = 1: the fourth call shifts
        rg, ro = run.dual_update(t), orc.dual_update(t)
        st, its = run.status()
        assert np.all(st == 0) and np.all(orc.status == 0)
        assert np.array_equal(its, orc.iters), (it, its, orc.iters)
        for key in ('x_i', 'z_ij', 'l_ij', 'l_ji', 'x_j'):
            assert np.abs(getattr(run, key).numpy() - getattr(orc, key)).max() < 1e-6, (it, key)
        assert abs(rg - ro) < 1e-6 * max(1., ro)


def _admm_rank(rank, world, port, out):
    import torch
    import torch.distributed as dist
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    emu_support.activate()
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    run = FormationADMMRunner(sc.config3(8, rank=rank, world=world), rank=rank, world=world,
                              device=torch.device('cpu'))
    hist = [run.dual_update(0.) for _ in range(4)]
    torch.save({'x_i': run.x_i, 'z_i': run.z_i, 'l_i': run.l_i, 'hist': hist, 'lo': run.lo},
               os.path.join(out, 'r%d.pt' % rank))
    dist.barrier()
    dist.destroy_process_group()


def test_formation_admm_two_ranks_gloo_through_the_emulated_kernels(emu, tmp_path):
    """BASELINE config 3's multi-rank path end to end on the CPU: 8 agents sharded over two
    processes (gloo), each running its batched x-update and consensus kernel in the kernel
    emulation, neighbour exchange and residual all-reduce over the process group -- the
    sharded run reproduces the single-process run of all agents bit for bit."""
    import torch
    import torch.multiprocessing as mp
    from omg_tools_b200.problems.admm_gpu import FormationADMMRunner
    port = 29900 + (os.getpid() % 90)
    mp.spawn(_admm_rank, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    single = FormationADMMRunner(sc.config3(8), device=torch.device('cpu'))
    hist = [single.dual_update(0.) for _ in range(4)]
    for rank in range(2):
        d = torch.load(os.path.join(str(tmp_path), 'r%d.pt' % rank))
        lo = d['lo']
        assert lo == 4 * rank
        for key in ('x_i', 'z_i', 'l_i'):
            assert torch.equal(d[key], getattr(single, key)[lo:lo + 4]), key
        assert np.allclose(d['hist'], hist, rtol=1e-12, atol=0.)


def _dd_rank(rank, world, port, out):
    import torch
    import torch.distributed as dist
    os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    emu_support.activate()
    from omg_tools_b200.problems.admm_gpu import FormationDDRunner
    run = FormationDDRunner(sc.config_formation_dd(8, options={'rho': 0.02}, rank=rank, world=world),
                            rank=rank, world=world, device=torch.device('cpu'))
    hist = [run.dual_update(0.) for _ in range(3)]
    torch.save({'x_i': run.x_i, 'z_ij': run.z_ij, 'l_ij': run.l_ij, 'l_ji': run.l_ji, 'hist': hist, 'lo': run.lo},
               os.path.join(out, 'r%d.pt' % rank))
    dist.barrier()
    dist.destroy_process_group()


def test_dual_decomposition_two_ranks_gloo(emu, tmp_path):
    """The multi-rank path of the dual decomposition on the CPU: 8 agents sharded over two
    processes (gloo), neighbour exchange of x_j and of the multipliers l_ji and the residual
    all-reduce over the process group -- the sharded run reproduces the single-process run of
    all agents bit for bit."""
    import torch
    import torch.multiprocessing as mp
    from omg_tools_b200.problems.admm_gpu import FormationDDRunner
    port = 29700 + (os.getpid() % 90)
    mp.spawn(_dd_rank, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    single = FormationDDRunner(sc.config_formation_dd(8, options={'rho': 0.02}), device=torch.device('cpu'))
    hist = [single.dual_update(0.) for _ in range(3)]
    for rank in range(2):
        d = torch.load(os.path.join(str(tmp_path), 'r%d.pt' % rank))
        lo = d['lo']
        assert lo == 4 * rank
        for key in ('x_i', 'z_ij', 'l_ij', 'l_ji'):
            assert torch.equal(d[key], getattr(single, key)[lo:lo + 4]), key
        assert np.allclose(d['hist'], hist, rtol=1e-12, atol=0.)


def test_batched_receding_horizon_config5_through_the_emulated_kernels(emu):
    """BASELINE config 5 (revolving door): the batched device-resident MPC loop
    (execution/batch_mpc.py: solve, device-side prediction from sampled splines, knot shift)
    equals the reference-style sequential loop Problem.predict/solve/store/simulate, step by
    step through the first knot crossing -- run on CPU tensors in the kernel emulation."""
    from omg_tools_b200.execution.batch_mpc import BatchMPC
    seq = sc.config5()
    seq.initialize(0.)
    import torch
    bat = BatchMPC(sc.config5(), batch=2, update_time=0.1, device=torch.device('cpu'))
    t, dt = 0., 0.1
    for k in range(12):                      # crosses the first knot at t = 1.0
        seq.predict(t, dt, 0.01)
        seq.solve(t, dt)
        bat.step()
        Xb = bat.X.numpy()
        xs = seq.father.get_variables().cat
        assert seq.problem.stats()['return_status'] == 'Solve_Succeeded'
        assert np.all(bat.history['status'][-1] == 0)
        assert np.abs(Xb - xs[None]).max() < 1e-6, k
        seq.store(t, dt, 0.01)
        seq.simulate(t, dt, 0.01)
        t = np.round(t + dt, 6)
    assert np.abs(bat.state[0] - seq.vehicles[0].signals['state'][:, -1]).max() < 1e-6


def test_changed_equality_pattern_raises(emu):
    """Bounds that turn an equality row into a free row: a clear error from the reference-facing
    call instead of Error_In_Step_Computation with the stale x (ADVICE r1)."""
    pr = sc.config1()
    tb = pr.father.tables
    X0, P = sc.instance_data(pr, 1)
    lb, ub = tb.lbg.copy(), tb.ubg.copy()
    k = int(np.nonzero(lb == ub)[0][0])
    lb[k], ub[k] = -np.inf, np.inf
    with pytest.raises(ValueError, match='equality pattern'):
        pr.problem(x0=X0[0], p=P[0], lbg=lb, ubg=ub)
    # the batched entry reports it per instance
    res = pr.problem.solve_batch(X0, P, lb, ub)
    assert res['status'][0] == 3 and res['iters'][0] == 0
