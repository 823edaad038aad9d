"""ctypes binding of libomgb200.so and the solver object that stands where the
reference holds ``nlpsol('solver','ipopt',...)``.

``B200Solver`` keeps the reference's call contract (problem.py:113-128):

    result = problem(x0=var, p=par, lbg=lb, ubg=ub)   # -> {'x','lam_g','f'}
    problem.stats()['return_status']                  # IPOPT status strings

and adds the batched entry points ``solve_batch`` (host numpy arrays; H2D/D2H
inside the C call) and ``solve_batch_device`` (torch CUDA tensors, zero-copy).
There is no CPU fallback: if the shared library or a CUDA device is missing the
constructor raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), 'csrc', 'libomgb200.so')

STATUS_STRINGS = {
    0: 'Solve_Succeeded', 1: 'Maximum_Iterations_Exceeded',
    2: 'Restoration_Failed', 3: 'Error_In_Step_Computation',
    4: 'Invalid_Number_Detected', 5: 'Infeasible_Problem_Detected'}

ABI_VERSION = 6
FEAS_STEPS = 30      # option 'feas_steps': LM steps of the feasibility phase (0 = off)

_i32p = C.POINTER(C.c_int32)
_f64p = C.POINTER(C.c_double)


class _TermList(C.Structure):
    _fields_ = [('n_out', C.c_int32), ('n_terms', C.c_int32), ('width', C.c_int32),
                ('ptr', _i32p), ('coef', _f64p), ('cidx', _i32p), ('xi', _i32p),
                ('lrow', _i32p)]


class _Tables(C.Structure):
    _fields_ = [
        ('abi_version', C.c_int32),
        ('n', C.c_int32), ('m', C.c_int32), ('n_par', C.c_int32),
        ('n_v', C.c_int32), ('degree', C.c_int32),
        ('n_tape', C.c_int32), ('n_tape_terms', C.c_int32), ('n_levels', C.c_int32),
        ('tape_func', _i32p), ('tape_ptr', _i32p), ('tape_coef', _f64p),
        ('tape_fac', _i32p), ('level_ptr', _i32p),
        ('G', _TermList), ('F', _TermList), ('DF', _TermList), ('J', _TermList),
        ('W', _TermList),
        ('nnz_j', C.c_int32), ('jrow', _i32p), ('jcol', _i32p), ('jrow_ptr', _i32p),
        ('n_mid', C.c_int32), ('nnz_jx', C.c_int32), ('n_jp', C.c_int32), ('n_mu', C.c_int32),
        ('jp_ptr', _i32p), ('jp_a', _i32p), ('jp_c', _i32p),
        ('mu_ptr', _i32p), ('mu_row', _i32p), ('mu_slot', _i32p),
        ('nnz_w', C.c_int32), ('wrow', _i32p), ('wcol', _i32p), ('w2h', _i32p),
        ('nnz_h', C.c_int32), ('n_hp', C.c_int32),
        ('hrow', _i32p), ('hcol', _i32p), ('hp_ptr', _i32p),
        ('hp_s1', _i32p), ('hp_s2', _i32p), ('hp_row', _i32p),
        ('lbg', _f64p), ('ubg', _f64p),
        ('kkt_n', C.c_int32), ('kkt_n_eq', C.c_int32), ('env_size', C.c_int32),
        ('n_panel_rows', C.c_int32), ('max_panel_rows', C.c_int32),
        ('kkt_eq_rows', _i32p), ('kkt_pos_var', _i32p), ('kkt_pos_eq', _i32p),
        ('kkt_sign', _i32p), ('env_first', _i32p), ('env_ptr', _i32p),
        ('kkt_hdst', _i32p), ('kkt_jdst', _i32p), ('kkt_diag', _i32p),
        ('kkt_panel_ptr', _i32p), ('kkt_panel_rows', _i32p),
        ('nnz_wx', C.c_int32), ('n_xq', C.c_int32), ('n_xp', C.c_int32),
        ('xq_h', _i32p), ('xq_ptr', _i32p), ('xq_w', _i32p), ('xq_a', _i32p), ('xq_b', _i32p)]


class _Options(C.Structure):
    _fields_ = [('tol', C.c_double), ('constr_viol_tol', C.c_double),
                ('dual_inf_tol', C.c_double), ('compl_inf_tol', C.c_double),
                ('mu_init', C.c_double), ('bound_push', C.c_double),
                ('bound_frac', C.c_double), ('mult_bound_push', C.c_double),
                ('bound_relax_factor', C.c_double),
                ('scaling_max_gradient', C.c_double),
                ('max_iter', C.c_int32), ('trace', C.c_int32),
                ('max_restarts', C.c_int32), ('soft_resto', C.c_int32),
                ('restart_mu', C.c_double), ('restart_push', C.c_double),
                ('inertia_mode', C.c_int32), ('reserved', C.c_int32)]


# include/omg_b200.h omg_mpc_desc: (name, kind), kind 'i' int32, 'd' float64, 'I' int32 array,
# 'D' float64 array; the records of an MPC file carry the same names
MPC_FIELDS = [('n', 'i'), ('n_par', 'i'), ('n_dim', 'i'), ('spl_offset', 'i'), ('L', 'i'), ('degree', 'i'),
              ('knots', 'D'), ('horizon', 'd'), ('knot_time', 'd'), ('update_time', 'd'), ('sample_time', 'd'),
              ('p_state0', 'i'), ('p_input0', 'i'), ('p_poseT', 'i'), ('p_t', 'i'), ('p_T', 'i'),
              ('n_obs', 'i'), ('obs_kind', 'I'), ('obs_off', 'I'), ('n_shift', 'i'), ('shift_off', 'I'),
              ('shift_len', 'I'), ('shift_ncol', 'I'), ('shift_T', 'D'), ('x_template', 'D'), ('p_template', 'D')]
_CTYPE = {'i': C.c_int32, 'd': C.c_double, 'I': _i32p, 'D': _f64p}


class _MpcDesc(C.Structure):
    _fields_ = [(name, _CTYPE[kind]) for name, kind in MPC_FIELDS]


# include/omg_b200.h omg_mpc_freeT_desc, in the same notation
MPC_FREET_FIELDS = [('n', 'i'), ('n_par', 'i'), ('n_dim', 'i'), ('spl_offset', 'i'), ('L', 'i'), ('degree', 'i'),
                    ('knots', 'D'), ('update_time', 'd'), ('sample_time', 'd'), ('stop_tol', 'd'), ('t_index', 'i'),
                    ('p_state0', 'i'), ('p_input0', 'i'), ('p_poseT', 'i'), ('n_obs', 'i'), ('obs_kind', 'I'),
                    ('obs_off', 'I'), ('n_blocks', 'i'), ('blk_off', 'I'), ('blk_len', 'I'), ('blk_ncol', 'I'),
                    ('blk_degree', 'I'), ('blk_knots', 'D'), ('x_template', 'D'), ('p_template', 'D')]


class _MpcFreeTDesc(C.Structure):
    _fields_ = [(name, _CTYPE[kind]) for name, kind in MPC_FREET_FIELDS]


# include/omg_b200.h omg_mpc_obstacles_desc, in the same notation
MPC_OBSTACLE_FIELDS = [('n_obs', 'i'), ('chk_off', 'I'), ('chk_len', 'I'), ('rad_off', 'I'), ('rad_len', 'I'),
                       ('row_off', 'I'), ('row_len', 'I')]


class _MpcObstaclesDesc(C.Structure):
    _fields_ = [(name, _CTYPE[kind]) for name, kind in MPC_OBSTACLE_FIELDS]


MPC_PREDICTION = {'ideal': 0, 'integrate': 1}
MPC_STOPPED = -1        # status of an instance that was not solved because it has stopped

EXPORTS = ['omg_abi_version', 'omg_last_error', 'omg_default_options',
           'omg_problem_create', 'omg_problem_destroy', 'omg_set_options',
           'omg_solve_batch', 'omg_solve_batch_host', 'omg_shift_batch',
           'omg_get_trace', 'omg_get_info', 'omg_structure_info', 'omg_envelope_layout', 'omg_last_timing',
           'omg_admm_zl_update', 'omg_sample_batch', 'omg_tables_read',
           'omg_tables_free', 'omg_integrate_rk4', 'omg_feas_batch', 'omg_feas_batch_host',
           'omg_comm_unique_id', 'omg_comm_create', 'omg_comm_destroy', 'omg_admm_exchange_x',
           'omg_admm_zl_update_dist', 'omg_closed_loop_step', 'omg_closed_loop_step_der',
           'omg_shift_free_batch', 'omg_eval_batch', 'omg_closed_loop_step_free', 'omg_closed_loop_step_fleet',
           'omg_mpc_read', 'omg_mpc_free_desc', 'omg_mpc_create', 'omg_mpc_destroy', 'omg_mpc_update',
           'omg_mpc_update_host', 'omg_mpc_recover', 'omg_mpc_time', 'omg_mpc_last_problem',
           'omg_mpc_freet_read', 'omg_mpc_freet_release', 'omg_mpc_create_freet', 'omg_mpc_motion_time',
           'omg_solve_batch_rows', 'omg_mpc_obstacles_read', 'omg_mpc_obstacles_release',
           'omg_mpc_attach_obstacles', 'omg_mpc_set_obstacles', 'omg_mpc_set_obstacles_host']

_lib = None


def load_library():
    """Load libomgb200.so (built by __graft_entry__.build() / csrc/Makefile).  There is exactly
    one library and no fallback: a missing build raises."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'libomgb200.so not found at %s: build it with '
            '`python -c "import __graft_entry__ as g; g.build()"` '
            '(there is no CPU fallback)' % LIB_PATH)
    _lib = bind(C.CDLL(LIB_PATH))
    return _lib


def bind(lib):
    """Declare the C signatures of include/omg_b200.h on a loaded library object."""
    lib.omg_abi_version.restype = C.c_int
    lib.omg_last_error.restype = C.c_char_p
    lib.omg_default_options.argtypes = [C.POINTER(_Options)]
    lib.omg_default_options.restype = None
    lib.omg_problem_create.argtypes = [C.POINTER(_Tables), C.POINTER(_Options), C.c_int]
    lib.omg_problem_create.restype = C.c_void_p
    lib.omg_problem_destroy.argtypes = [C.c_void_p]
    lib.omg_problem_destroy.restype = None
    lib.omg_set_options.argtypes = [C.c_void_p, C.POINTER(_Options)]
    vp = C.c_void_p
    lib.omg_solve_batch.argtypes = [vp, C.c_int32, vp, vp, vp, vp, C.c_int32, vp,
                                    vp, vp, vp, vp, vp, vp]
    lib.omg_solve_batch_host.argtypes = [vp, C.c_int32, vp, vp, vp, vp, C.c_int32,
                                         vp, vp, vp, vp, vp, vp]
    lib.omg_shift_batch.argtypes = [vp, C.c_int32, vp, C.c_int32, vp, vp, vp, vp, vp]
    lib.omg_feas_batch.argtypes = [vp, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp, vp]
    lib.omg_feas_batch_host.argtypes = [vp, C.c_int32, vp, vp, vp, vp, C.c_int32, C.c_int32, vp, vp, vp]
    lib.omg_get_trace.argtypes = [vp, vp, C.c_int32]
    lib.omg_get_info.argtypes = [vp] + [_i32p] * 6
    lib.omg_structure_info.argtypes = [vp]
    lib.omg_structure_info.restype = C.c_char_p
    lib.omg_envelope_layout.argtypes = [vp]
    lib.omg_envelope_layout.restype = C.c_char_p
    lib.omg_comm_unique_id.argtypes = [vp]
    lib.omg_comm_create.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
    lib.omg_comm_create.restype = C.c_void_p
    lib.omg_comm_destroy.argtypes = [vp]
    lib.omg_comm_destroy.restype = None
    lib.omg_admm_exchange_x.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp, vp]
    lib.omg_admm_zl_update_dist.argtypes = [vp] + [C.c_int32] * 4 + [vp] * 4 + [C.c_double] + [vp] * 13
    lib.omg_last_timing.argtypes = [vp, C.POINTER(C.c_float), _i32p]
    lib.omg_admm_zl_update.argtypes = [C.c_int32] * 4 + [vp] * 4 + [C.c_double] + [vp] * 8
    lib.omg_sample_batch.argtypes = [C.c_int32, C.c_int32, vp, C.c_int32] + [vp] * 7
    lib.omg_integrate_rk4.argtypes = [C.c_int32] * 4 + [vp, vp, C.c_double, C.c_int32, vp, vp]
    lib.omg_closed_loop_step.argtypes = ([C.c_int32] * 5 + [vp, C.c_int32, C.c_int32, vp, vp, C.c_double,
                                         C.c_int32, C.c_double, C.c_int32, C.c_int32, vp, vp, vp,
                                         C.c_uint64, C.c_int32] + [vp] * 8)
    lib.omg_closed_loop_step_der.argtypes = ([C.c_int32] * 5 + [vp, C.c_int32, C.c_int32, C.c_int32, vp,
                                             C.c_double, C.c_int32, C.c_double, C.c_int32, C.c_int32,
                                             vp, vp, vp, C.c_uint64, C.c_int32] + [vp] * 8)
    lib.omg_closed_loop_step_fleet.argtypes = ([C.c_int32] * 6 + [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp,
                                               C.c_double, C.c_int32, C.c_double, C.c_int32, C.c_int32,
                                               vp, vp, vp, C.c_uint64, C.c_int32] + [vp] * 8)
    lib.omg_closed_loop_step_free.argtypes = ([C.c_int32] * 5 + [vp] + [C.c_int32] * 4 + [vp, C.c_int32, C.c_int32,
                                              vp, vp, C.c_double, C.c_int32, C.c_double, C.c_int32,
                                              vp, vp, vp, C.c_uint64, C.c_int32] + [vp] * 8)
    lib.omg_shift_free_batch.argtypes = [vp, C.c_int32, vp, C.c_int32, C.c_double, vp, C.c_int32] + [vp] * 6
    lib.omg_eval_batch.argtypes = [C.c_int32, C.c_int32, vp, C.c_int32] + [vp] * 5 + [C.c_int32, vp, vp, C.c_int32,
                                                                                    vp, vp]
    lib.omg_mpc_read.argtypes = [C.c_char_p]
    lib.omg_mpc_read.restype = C.POINTER(_MpcDesc)
    lib.omg_mpc_free_desc.argtypes = [C.POINTER(_MpcDesc)]
    lib.omg_mpc_free_desc.restype = None
    lib.omg_mpc_create.argtypes = [vp, C.POINTER(_MpcDesc), C.c_int32, C.c_int32, C.c_int32]
    lib.omg_mpc_create.restype = C.c_void_p
    lib.omg_mpc_destroy.argtypes = [vp]
    lib.omg_mpc_destroy.restype = None
    lib.omg_mpc_update.argtypes = [vp] * 9
    lib.omg_mpc_update_host.argtypes = [vp] * 8
    lib.omg_mpc_recover.argtypes = [vp, vp]
    lib.omg_mpc_time.argtypes = [vp, vp]
    lib.omg_mpc_last_problem.argtypes = [vp] * 4
    lib.omg_mpc_freet_read.argtypes = [C.c_char_p]
    lib.omg_mpc_freet_read.restype = C.POINTER(_MpcFreeTDesc)
    lib.omg_mpc_freet_release.argtypes = [C.POINTER(_MpcFreeTDesc)]
    lib.omg_mpc_freet_release.restype = None
    lib.omg_mpc_create_freet.argtypes = [vp, C.POINTER(_MpcFreeTDesc), C.c_int32, C.c_int32, C.c_int32]
    lib.omg_mpc_create_freet.restype = C.c_void_p
    lib.omg_mpc_motion_time.argtypes = [vp] * 3
    lib.omg_mpc_obstacles_read.argtypes = [C.c_char_p]
    lib.omg_mpc_obstacles_read.restype = C.POINTER(_MpcObstaclesDesc)
    lib.omg_mpc_obstacles_release.argtypes = [C.POINTER(_MpcObstaclesDesc)]
    lib.omg_mpc_obstacles_release.restype = None
    lib.omg_mpc_attach_obstacles.argtypes = [vp, C.POINTER(_MpcObstaclesDesc)]
    lib.omg_mpc_set_obstacles.argtypes = [vp] * 4
    lib.omg_mpc_set_obstacles_host.argtypes = [vp] * 3
    lib.omg_solve_batch_rows.argtypes = [vp, C.c_int32, vp, vp, vp, vp, C.c_int32, vp] + [vp] * 8
    lib.omg_tables_read.argtypes = [C.c_char_p]
    lib.omg_tables_read.restype = C.POINTER(_Tables)
    lib.omg_tables_free.argtypes = [C.POINTER(_Tables)]
    lib.omg_tables_free.restype = None
    return lib


def _ptr(arr, typ):
    return arr.ctypes.data_as(typ)


def _check_device_tensors(tensors, lib=None):
    """Device-pointer API: contiguous float64 CUDA tensors, nothing else."""
    import torch
    for t in tensors:
        if t.dtype != torch.float64 or not t.is_cuda or not t.is_contiguous():
            raise ValueError('expected contiguous float64 CUDA tensors')
    return True


def _check_int_tensors(tensors):
    import torch
    for t in tensors:
        if t.dtype != torch.int32 or not t.is_cuda or not t.is_contiguous():
            raise ValueError('expected contiguous int32 CUDA tensors')


def _stream_handle(on_gpu, device, stream):
    import torch
    if not on_gpu:
        return None
    if stream is None:
        stream = torch.cuda.current_stream(device)
    return C.c_void_p(stream.cuda_stream)


class _Keep(object):
    """Owns contiguous numpy copies referenced by a ctypes struct."""

    def __init__(self):
        self.arrays = []

    def i32(self, a):
        a = np.ascontiguousarray(a, dtype=np.int32)
        self.arrays.append(a)
        return _ptr(a, _i32p)

    def f64(self, a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        self.arrays.append(a)
        return _ptr(a, _f64p)


def pack_tables(tb):
    """NLPTables -> (ctypes omg_tables, keep-alive object)."""
    keep = _Keep()

    def tl(t, with_lrow=False):
        s = _TermList()
        s.n_out, s.n_terms, s.width = t.n_out, t.n_terms, t.width
        s.ptr, s.coef = keep.i32(t.ptr), keep.f64(t.coef)
        s.cidx, s.xi = keep.i32(t.cidx), keep.i32(t.xi.reshape(-1))
        s.lrow = keep.i32(t.lrow) if with_lrow else None
        return s

    T = _Tables()
    T.abi_version = ABI_VERSION
    T.n, T.m, T.n_par, T.n_v, T.degree = tb.n, tb.m, tb.n_par, tb.n_v, tb.degree
    T.n_tape, T.n_tape_terms = len(tb.tape_func), len(tb.tape_coef)
    T.n_levels = len(tb.level_ptr) - 1
    T.tape_func, T.tape_ptr = keep.i32(tb.tape_func), keep.i32(tb.tape_ptr)
    T.tape_coef, T.tape_fac = keep.f64(tb.tape_coef), keep.i32(tb.tape_fac.reshape(-1))
    T.level_ptr = keep.i32(tb.level_ptr)
    T.G, T.F, T.DF, T.J = tl(tb.G), tl(tb.F), tl(tb.DF), tl(tb.J)
    T.W = tl(tb.W, True)
    T.nnz_j = tb.nnz_j
    T.jrow, T.jcol, T.jrow_ptr = keep.i32(tb.jrow), keep.i32(tb.jcol), keep.i32(tb.jrow_ptr)
    T.n_mid = getattr(tb, 'n_mid', 0)
    T.nnz_jx = getattr(tb, 'nnz_jx', tb.nnz_j)
    if T.n_mid:
        T.n_jp, T.n_mu = len(tb.jp_a), len(tb.mu_row)
        T.jp_ptr, T.jp_a, T.jp_c = keep.i32(tb.jp_ptr), keep.i32(tb.jp_a), keep.i32(tb.jp_c)
        T.mu_ptr, T.mu_row, T.mu_slot = (keep.i32(tb.mu_ptr), keep.i32(tb.mu_row),
                                         keep.i32(tb.mu_slot))
    T.nnz_w = tb.nnz_w
    T.wrow, T.wcol, T.w2h = keep.i32(tb.wrow), keep.i32(tb.wcol), keep.i32(tb.w2h)
    T.nnz_h, T.n_hp = tb.nnz_h, len(tb.hp_s1)
    T.hrow, T.hcol, T.hp_ptr = keep.i32(tb.hrow), keep.i32(tb.hcol), keep.i32(tb.hp_ptr)
    T.hp_s1, T.hp_s2, T.hp_row = keep.i32(tb.hp_s1), keep.i32(tb.hp_s2), keep.i32(tb.hp_row)
    T.lbg, T.ubg = keep.f64(tb.lbg), keep.f64(tb.ubg)
    T.kkt_n, T.kkt_n_eq, T.env_size = tb.kkt_n, tb.kkt_n_eq, tb.env_size
    T.n_panel_rows, T.max_panel_rows = len(tb.kkt_panel_rows), tb.kkt_max_panel_rows
    T.kkt_eq_rows, T.kkt_pos_var = keep.i32(tb.kkt_eq_rows), keep.i32(tb.kkt_pos_var)
    T.kkt_pos_eq, T.kkt_sign = keep.i32(tb.kkt_pos_eq), keep.i32(tb.kkt_sign)
    T.env_first, T.env_ptr = keep.i32(tb.env_first), keep.i32(tb.env_ptr)
    T.kkt_hdst, T.kkt_jdst = keep.i32(tb.kkt_hdst), keep.i32(tb.kkt_jdst)
    T.kkt_diag = keep.i32(tb.kkt_diag)
    T.kkt_panel_ptr = keep.i32(tb.kkt_panel_ptr)
    T.kkt_panel_rows = keep.i32(tb.kkt_panel_rows)
    T.nnz_wx = getattr(tb, 'nnz_wx', 0)
    if T.nnz_wx:
        T.n_xq, T.n_xp = tb.n_xq, len(tb.xq_w)
        T.xq_h, T.xq_ptr = keep.i32(tb.xq_h), keep.i32(tb.xq_ptr)
        T.xq_w, T.xq_a, T.xq_b = keep.i32(tb.xq_w), keep.i32(tb.xq_a), keep.i32(tb.xq_b)
    return T, keep


_NO_EFFECT_IPOPT_OPTIONS = frozenset([
    'print_level', 'print_time', 'sb', 'file_print_level', 'output_file',
    'print_timing_statistics', 'print_user_options', 'linear_solver',
    'warm_start_init_point', 'fixed_variable_treatment', 'ma57_automatic_scaling',
    'hessian_approximation', 'verbose'])

_TERMLIST_FIELDS = ('G', 'F', 'DF', 'J', 'W')


def _table_records(tb):
    """[(name, dtype, array)] in the order of include/omg_b200.h; dtype 0 =
    int32, 1 = float64; scalars are int32 arrays of length 1."""
    T, keep = pack_tables(tb)
    rec = []

    def scalar(name, v):
        rec.append((name, 0, np.array([v], dtype=np.int32)))

    def arr(name, a, dtype):
        a = np.ascontiguousarray(a, dtype=np.float64 if dtype else np.int32).reshape(-1)
        rec.append((name, dtype, a))

    for f in ('n', 'm', 'n_par', 'n_v', 'degree', 'n_tape', 'n_tape_terms', 'n_levels'):
        scalar(f, getattr(T, f))
    arr('tape_func', tb.tape_func, 0), arr('tape_ptr', tb.tape_ptr, 0)
    arr('tape_coef', tb.tape_coef, 1), arr('tape_fac', tb.tape_fac, 0)
    arr('level_ptr', tb.level_ptr, 0)
    for l in _TERMLIST_FIELDS:
        t = getattr(tb, l)
        scalar(l + '.n_out', t.n_out), scalar(l + '.n_terms', t.n_terms)
        scalar(l + '.width', t.width)
        arr(l + '.ptr', t.ptr, 0), arr(l + '.coef', t.coef, 1), arr(l + '.cidx', t.cidx, 0)
        arr(l + '.xi', t.xi, 0)
        if l == 'W':
            arr(l + '.lrow', t.lrow, 0)
    scalar('nnz_j', tb.nnz_j)
    arr('jrow', tb.jrow, 0), arr('jcol', tb.jcol, 0), arr('jrow_ptr', tb.jrow_ptr, 0)
    n_mid = getattr(tb, 'n_mid', 0)
    scalar('n_mid', n_mid), scalar('nnz_jx', getattr(tb, 'nnz_jx', tb.nnz_j))
    scalar('n_jp', len(tb.jp_a) if n_mid else 0), scalar('n_mu', len(tb.mu_row) if n_mid else 0)
    empty = np.zeros(0, dtype=np.int32)
    for f in ('jp_ptr', 'jp_a', 'jp_c', 'mu_ptr', 'mu_row', 'mu_slot'):
        arr(f, getattr(tb, f) if n_mid else empty, 0)
    scalar('nnz_w', tb.nnz_w)
    arr('wrow', tb.wrow, 0), arr('wcol', tb.wcol, 0), arr('w2h', tb.w2h, 0)
    scalar('nnz_h', tb.nnz_h), scalar('n_hp', len(tb.hp_s1))
    for f in ('hrow', 'hcol', 'hp_ptr', 'hp_s1', 'hp_s2', 'hp_row'):
        arr(f, getattr(tb, f), 0)
    arr('lbg', tb.lbg, 1), arr('ubg', tb.ubg, 1)
    scalar('kkt_n', tb.kkt_n), scalar('kkt_n_eq', tb.kkt_n_eq), scalar('env_size', tb.env_size)
    scalar('n_panel_rows', len(tb.kkt_panel_rows)), scalar('max_panel_rows', tb.kkt_max_panel_rows)
    for f in ('kkt_eq_rows', 'kkt_pos_var', 'kkt_pos_eq', 'kkt_sign', 'env_first', 'env_ptr',
              'kkt_hdst', 'kkt_jdst', 'kkt_diag', 'kkt_panel_ptr', 'kkt_panel_rows'):
        arr(f, getattr(tb, f), 0)
    nnz_wx = getattr(tb, 'nnz_wx', 0)
    scalar('nnz_wx', nnz_wx), scalar('n_xq', tb.n_xq if nnz_wx else 0)
    scalar('n_xp', len(tb.xq_w) if nnz_wx else 0)
    for f in ('xq_h', 'xq_ptr', 'xq_w', 'xq_a', 'xq_b'):
        arr(f, getattr(tb, f) if nnz_wx else empty, 0)
    del keep
    return rec


def save_tables(tb, path):
    """Write the lowered NLP to a table file (include/omg_b200.h:
    omg_tables_read) -- the deployable artefact for native callers, in place
    of the nlp.c/.so bundle of the reference's exporter."""
    import struct
    rec = _table_records(tb)
    with open(path, 'wb') as fp:
        fp.write(b'OMGTBL\0\0')
        fp.write(struct.pack('<ii', ABI_VERSION, len(rec)))
        for name, dtype, a in rec:
            nb = name.encode()
            if len(nb) > 23:
                raise ValueError('record name too long: %s' % name)
            fp.write(nb.ljust(24, b'\0'))
            fp.write(struct.pack('<iiq', dtype, 0, a.size))
            fp.write(a.tobytes())


def _mpc_vehicle(problem):
    """The vehicle, parameter and variable entries and obstacle records both device MPC descriptors
    share; raises NotImplementedError naming the cause for what the device MPC update does not run."""
    if len(problem.vehicles) != 1:
        raise NotImplementedError('the device MPC update runs one vehicle, this problem has %d'
                                  % len(problem.vehicles))
    veh = problem.vehicles[0]
    if type(veh).__name__ not in ('Holonomic', 'Holonomic3D'):
        raise NotImplementedError('the device MPC update runs a Holonomic or Holonomic3D vehicle, not %s'
                                  % type(veh).__name__)
    nd = veh.n_dim
    for o in problem.environment.obstacles:
        if o.options.get('spline_traj'):
            raise NotImplementedError('the device MPC update takes obstacles that move with x/v/a or rotate, '
                                      'not %s with a spline trajectory (spline_traj)' % o.label)
        if o.n_dim != nd:
            raise NotImplementedError('obstacle %s has %d dimensions, the vehicle %d' % (o.label, o.n_dim, nd))
    father = problem.father
    par = father._par_struct.entries
    var = father._var_struct.entries
    kind, off = [], []
    for o in problem.environment.obstacles:
        rot = (o.label, 'theta') in par
        kind.append(int(rot))
        off.append([par[(o.label, k)][0] for k in ('x', 'v', 'a')] + [par[(o.label, 'theta')][0] if rot else -1])
    basis = veh.basis
    return veh, par, var, {
        'n': father.tables.n, 'n_par': father.tables.n_par, 'n_dim': nd,
        'spl_offset': var[(veh.label, 'splines_seg0')][0], 'L': len(basis), 'degree': basis.degree,
        'knots': np.asarray(basis.knots, dtype=np.float64),
        'p_state0': par[(veh.label, 'state0')][0], 'p_input0': par[(veh.label, 'input0')][0],
        'p_poseT': par[(veh.label, 'poseT')][0],
        'n_obs': len(kind), 'obs_kind': np.array(kind, dtype=np.int32),
        'obs_off': np.array(off, dtype=np.int32).reshape(-1),
        'x_template': np.asarray(father.get_variables().cat, dtype=np.float64),
        'p_template': np.asarray(father.set_parameters(0.).cat, dtype=np.float64)}


def mpc_desc(problem, update_time=0.1, sample_time=0.01):
    """The descriptor of the device-resident MPC update (include/omg_b200.h, omg_mpc_desc) of a
    fixed-horizon Point2point with one Holonomic or Holonomic3D vehicle, as a dict of the
    MPC_FIELDS.  Raises NotImplementedError naming the cause for anything else (mpc_freeT_desc
    describes a free motion time)."""
    from ..problems.point2point import FreeTPoint2point
    if isinstance(problem, FreeTPoint2point):
        raise NotImplementedError('the device MPC update has a fixed horizon only, not a free motion time '
                                  '(FreeTPoint2point)')
    veh, par, var, desc = _mpc_vehicle(problem)
    shifted = problem.father.shifted_entries()
    lab = problem.label
    desc.update({
        'horizon': float(problem.options['horizon_time']), 'knot_time': float(problem.knot_time),
        'update_time': float(update_time), 'sample_time': float(sample_time),
        'p_t': par[(lab, 't')][0], 'p_T': par[(lab, 'T')][0],
        'n_shift': len(shifted), 'shift_off': np.array([e[2] for e in shifted], dtype=np.int32),
        'shift_len': np.array([e[3][0] for e in shifted], dtype=np.int32),
        'shift_ncol': np.array([e[3][1] for e in shifted], dtype=np.int32),
        'shift_T': np.concatenate([np.asarray(e[4], dtype=np.float64).reshape(-1) for e in shifted] + [np.zeros(0)])})
    return desc


def mpc_freeT_desc(problem, update_time=0.1, sample_time=0.01):
    """The descriptor of the device-resident MPC update with a free motion time (include/omg_b200.h,
    omg_mpc_freeT_desc) of a FreeTPoint2point with one Holonomic or Holonomic3D vehicle, as a dict
    of the MPC_FREET_FIELDS.  Raises NotImplementedError naming the cause for anything else."""
    from ..problems.point2point import FreeTPoint2point
    if not isinstance(problem, FreeTPoint2point):
        raise NotImplementedError('mpc_freeT_desc describes a free motion time (FreeTPoint2point); '
                                  'mpc_desc describes a fixed horizon')
    veh, par, var, desc = _mpc_vehicle(problem)
    blocks = spline_blocks(problem.father)
    desc.update({
        'update_time': float(update_time), 'sample_time': float(sample_time),
        'stop_tol': float(veh.options['stop_tol']), 't_index': var[(problem.label, 'T')][0],
        'n_blocks': len(blocks), 'blk_off': np.array([b[0] for b in blocks], dtype=np.int32),
        'blk_len': np.array([b[1] for b in blocks], dtype=np.int32),
        'blk_ncol': np.array([b[2] for b in blocks], dtype=np.int32),
        'blk_degree': np.array([b[3] for b in blocks], dtype=np.int32),
        'blk_knots': np.concatenate([np.asarray(b[4], dtype=np.float64) for b in blocks] + [np.zeros(0)])})
    return desc


def mpc_obstacles_desc(problem):
    """The obstacle descriptor of the device MPC update (include/omg_b200.h, omg_mpc_obstacles_desc)
    of a problem mpc_desc or mpc_freeT_desc describes, as a dict of the MPC_OBSTACLE_FIELDS: per
    obstacle, in environment order, the p entries of its checkpoints and radii and the g rows of its
    own constraints, the rows the reference's updateBounds frees when the obstacle is not avoided
    (export.py _create_updateBounds).  Raises NotImplementedError as those do."""
    _, par, _, desc = _mpc_vehicle(problem)
    father = problem.father
    cons = father._con_struct.entries
    out = {k: [] for k, _ in MPC_OBSTACLE_FIELDS[1:]}
    for o in problem.environment.obstacles:
        chk, rad = par[(o.label, 'checkpoints')], par[(o.label, 'rad')]
        rows = [cons[(None, o._add_label(name))][:2] for name in o._constraints]
        lo = rows[0][0] if rows else 0
        if any(r[0] != lo + sum(q[1] for q in rows[:i]) for i, r in enumerate(rows)):
            raise NotImplementedError('the constraint rows of obstacle %s are not one contiguous run' % o.label)
        for key, v in (('chk_off', chk[0]), ('chk_len', chk[1]), ('rad_off', rad[0]), ('rad_len', rad[1]),
                       ('row_off', lo), ('row_len', sum(r[1] for r in rows))):
            out[key].append(v)
    out = {k: np.array(v, dtype=np.int32) for k, v in out.items()}
    out['n_obs'] = desc['n_obs']
    return out


def _pack(desc, fields, cls):
    keep, D = _Keep(), cls()
    for name, kind in fields:
        v = desc[name]
        cast = {'i': int, 'd': float, 'I': keep.i32, 'D': keep.f64}[kind]
        setattr(D, name, cast(v))
    return D, keep


def pack_mpc_desc(desc):
    """mpc_desc dict -> (ctypes omg_mpc_desc, keep-alive object)."""
    return _pack(desc, MPC_FIELDS, _MpcDesc)


def pack_mpc_obstacles_desc(desc):
    """mpc_obstacles_desc dict -> (ctypes omg_mpc_obstacles_desc, keep-alive object)."""
    return _pack(desc, MPC_OBSTACLE_FIELDS, _MpcObstaclesDesc)


def pack_mpc_freeT_desc(desc):
    """mpc_freeT_desc dict -> (ctypes omg_mpc_freeT_desc, keep-alive object)."""
    return _pack(desc, MPC_FREET_FIELDS, _MpcFreeTDesc)


def _write_mpc(desc, fields, path, magic=b'OMGMPC\0\0'):
    import struct
    with open(path, 'wb') as fp:
        fp.write(magic)
        fp.write(struct.pack('<ii', ABI_VERSION, len(fields)))
        for name, kind in fields:
            dtype = 1 if kind in 'dD' else 0
            a = np.ascontiguousarray(desc[name], dtype=np.float64 if dtype else np.int32).reshape(-1)
            fp.write(name.encode().ljust(24, b'\0'))
            fp.write(struct.pack('<iiq', dtype, 0, a.size))
            fp.write(a.tobytes())


def save_mpc(problem, path, update_time=0.1, sample_time=0.01):
    """Write the descriptor of the device MPC update to an MPC file (include/omg_b200.h:
    omg_mpc_read), the companion of save_tables for native callers of omg_mpc_update."""
    _write_mpc(mpc_desc(problem, update_time, sample_time), MPC_FIELDS, path)


def save_mpc_freeT(problem, path, update_time=0.1, sample_time=0.01):
    """Write the free-T descriptor of the device MPC update to an MPC file (include/omg_b200.h:
    omg_mpc_freet_read)."""
    _write_mpc(mpc_freeT_desc(problem, update_time, sample_time), MPC_FREET_FIELDS, path)


def save_mpc_obstacles(problem, path):
    """Write the obstacle descriptor of the device MPC update to an obstacle file (include/omg_b200.h:
    omg_mpc_obstacles_read), for native callers of omg_mpc_attach_obstacles."""
    _write_mpc(mpc_obstacles_desc(problem), MPC_OBSTACLE_FIELDS, path, b'OMGOBS\0\0')


class B200Solver(object):
    """Batched interior-point solver on one GPU for one NLP structure."""

    def __init__(self, tables, options=None, device=None):
        self.lib = load_library()
        if self.lib.omg_abi_version() != ABI_VERSION:
            raise RuntimeError('libomgb200.so ABI version mismatch')
        self.tables = tables
        self.n, self.m, self.n_par = tables.n, tables.m, tables.n_par
        self._opt = _Options()
        self.lib.omg_default_options(C.byref(self._opt))
        self._apply_options(options or {})
        if device is None:
            device = int(os.environ.get('LOCAL_RANK', '0')) \
                if 'OMG_B200_DEVICE' not in os.environ \
                else int(os.environ['OMG_B200_DEVICE'])
        self.device = device
        T, keep = pack_tables(tables)
        self._handle = self.lib.omg_problem_create(C.byref(T), C.byref(self._opt),
                                                   int(device))
        del keep
        if not self._handle:
            raise RuntimeError('omg_problem_create failed: %s' %
                               self.lib.omg_last_error().decode())
        self._stats = {'return_status': None, 'iter_count': 0}

    def _apply_options(self, options):
        import warnings
        fields = dict((f[0], f[1]) for f in _Options._fields_)
        for key, value in options.items():
            if key in fields and key != 'reserved':
                setattr(self._opt, key, value)
            elif key == 'retry_mu':
                self._retry_mu = float(value)
            elif key == 'feas_steps':
                self._feas_steps = int(value)
            elif key in _NO_EFFECT_IPOPT_OPTIONS:
                # printing / linear-solver selection, and warm_start_init_point: the
                # warm-start pushes are always the 'yes' variants the reference sets
                pass
            else:
                # an IPOPT option that changes the algorithm would silently be lost
                warnings.warn('solver option %r is not supported by the b200 solver and '
                              'is ignored' % key)

    def set_options(self, options):
        self._apply_options(options)
        self._check(self.lib.omg_set_options(self._handle, C.byref(self._opt)))

    def __del__(self):
        try:
            if getattr(self, '_handle', None):
                self.lib.omg_problem_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError('libomgb200: %s' % self.lib.omg_last_error().decode())

    # ------------------------------------------------------------------
    def info(self):
        vals = [C.c_int32() for _ in range(6)]
        self._check(self.lib.omg_get_info(self._handle, *[C.byref(v) for v in vals]))
        keys = ('n', 'm', 'n_par', 'smem_bytes', 'ctas_per_sm', 'n_sm')
        return dict(zip(keys, [v.value for v in vals]))

    @property
    def structure(self):
        """One-line report of the kernel family / factor structure chosen for this problem."""
        return self.lib.omg_structure_info(self._handle).decode()

    @property
    def envelope_layout(self):
        """Layout of the envelope kernels for this problem (include/omg_b200.h,
        omg_envelope_layout)."""
        return self.lib.omg_envelope_layout(self._handle).decode()

    def last_timing(self):
        ms, nl = C.c_float(), C.c_int32()
        self._check(self.lib.omg_last_timing(self._handle, C.byref(ms), C.byref(nl)))
        return ms.value, nl.value

    def trace(self, max_rows=512):
        out = np.zeros((max_rows, 8))
        rows = self.lib.omg_get_trace(self._handle, out.ctypes.data, max_rows)
        if rows < 0:
            self._check(rows)
        return out[:rows]

    # ------------------------------------------------------------------
    def _bounds(self, lbg, ubg, B):
        lbg = self.tables.lbg if lbg is None else np.asarray(lbg, dtype=np.float64)
        ubg = self.tables.ubg if ubg is None else np.asarray(ubg, dtype=np.float64)
        lbg = np.ascontiguousarray(np.asarray(lbg, dtype=np.float64))
        ubg = np.ascontiguousarray(np.asarray(ubg, dtype=np.float64))
        shared = 1 if lbg.ndim == 1 else 0
        if (shared and lbg.size != self.m) or (not shared and lbg.shape != (B, self.m)):
            raise ValueError('lbg/ubg must have shape (m,) or (B, m)')
        if ubg.shape != lbg.shape:
            raise ValueError('lbg and ubg shapes differ')
        return lbg, ubg, shared

    def solve_batch(self, X0, P, lbg=None, ubg=None, lam_g0=None, _retry=True):
        """Host arrays in, host arrays out (H2D + solve + D2H in one C call).

        Instances that end in Restoration_Failed go through the feasibility phase
        (option ``feas_steps``, default 30 Levenberg-Marquardt steps, 0 = off) and are
        solved once more from the point it returns; their iteration counts add up.

        Option ``retry_mu`` > 0 (default 0 = off): instances that did not succeed are
        solved once more from the same start with ``mu_init = retry_mu`` (e.g. 1e-3).
        A small initial barrier parameter keeps the iterates near an infeasible warm
        start instead of pushing every slack to the centre first; it rescues the warm
        starts that IPOPT leaves to its restoration phase (DESIGN.md section 2)."""
        X0 = np.ascontiguousarray(X0, dtype=np.float64).reshape(-1, self.n)
        B = X0.shape[0]
        P = np.ascontiguousarray(P, dtype=np.float64).reshape(B, self.n_par)
        lbg, ubg, shared = self._bounds(lbg, ubg, B)
        lam0 = None
        if lam_g0 is not None:
            lam0 = np.ascontiguousarray(lam_g0, dtype=np.float64).reshape(B, self.m)
        X = np.empty((B, self.n))
        LAM = np.empty((B, self.m))
        F = np.empty(B)
        status = np.empty(B, dtype=np.int32)
        iters = np.empty(B, dtype=np.int32)
        self._check(self.lib.omg_solve_batch_host(
            self._handle, B, X0.ctypes.data, P.ctypes.data, lbg.ctypes.data,
            ubg.ctypes.data, shared, lam0.ctypes.data if lam0 is not None else None,
            X.ctypes.data, LAM.ctypes.data, F.ctypes.data, status.ctypes.data,
            iters.ctypes.data))
        res = {'x': X, 'lam_g': LAM, 'f': F, 'status': status, 'iters': iters}
        n_feas = getattr(self, '_feas_steps', FEAS_STEPS)
        if _retry and n_feas > 0 and (status == 2).any():
            # Restoration_Failed: feasibility phase from the point where the line search
            # gave up, then one more solve from there (DESIGN.md section 2)
            idx = np.nonzero(status == 2)[0]
            lb_i, ub_i = (lbg, ubg) if shared else (lbg[idx], ubg[idx])
            x1, _, _ = self.feasibility_batch(X[idx], P[idx], lb_i, ub_i, n_feas)
            r2 = self.solve_batch(x1, P[idx], lb_i, ub_i, None, _retry=False)
            ok = r2['status'] == 0          # the first result stands unless the re-solve succeeds
            for key in ('x', 'lam_g', 'f', 'status'):
                res[key][idx[ok]] = r2[key][ok]
            res['iters'][idx] += r2['iters']
        mu_r = getattr(self, '_retry_mu', 0.)
        if _retry and mu_r > 0. and (status != 0).any():
            idx = np.nonzero(status != 0)[0]
            mu_old = self._opt.mu_init
            self.set_options({'mu_init': mu_r})
            try:
                r2 = self.solve_batch(X0[idx], P[idx], lbg if shared else lbg[idx],
                                      ubg if shared else ubg[idx],
                                      None if lam0 is None else lam0[idx], _retry=False)
            finally:
                self.set_options({'mu_init': mu_old})
            ok = r2['status'] == 0
            for key in ('x', 'lam_g', 'f', 'status'):
                res[key][idx[ok]] = r2[key][ok]
            res['iters'][idx] += r2['iters']
        return res

    def feasibility_batch(self, X0, P, lbg=None, ubg=None, max_steps=None):
        """Host arrays in / out: up to ``max_steps`` Levenberg-Marquardt steps on the
        constraint violation from X0 (omg_feas_batch_host).  Returns (X, max |violation|
        per instance, steps taken per instance)."""
        X0 = np.ascontiguousarray(X0, dtype=np.float64).reshape(-1, self.n)
        B = X0.shape[0]
        P = np.ascontiguousarray(P, dtype=np.float64).reshape(B, self.n_par)
        lbg, ubg, shared = self._bounds(lbg, ubg, B)
        if max_steps is None:
            max_steps = getattr(self, '_feas_steps', FEAS_STEPS)
        X = np.empty((B, self.n))
        viol = np.empty(B)
        steps = np.empty(B, dtype=np.int32)
        self._check(self.lib.omg_feas_batch_host(
            self._handle, B, X0.ctypes.data, P.ctypes.data, lbg.ctypes.data, ubg.ctypes.data,
            shared, int(max_steps), X.ctypes.data, viol.ctypes.data, steps.ctypes.data))
        return X, viol, steps

    def solve_batch_device(self, X0, P, LBG, UBG, X, LAM, F, STATUS, ITERS,
                           lam_g0=None, stream=None):
        """torch CUDA tensors (float64 / int32, contiguous); asynchronous on
        ``stream`` (torch.cuda.Stream or None = current)."""
        B = X0.shape[0]
        on_gpu = _check_device_tensors((X0, P, LBG, UBG, X, LAM, F) +
                                       ((lam_g0,) if lam_g0 is not None else ()), self.lib)
        _check_int_tensors((STATUS, ITERS))
        if (X0.shape != (B, self.n) or P.shape != (B, self.n_par) or X.shape != (B, self.n) or
                LAM.shape != (B, self.m) or F.numel() != B or STATUS.numel() != B or ITERS.numel() != B or
                (lam_g0 is not None and lam_g0.shape != (B, self.m))):
            raise ValueError('tensor shapes do not match the batch / problem sizes')
        shared = 1 if LBG.dim() == 1 else 0
        self._check(self.lib.omg_solve_batch(
            self._handle, B, X0.data_ptr(), P.data_ptr(), LBG.data_ptr(),
            UBG.data_ptr(), shared, lam_g0.data_ptr() if lam_g0 is not None else None,
            X.data_ptr(), LAM.data_ptr(), F.data_ptr(), STATUS.data_ptr(),
            ITERS.data_ptr(), _stream_handle(on_gpu, X0.device, stream)))

    def shift_batch_device(self, X, blocks, stream=None):
        """In-place warm-start shift of spline variables (torch CUDA tensor X
        [B, n]); blocks = [(offset, len_basis, n_columns, T)], T of shape
        len_basis x len_basis."""
        offs = np.array([b[0] for b in blocks], dtype=np.int32)
        lens = np.array([b[1] for b in blocks], dtype=np.int32)
        ncols = np.array([b[2] for b in blocks], dtype=np.int32)
        for b in blocks:
            if np.shape(b[3]) != (b[1], b[1]):
                raise ValueError('a block of length %d needs a %d x %d T, got %s'
                                 % (b[1], b[1], b[1], np.shape(b[3])))
        Tm = np.concatenate([np.asarray(b[3], dtype=np.float64).reshape(-1)
                             for b in blocks])
        on_gpu = _check_device_tensors((X,), self.lib)
        if X.dim() != 2 or X.shape[1] != self.n:
            raise ValueError('X must be [B, n]')
        self._check(self.lib.omg_shift_batch(
            self._handle, X.shape[0], X.data_ptr(), len(blocks), offs.ctypes.data,
            lens.ctypes.data, ncols.ctypes.data, Tm.ctypes.data,
            _stream_handle(on_gpu, X.device, stream)))

    def shift_free_batch_device(self, X, blocks, t_index, update_time, active=None, stream=None):
        """Free-T warm start in place (omg_shift_free_batch): for every active instance of the torch
        CUDA tensor X [B, n], shift_spline of each block by tau = u / target from its own motion
        time X[b, t_index], which becomes target.  blocks = [(offset, len_basis, n_columns, degree,
        knots)], e.g. spline_blocks(father); active: int32 CUDA tensor [B] (nonzero = shift) or
        None for all."""
        desc = _spline_desc(blocks)
        on_gpu = _check_device_tensors((X,), self.lib)
        if active is not None:
            _check_int_tensors((active,))
            if active.numel() != X.shape[0]:
                raise ValueError('active must hold one flag per instance')
        if X.dim() != 2 or X.shape[1] != self.n:
            raise ValueError('X must be [B, n]')
        self._check(self.lib.omg_shift_free_batch(
            self._handle, X.shape[0], X.data_ptr(), int(t_index), float(update_time),
            active.data_ptr() if active is not None else None, len(blocks),
            *[a.ctypes.data for a in desc], _stream_handle(on_gpu, X.device, stream)))

    # ------------------------------------------------------------------
    # the reference's single-instance call contract
    # ------------------------------------------------------------------
    def __call__(self, x0=None, p=None, lbg=None, ubg=None, lam_g0=None, **kwargs):
        x0 = np.asarray(x0, dtype=np.float64).reshape(1, self.n)
        p = np.asarray(p, dtype=np.float64).reshape(1, self.n_par)
        lb = None if lbg is None else np.asarray(lbg, dtype=np.float64).reshape(-1)
        ub = None if ubg is None else np.asarray(ubg, dtype=np.float64).reshape(-1)
        lam0 = None if lam_g0 is None else \
            np.asarray(lam_g0, dtype=np.float64).reshape(1, self.m)
        if lb is not None and ub is not None:
            # the equality rows are part of the factorised structure: bounds that turn an equality
            # into an inequality (or the reverse) need a re-lowered problem, not another call
            eq_now, eq_built = (lb == ub), (self.tables.lbg == self.tables.ubg)
            if not np.array_equal(eq_now, eq_built):
                rows = np.nonzero(eq_now != eq_built)[0][:5].tolist()
                raise ValueError('lbg/ubg change which rows are equalities (rows %s ...): the '
                                 'equality pattern is fixed when the problem is lowered' % rows)
        res = self.solve_batch(x0, p, lb, ub, lam0)
        self._stats = {'return_status': STATUS_STRINGS[int(res['status'][0])],
                       'iter_count': int(res['iters'][0]),
                       'success': int(res['status'][0]) == 0}
        return {'x': res['x'][0], 'lam_g': res['lam_g'][0], 'f': float(res['f'][0])}

    def stats(self):
        return dict(self._stats)


def admm_zl_update(PzT, c, Tf, Tb, rho, x_i, x_j, z_i, z_ij, l_i, l_ij, res, L, stream=None):
    """Consensus step (z, lambda, residuals) for the agents held in the given
    torch CUDA tensors; z_*, l_* are updated in place (omg_admm_zl_update)."""
    import torch
    lib = load_library()
    n_agents, nsh = x_i.shape
    nn = x_j.shape[1]
    on_gpu = _check_device_tensors((PzT, c, Tf, Tb, x_i, x_j, z_i, z_ij, l_i, l_ij, res), lib)
    rc = lib.omg_admm_zl_update(n_agents, nsh, nn, L, PzT.data_ptr(), c.data_ptr(),
                                Tf.data_ptr(), Tb.data_ptr(), float(rho), x_i.data_ptr(),
                                x_j.data_ptr(), z_i.data_ptr(), z_ij.data_ptr(),
                                l_i.data_ptr(), l_ij.data_ptr(), res.data_ptr(),
                                _stream_handle(on_gpu, x_i.device, stream))
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())


class AdmmComm(object):
    """The library's NCCL communicator for the formation ADMM exchange (include/omg_b200.h:
    omg_comm_*).  The 128-byte unique id is created on rank 0 and handed to the other ranks by
    the caller's bootstrap -- here a torch.distributed broadcast; a C++ caller uses whatever it
    has (MPI, a socket, a file)."""

    def __init__(self, rank=0, world=1, device=0, group=None):
        import torch
        self.lib = load_library()
        idbuf = (C.c_char * 128)()
        if world > 1:
            import torch.distributed as dist
            t = torch.zeros(128, dtype=torch.uint8, device=torch.device('cuda', device))
            if rank == 0:
                if self.lib.omg_comm_unique_id(idbuf) != 0:
                    raise RuntimeError('libomgb200: %s' % self.lib.omg_last_error().decode())
                t.copy_(torch.frombuffer(bytearray(idbuf.raw), dtype=torch.uint8))
            dist.broadcast(t, src=0, group=group)
            idbuf.raw = bytes(t.cpu().numpy().tobytes())
        self.handle = self.lib.omg_comm_create(idbuf, world, rank, device)
        if not self.handle:
            raise RuntimeError('libomgb200: %s' % self.lib.omg_last_error().decode())
        self.rank, self.world, self.device = rank, world, device

    def exchange_x(self, nghb, x_i, x_j, stream=None):
        n_local, nsh = x_i.shape
        rc = self.lib.omg_admm_exchange_x(self.handle, n_local, nsh, x_j.shape[1], nghb.data_ptr(),
                                          x_i.data_ptr(), x_j.data_ptr(), _stream_handle(True, x_i.device, stream))
        if rc != 0:
            raise RuntimeError('libomgb200: %s' % self.lib.omg_last_error().decode())

    def zl_update(self, PzT, c, Tf, Tb, rho, x_i, x_j, z_i, z_ij, l_i, l_ij, res, L, nghb, back,
                  z_ji, l_ji, res_total, stream=None):
        """Consensus kernel + residual all-reduce + second exchange, one stream-ordered call."""
        n_local, nsh = x_i.shape
        rc = self.lib.omg_admm_zl_update_dist(
            self.handle, n_local, nsh, x_j.shape[1], L, PzT.data_ptr(), c.data_ptr(), Tf.data_ptr(),
            Tb.data_ptr(), float(rho), x_i.data_ptr(), x_j.data_ptr(), z_i.data_ptr(), z_ij.data_ptr(),
            l_i.data_ptr(), l_ij.data_ptr(), res.data_ptr(), nghb.data_ptr(), back.data_ptr(),
            z_ji.data_ptr(), l_ji.data_ptr(), res_total.data_ptr(), _stream_handle(True, x_i.device, stream))
        if rc != 0:
            raise RuntimeError('libomgb200: %s' % self.lib.omg_last_error().decode())

    def __del__(self):
        try:
            if self.handle:
                self.lib.omg_comm_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def sample_batch(X, blocks, stream=None):
    """Apply sampling matrices to spline variables of a batch on the device.
    X: torch CUDA tensor [B, n]; blocks = [(offset, len_basis, n_columns, S[nsamp, len])].
    Returns a CUDA tensor [B, sum(nsamp * n_columns)] laid out block / column / sample."""
    import torch
    lib = load_library()
    offs = np.array([b[0] for b in blocks], dtype=np.int32)
    lens = np.array([b[1] for b in blocks], dtype=np.int32)
    ncols = np.array([b[2] for b in blocks], dtype=np.int32)
    for b in blocks:
        if np.ndim(b[3]) != 2 or np.shape(b[3])[1] != b[1]:
            raise ValueError('a block of length %d needs an S with %d columns, got shape %s'
                             % (b[1], b[1], np.shape(b[3])))
    if X.dim() != 2:
        raise ValueError('X must be [B, n]')
    nsamp = np.array([np.asarray(b[3]).shape[0] for b in blocks], dtype=np.int32)
    Sm = np.concatenate([np.ascontiguousarray(b[3], dtype=np.float64).reshape(-1) for b in blocks])
    out = torch.empty((X.shape[0], int((nsamp * ncols).sum())), dtype=torch.float64, device=X.device)
    on_gpu = _check_device_tensors((X,), lib)
    rc = lib.omg_sample_batch(X.shape[0], X.shape[1], X.data_ptr(), len(blocks), offs.ctypes.data,
                              lens.ctypes.data, ncols.ctypes.data, nsamp.ctypes.data,
                              Sm.ctypes.data, out.data_ptr(), _stream_handle(on_gpu, X.device, stream))
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())
    return out


def _spline_desc(blocks):
    """[(offset, len_basis, n_columns, degree, knots)] -> host arrays offs, lens, ncols, degrees and
    the concatenated knots (len_basis + degree + 1 per block)."""
    desc = [np.array([b[k] for b in blocks], dtype=np.int32) for k in range(4)]
    knots = [np.ascontiguousarray(b[4], dtype=np.float64).reshape(-1) for b in blocks]
    for b, k in zip(blocks, knots):
        if k.size != b[1] + b[3] + 1:
            raise ValueError('a block of length %d and degree %d needs %d knots, got %d'
                             % (b[1], b[3], b[1] + b[3] + 1, k.size))
    return desc + [np.concatenate(knots) if knots else np.zeros(1)]


def spline_blocks(father, vehicle=None):
    """The blocks of shift_free_batch_device / eval_batch: [(offset, len_basis, n_columns, degree,
    knots)] of the spline variables the warm start transforms (father.shifted_entries()), or,
    with ``vehicle``, of that vehicle's splines_seg0."""
    out = []
    for label, name, off, shape, _ in father.shifted_entries():
        if vehicle is not None and (label, name) != (vehicle.label, 'splines_seg0'):
            continue
        basis = father.children[label]._splines_prim[name]['basis']
        out.append((off, shape[0], shape[1], basis.degree, basis.knots))
    return out


def eval_batch(X, blocks, tau, scale, n_der, stream=None):
    """Per-instance spline evaluation on the device (omg_eval_batch).  X: torch CUDA tensor
    [B, n]; blocks = [(offset, len_basis, n_columns, degree, knots)]; tau: CUDA tensor
    [B, n_pts] of abscissae in the knot span (padding points anywhere; they evaluate to 0 outside
    it); scale: CUDA tensor [B].  Returns a CUDA tensor [B, sum(n_columns) * n_pts * n_der] laid
    out block / column / point / derivative, derivative d divided by scale^d."""
    import torch
    lib = load_library()
    desc = _spline_desc(blocks)
    on_gpu = _check_device_tensors((X, tau, scale), lib)
    B = X.shape[0]
    if X.dim() != 2 or tau.dim() != 2 or tau.shape[0] != B or scale.numel() != B:
        raise ValueError('X must be [B, n], tau [B, n_pts] and scale [B]')
    n_pts = tau.shape[1]
    out = torch.empty((B, int(desc[2].sum()) * n_pts * int(n_der)), dtype=torch.float64, device=X.device)
    rc = lib.omg_eval_batch(B, X.shape[1], X.data_ptr(), len(blocks), *[a.ctypes.data for a in desc], n_pts,
                            tau.data_ptr(), scale.data_ptr(), int(n_der), out.data_ptr(),
                            _stream_handle(on_gpu, X.device, stream))
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())
    return out


ODE_MODELS = {'Holonomic': 0, 'Holonomic1D': 0, 'Holonomic3D': 0, 'Quadrotor3D': 1, 'Quadrotor': 2,
              'Dubins': 3, 'HolonomicOrient': 4, 'SimpleQuadrotor3D': 5}


def integrate_rk4(model, state0, inputs, sample_time, stream=None):
    """Non-ideal prediction on the device (omg_integrate_rk4): state0 [B, n_state] and the
    planned inputs [B, steps+1, n_input] are torch CUDA float64 tensors; returns the states
    after steps*sample_time.  ``model`` is a vehicle class name or a model id."""
    import torch
    lib = load_library()
    mid = ODE_MODELS[model] if isinstance(model, str) else int(model)
    on_gpu = _check_device_tensors((state0, inputs), lib)
    B, ns = state0.shape
    steps, ni = inputs.shape[1] - 1, inputs.shape[2]
    out = torch.empty_like(state0)
    rc = lib.omg_integrate_rk4(mid, B, ns, ni, state0.data_ptr(), inputs.data_ptr(),
                               float(sample_time), steps, out.data_ptr(),
                               _stream_handle(on_gpu, state0.device, stream))
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())
    return out


def disturbance_filter(fc):
    """{b, a, lfilter_zi} of the reference's input-disturbance filter butter(3, fc, 'low')
    (vehicle.py:444), flattened as omg_closed_loop_step takes it."""
    from scipy.signal import butter, lfilter_zi
    b, a = butter(3, fc, 'low')
    return np.ascontiguousarray(np.r_[b, a, lfilter_zi(b, a)], dtype=np.float64)


def closed_loop_step(model, X, L, R0, R1, sample_time, plant_x, plant_u, out, step, seed=0,
                     time_constant=None, disturbance=None, stream=None, higher=None):
    """Plant step of MPC step ``step`` for a batch (omg_closed_loop_step): the non-ideal
    simulate and predict of the reference's Vehicle from the plant state / last applied input
    (plant_x [B, n_state], plant_u [B, n_input]) along the trajectories of the spline
    coefficients X [B, n], sampled by the host rows R0, R1 [n_samp+1, L].
    out = (plant_x_next, plant_u_next, pred_x, pred_u), written in place (the plant outputs may
    be plant_x / plant_u themselves).  time_constant: first-order actuator lag (None = off).
    disturbance: (filt, mean, stdev, n_traj, scratch) with filt from disturbance_filter(fc) and
    scratch a float64 tensor of at least B * n_input * (n_traj + 24) elements (None = off).
    higher: the rows of derivatives 2 and 3 [k, n_samp+1, L] (divided by T^2, T^3), which the
    quadrotor models read; with them, or for a model other than 0 and 1, the call goes to
    omg_closed_loop_step_der."""
    lib = load_library()
    mid = ODE_MODELS[model] if isinstance(model, str) else int(model)
    tensors = (X, plant_x, plant_u) + tuple(out)
    if disturbance is not None:
        filt, mean, stdev, n_traj, scratch = disturbance
        tensors += (scratch,)
        if scratch.numel() < X.shape[0] * plant_u.shape[1] * (n_traj + 24):
            raise ValueError('disturbance scratch too small')
        filt, mean, stdev = (np.ascontiguousarray(a, dtype=np.float64) for a in (filt, mean, stdev))
        if filt.size != 11 or mean.size != plant_u.shape[1] or stdev.size != plant_u.shape[1]:
            raise ValueError('disturbance filter / mean / stdev sizes')
    on_gpu = _check_device_tensors(tensors, lib)
    B, ns = plant_x.shape
    ni = plant_u.shape[1]
    R0 = np.ascontiguousarray(R0, dtype=np.float64)
    R1 = np.ascontiguousarray(R1, dtype=np.float64)
    if R0.shape != R1.shape or R0.ndim != 2 or R0.shape[1] != L:
        raise ValueError('R0 / R1 must both be [n_samp + 1, L]')
    for t, shape in zip(out, ((B, ns), (B, ni), (B, ns), (B, ni))):
        if tuple(t.shape) != shape:
            raise ValueError('output tensor shapes do not match the plant state / input')
    d = disturbance is not None
    rest = (float(sample_time), int(time_constant is not None),
            float(time_constant) if time_constant is not None else 0., int(d), int(n_traj) if d else 0,
            filt.ctypes.data if d else None, mean.ctypes.data if d else None,
            stdev.ctypes.data if d else None, int(seed) & 0xFFFFFFFFFFFFFFFF, int(step),
            plant_x.data_ptr(), plant_u.data_ptr(), *[t.data_ptr() for t in out],
            scratch.data_ptr() if d else None, _stream_handle(on_gpu, X.device, stream))
    if higher is None and mid in (0, 1):
        rc = lib.omg_closed_loop_step(mid, B, ns, ni, X.shape[1], X.data_ptr(), L, R0.shape[0] - 1,
                                      R0.ctypes.data, R1.ctypes.data, *rest)
    else:
        rows = [R0[None], R1[None]]
        if higher is not None:
            higher = np.asarray(higher, dtype=np.float64)
            if higher.ndim != 3 or higher.shape[1:] != R0.shape:
                raise ValueError('higher must be [k, n_samp + 1, L]')
            rows.append(higher)
        R = np.ascontiguousarray(np.concatenate(rows))
        rc = lib.omg_closed_loop_step_der(mid, B, ns, ni, X.shape[1], X.data_ptr(), L, R0.shape[0] - 1,
                                          R.shape[0], R.ctypes.data, *rest)
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())


def closed_loop_step_fleet(model, X, offsets, L, R, sample_time, plant_x, plant_u, out, step, seed=0,
                           time_constant=None, disturbance=None, stream=None):
    """closed_loop_step for a fleet of vehicles of one model and one spline basis in every row of X
    (omg_closed_loop_step_fleet): vehicle v's input splines start at column offsets[v] of X.
    R: the derivative rows [n_der, n_samp + 1, L] (plant_rows_der; n_der from the model's to 4).
    plant_x [B, n_veh, n_state], plant_u [B, n_veh, n_input] and the four tensors of ``out`` carry
    a vehicle axis; disturbance = (filt, mean, stdev, n_traj, scratch) with scratch of at least
    B * n_veh * n_input * (n_traj + 24) elements.  The noise of vehicle v's input j is keyed as
    signal v * n_input + j of the instance.  Every other argument is closed_loop_step's."""
    lib = load_library()
    mid = ODE_MODELS[model] if isinstance(model, str) else int(model)
    tensors = (X, plant_x, plant_u) + tuple(out)
    if plant_x.dim() != 3 or plant_u.dim() != 3:
        raise ValueError('plant_x / plant_u must be [B, n_veh, n_state | n_input]')
    B, nv, ns = plant_x.shape
    ni = plant_u.shape[2]
    offsets = np.ascontiguousarray(offsets, dtype=np.int32).reshape(-1)
    if offsets.size != nv or tuple(plant_u.shape[:2]) != (B, nv):
        raise ValueError('one spline offset per vehicle of plant_x / plant_u')
    d = disturbance is not None
    if d:
        filt, mean, stdev, n_traj, scratch = disturbance
        tensors += (scratch,)
        if scratch.numel() < B * nv * ni * (n_traj + 24):
            raise ValueError('disturbance scratch too small')
        filt, mean, stdev = (np.ascontiguousarray(a, dtype=np.float64) for a in (filt, mean, stdev))
        if filt.size != 11 or mean.size != ni or stdev.size != ni:
            raise ValueError('disturbance filter / mean / stdev sizes')
    on_gpu = _check_device_tensors(tensors, lib)
    if X.dim() != 2 or X.shape[0] != B:
        raise ValueError('X must be [B, n] with the batch of plant_x')
    for t, shape in zip(out, ((B, nv, ns), (B, nv, ni), (B, nv, ns), (B, nv, ni))):
        if tuple(t.shape) != shape:
            raise ValueError('output tensor shapes do not match the plant state / input')
    R = np.ascontiguousarray(R, dtype=np.float64)
    if R.ndim != 3 or R.shape[2] != L:
        raise ValueError('R must be [n_der, n_samp + 1, L]')
    rc = lib.omg_closed_loop_step_fleet(
        mid, B, nv, ns, ni, X.shape[1], X.data_ptr(), offsets.ctypes.data, int(L), R.shape[1] - 1, R.shape[0],
        R.ctypes.data, float(sample_time), int(time_constant is not None),
        float(time_constant) if time_constant is not None else 0., int(d), int(n_traj) if d else 0,
        filt.ctypes.data if d else None, mean.ctypes.data if d else None, stdev.ctypes.data if d else None,
        int(seed) & 0xFFFFFFFFFFFFFFFF, int(step), plant_x.data_ptr(), plant_u.data_ptr(),
        *[t.data_ptr() for t in out], scratch.data_ptr() if d else None, _stream_handle(on_gpu, X.device, stream))
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())


def closed_loop_step_free(model, X, block, t_index, n_der, n_samp, sample_time, plant_x, plant_u, out, step,
                          seed=0, time_constant=None, disturbance=None, stream=None):
    """closed_loop_step with a free motion time (omg_closed_loop_step_free): instance b samples its
    plan at s * sample_time / T_b, T_b = X[b, t_index], for s = 0..n_samp[b] (0 = b is left alone).
    block = (offset, len_basis, n_columns, degree, knots) of the spline block whose first columns
    are the input splines (spline_blocks(father, vehicle)[0]); n_der: derivative rows the model
    reads (2 to 4).  n_samp: host int array [B].  disturbance: (filt, mean, stdev, n_traj, scratch)
    with n_traj a host int array [B] (0 = no disturbance for that instance) and scratch a float64
    tensor of at least B * n_input * (max(n_traj) + 24) elements (None = off).  Every other
    argument is closed_loop_step's."""
    lib = load_library()
    mid = ODE_MODELS[model] if isinstance(model, str) else int(model)
    tensors = (X, plant_x, plant_u) + tuple(out)
    B, ns = plant_x.shape
    ni = plant_u.shape[1]
    n_samp = np.ascontiguousarray(n_samp, dtype=np.int32).reshape(-1)
    if n_samp.size != B:
        raise ValueError('n_samp must hold one count per instance')
    d = disturbance is not None
    if d:
        filt, mean, stdev, n_traj, scratch = disturbance
        tensors += (scratch,)
        n_traj = np.ascontiguousarray(n_traj, dtype=np.int32).reshape(-1)
        if n_traj.size != B:
            raise ValueError('n_traj must hold one count per instance')
        if scratch.numel() < B * ni * (int(n_traj.max(initial=0)) + 24):
            raise ValueError('disturbance scratch too small')
        filt, mean, stdev = (np.ascontiguousarray(a, dtype=np.float64) for a in (filt, mean, stdev))
        if filt.size != 11 or mean.size != ni or stdev.size != ni:
            raise ValueError('disturbance filter / mean / stdev sizes')
    on_gpu = _check_device_tensors(tensors, lib)
    if X.dim() != 2 or X.shape[0] != B:
        raise ValueError('X must be [B, n] with the batch of plant_x')
    for t, shape in zip(out, ((B, ns), (B, ni), (B, ns), (B, ni))):
        if tuple(t.shape) != shape:
            raise ValueError('output tensor shapes do not match the plant state / input')
    off, L, nc, degree, knots = block
    knots = np.ascontiguousarray(knots, dtype=np.float64).reshape(-1)
    if knots.size != L + degree + 1:
        raise ValueError('a block of length %d and degree %d needs %d knots, got %d'
                         % (L, degree, L + degree + 1, knots.size))
    rc = lib.omg_closed_loop_step_free(
        mid, B, ns, ni, X.shape[1], X.data_ptr(), int(off), int(L), int(nc), int(degree), knots.ctypes.data,
        int(t_index), int(n_der), n_samp.ctypes.data, n_traj.ctypes.data if d else None, float(sample_time),
        int(time_constant is not None), float(time_constant) if time_constant is not None else 0., int(d),
        filt.ctypes.data if d else None, mean.ctypes.data if d else None, stdev.ctypes.data if d else None,
        int(seed) & 0xFFFFFFFFFFFFFFFF, int(step), plant_x.data_ptr(), plant_u.data_ptr(),
        *[t.data_ptr() for t in out], scratch.data_ptr() if d else None, _stream_handle(on_gpu, X.device, stream))
    if rc != 0:
        raise RuntimeError('libomgb200: %s' % lib.omg_last_error().decode())
