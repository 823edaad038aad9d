"""Device-resident receding-horizon loop: B independent copies of the reference's exported
Point2Point::update() (omgtools/export/point2point/Point2Point.cpp:119-231) for a fixed-horizon
Point2point with one Holonomic or Holonomic3D vehicle, one stream-ordered C call per update
(include/omg_b200.h, omg_mpc_update).

Unlike BatchMPC, nothing of the loop runs on the host: the warm start and its knot shift, the
prediction, the parameter rows, the solve and the trajectory sampling all stay on the device, and
each instance keeps its own time.  The caller is the plant: it hands every update the measured
state (read on a cold start, and by the 'integrate' prediction), the goal and the obstacles'
current x, v, a (and theta), as the reference's obstacle_t, and receives the planned state and
input trajectories.  An update makes no synchronous CUDA call and no allocation after the first
one, so a sequence of updates can be captured in a CUDA graph.

With a FreeTPoint2point (the motion time T a decision variable) every instance runs the reference's
free-T loop on its own T (include/omg_b200.h, omg_mpc_create_freet): the warm start is re-expressed
from the plan's own T, the prediction and the trajectory samples are taken on the plan's own time
axis, and an instance whose plan is shorter than update_time, or that has arrived at its goal, stops:
it is not solved again (status MPC_STOPPED = -1, 0 iterations) until recover().  motion_time() gives
each instance's T, and so how much of the returned trajectory is plan.

The rest of the reference's obstacle_t, each obstacle's shape (checkpoints and radii) and its avoid
flag, is per-instance state that set_obstacles() changes (include/omg_b200.h,
omg_mpc_set_obstacles): an obstacle that is not avoided has its own constraint rows freed for that
instance's solves, as the reference's updateBounds does.
"""
import ctypes as C

import numpy as np

from ..solver import b200


class DeviceMPC(object):
    """``update(state0, stateT, obstacles)`` advances every instance by one update.

    state0, stateT: float64 device tensors [B, n_dim]; obstacles: [B, n_obs, 3 * n_dim + 1] with
    each obstacle's {x, v, a, theta} (theta read for a rotating obstacle only; None without
    obstacles).  Returns the device tensors (state_traj, input_traj [B, trajectory_length, n_dim],
    status, iters [B]) without synchronising.  They are the handle's own buffers, rewritten by the
    next update: an instance whose solve fails keeps its previous rows, its warm start and its
    time (Point2Point::update returning false).  prediction: 'ideal' (the plan's value at
    t + update_time) or 'integrate' (RK4 from state0 over the planned inputs; state0 is then the
    measured state at the start of the previous plan)."""

    def __init__(self, problem, batch, update_time=0.1, sample_time=0.01, trajectory_length=None,
                 prediction='ideal', device=None):
        import torch
        if prediction not in b200.MPC_PREDICTION:
            raise ValueError('prediction must be one of %s' % sorted(b200.MPC_PREDICTION))
        from ..problems.point2point import FreeTPoint2point
        self.free_T = isinstance(problem, FreeTPoint2point)
        if self.free_T:
            desc = b200.mpc_freeT_desc(problem, update_time, sample_time)
            horizon, pack, create = desc['x_template'][desc['t_index']], b200.pack_mpc_freeT_desc, 'omg_mpc_create_freet'
        else:
            desc = b200.mpc_desc(problem, update_time, sample_time)
            horizon, pack, create = desc['horizon'], b200.pack_mpc_desc, 'omg_mpc_create'
        self.solver = problem.problem
        self.lib = self.solver.lib
        self.B, self.n_dim, self.n_obs = int(batch), desc['n_dim'], desc['n_obs']
        if trajectory_length is None:
            trajectory_length = int(np.round(horizon / sample_time, 6))
        self.trajectory_length = int(trajectory_length)
        self.dev = device if device is not None else torch.device('cuda', self.solver.device)
        D, keep = pack(desc)
        self._handle = getattr(self.lib, create)(self.solver._handle, C.byref(D), self.B, self.trajectory_length,
                                                 b200.MPC_PREDICTION[prediction])
        del keep
        if not self._handle:
            raise RuntimeError('%s failed: %s' % (create, self.lib.omg_last_error().decode()))
        self.n, self.n_par = desc['n'], desc['n_par']
        self._problem, self._obs_desc, self._attached = problem, None, False
        f64 = dict(dtype=torch.float64, device=self.dev)
        i32 = dict(dtype=torch.int32, device=self.dev)
        shape = (self.B, self.trajectory_length, self.n_dim)
        self.state_traj, self.input_traj = torch.zeros(shape, **f64), torch.zeros(shape, **f64)
        self.status, self.iters = torch.zeros(self.B, **i32), torch.zeros(self.B, **i32)
        self._no_obs = torch.zeros(1, **f64)

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError('libomgb200: %s' % self.lib.omg_last_error().decode())

    def update(self, state0, stateT, obstacles=None, stream=None):
        B, nd = self.B, self.n_dim
        if obstacles is None:
            if self.n_obs:
                raise ValueError('this problem has %d obstacles: obstacles is required' % self.n_obs)
            obstacles = self._no_obs
        elif tuple(obstacles.shape) != (B, self.n_obs, 3 * nd + 1):
            raise ValueError('obstacles must be [B, n_obs, 3 * n_dim + 1] = [%d, %d, %d]'
                             % (B, self.n_obs, 3 * nd + 1))
        on_gpu = b200._check_device_tensors((state0, stateT, obstacles), self.lib)
        if tuple(state0.shape) != (B, nd) or tuple(stateT.shape) != (B, nd):
            raise ValueError('state0 and stateT must be [B, n_dim] = [%d, %d]' % (B, nd))
        self._check(self.lib.omg_mpc_update(
            self._handle, state0.data_ptr(), stateT.data_ptr(), obstacles.data_ptr(), self.state_traj.data_ptr(),
            self.input_traj.data_ptr(), self.status.data_ptr(), self.iters.data_ptr(),
            b200._stream_handle(on_gpu, state0.device, stream)))
        return self.state_traj, self.input_traj, self.status, self.iters

    def _obstacles(self):
        if self._obs_desc is None:
            self._obs_desc = b200.mpc_obstacles_desc(self._problem)
        return self._obs_desc

    @property
    def shape_layout(self):
        """The record set_obstacles takes per instance: a list with, per obstacle, the slices of its
        checkpoints (x0, y0, x1, y1, ... : n_chk * n_dim values) and of its radii (n_chk values), and
        the record's length."""
        d, out, o = self._obstacles(), [], 0
        for k in range(self.n_obs):
            nc, nr = int(d['chk_len'][k]), int(d['rad_len'][k])
            out.append((slice(o, o + nc), slice(o + nc, o + nc + nr)))
            o += nc + nr
        return out, o

    def set_obstacles(self, shapes=None, avoid=None, stream=None):
        """Set the obstacles' shapes and avoid flags of every instance for this and the following
        updates, until the next call (recover() does not change them).  shapes: float64 device tensor
        [B, record length of shape_layout], per obstacle its checkpoints and then its radii; avoid:
        int32 device tensor [B, n_obs], nonzero to avoid the obstacle.  None keeps that part.  Before
        the first call every shape is the problem's own and every obstacle is avoided.

        The first call attaches the obstacle state to the handle, which allocates and synchronises
        the device; every later call is stream-ordered and can be captured in a CUDA graph."""
        B, n_shape = self.B, self.shape_layout[1]
        if shapes is not None:
            b200._check_device_tensors((shapes,), self.lib)
            if tuple(shapes.shape) != (B, n_shape):
                raise ValueError('shapes must be [B, %d] = [%d, %d]' % (n_shape, B, n_shape))
        if avoid is not None:
            b200._check_int_tensors((avoid,))
            if tuple(avoid.shape) != (B, self.n_obs):
                raise ValueError('avoid must be [B, n_obs] = [%d, %d]' % (B, self.n_obs))
        ref = shapes if shapes is not None else avoid
        if not self._attached:
            D, keep = b200.pack_mpc_obstacles_desc(self._obstacles())
            self._check(self.lib.omg_mpc_attach_obstacles(self._handle, C.byref(D)))
            del keep
            self._attached = True
        if ref is None:
            return
        self._check(self.lib.omg_mpc_set_obstacles(
            self._handle, None if shapes is None else shapes.data_ptr(), None if avoid is None else avoid.data_ptr(),
            b200._stream_handle(ref.is_cuda, ref.device, stream)))

    def recover(self, mask):
        """Cold-start the instances with mask[b] true on their next update (Point2Point::recover)."""
        m = np.ascontiguousarray(np.broadcast_to(np.asarray(mask, dtype=bool), (self.B,)), dtype=np.int32)
        self._check(self.lib.omg_mpc_recover(self._handle, m.ctypes.data))

    @property
    def time(self):
        """Every instance's current time (numpy [B]; synchronises the device)."""
        t = np.empty(self.B)
        self._check(self.lib.omg_mpc_time(self._handle, t.ctypes.data))
        return t

    def motion_time(self, stream=None):
        """Every instance's motion time T of its last accepted plan (the template's before the first;
        the horizon with a fixed horizon): device tensor [B], without synchronising."""
        import torch
        T = torch.empty(self.B, dtype=torch.float64, device=self.dev)
        on_gpu = b200._check_device_tensors((T,), self.lib)
        self._check(self.lib.omg_mpc_motion_time(self._handle, T.data_ptr(),
                                                 b200._stream_handle(on_gpu, T.device, stream)))
        return T

    def last_problem(self, stream=None):
        """The warm start and parameter rows handed to the last solve: device tensors [B, n], [B, n_par]."""
        import torch
        x0 = torch.empty((self.B, self.n), dtype=torch.float64, device=self.dev)
        p = torch.empty((self.B, self.n_par), dtype=torch.float64, device=self.dev)
        on_gpu = b200._check_device_tensors((x0, p), self.lib)
        self._check(self.lib.omg_mpc_last_problem(self._handle, x0.data_ptr(), p.data_ptr(),
                                                  b200._stream_handle(on_gpu, x0.device, stream)))
        return x0, p

    def __del__(self):
        try:
            if getattr(self, '_handle', None):
                self.lib.omg_mpc_destroy(self._handle)
                self._handle = None
        except Exception:
            pass
