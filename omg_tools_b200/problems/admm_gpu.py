"""Device-resident, multi-GPU execution of the formation ADMM iteration.

Agents are sharded contiguously over the ranks (one process per GPU).  One ADMM
iteration = reference ``ADMMProblem.dual_update`` (admm.py:584-628):

    init_step     knot shift of x, z, l copies            (admm.py:477-491)
    update_x      ONE batched NLP solve (omg_solve_batch)  (admm.py:383-398)
    communicate   x_j <- neighbours' x_i        [NCCL all-gather]   (468-475)
    update_z/l    ONE kernel (omg_admm_zl_update)          (407-466, 493-508)
    residuals     sum over agents               [NCCL all-reduce, 3 doubles] (597-605)
    accelerate    optional Nesterov extrapolation of z, l  (admm.py:510-554)
    communicate   z_ji, l_ji <- neighbours' z_ij, l_ij     [NCCL all-gather]

The exchange is the only collective of the framework; message sizes are tiny
(26 doubles per agent and neighbour), so it is latency bound and a plain
all-gather over NVLink serves every interconnection topology of ``Fleet``.
"""
import numpy as np


class AgentExchange(object):
    """Neighbour exchange for contiguous agent shards (any torch device /
    backend: NCCL on GPUs, gloo in the CPU tests)."""

    def __init__(self, n_agents, nghb, back, rank=0, world=1, group=None):
        import torch
        self.torch = torch
        self.N, self.rank, self.world, self.group = n_agents, rank, world, group
        if n_agents % world != 0:
            raise ValueError('number of agents must be a multiple of the number of ranks')
        self.per = n_agents // world
        self.lo, self.hi = rank * self.per, (rank + 1) * self.per
        self.nghb_np, self.back_np = np.asarray(nghb), np.asarray(back)
        self._idx = {}

    def _index(self, device):
        key = str(device)
        if key not in self._idx:
            t = self.torch
            ng = t.as_tensor(self.nghb_np[self.lo:self.hi], device=device)
            bk = t.as_tensor(self.back_np[self.lo:self.hi], device=device)
            self._idx[key] = (ng, bk)
        return self._idx[key]

    def _all_gather(self, local):
        t = self.torch
        if self.world == 1:
            return local
        out = t.empty((self.world * local.shape[0],) + tuple(local.shape[1:]),
                      dtype=local.dtype, device=local.device)
        import torch.distributed as dist
        dist.all_gather_into_tensor(out, local.contiguous(), group=self.group)
        return out

    def gather_x(self, x_i_local):
        """x_j[i, k] = x_i of the k-th neighbour of local agent i."""
        ng, _ = self._index(x_i_local.device)
        allx = self._all_gather(x_i_local)
        return allx[ng].contiguous()

    def gather_zl(self, z_ij_local, l_ij_local):
        """z_ji[i, k] = z_ij held by neighbour j = nghb[i, k] for agent i."""
        ng, bk = self._index(z_ij_local.device)
        allz = self._all_gather(z_ij_local)
        alll = self._all_gather(l_ij_local)
        return allz[ng, bk].contiguous(), alll[ng, bk].contiguous()

    def allreduce_sum(self, vec):
        if self.world > 1:
            import torch.distributed as dist
            dist.all_reduce(vec, group=self.group)
        return vec


class FormationADMMRunner(object):
    """Runs ``FormationPoint2point`` (problems/admm.py) on this rank's GPU."""

    def __init__(self, problem, rank=0, world=1, group=None, device=None, formations=1, spread=0.):
        """``formations`` > 1 runs that many independent copies of the formation side by side:
        agent a of copy f is global agent f*N + a, its neighbours are offset the same way, so one
        x-update launch, one consensus kernel and one set of collectives advance all copies by one
        ADMM iteration (one 64-agent formation leaves most of a GPU's resident blocks idle).
        ``spread`` perturbs copy f's initial guess (relative, seeded by f) so the copies do not
        iterate in lock step.  ``formation_residuals()`` gives the residuals per copy."""
        import torch
        from ..solver import b200
        self.torch, self.b200 = torch, b200
        self.pr = problem
        self.solver = problem.solver
        self.formations, F, N = int(formations), int(formations), problem.N
        if F > 1:
            problem = _Tiled(problem, F, spread)
        self.ex = AgentExchange(N * F, problem.nghb, problem.back, rank, world, group)
        lo, hi = self.ex.lo, self.ex.hi
        self.lo, self.hi = lo, hi
        dev = device if isinstance(device, torch.device) else \
            torch.device('cuda', self.solver.device if device is None else device)
        self.dev = dev
        td = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)
        p = problem
        self.X = td(p.X[lo:hi])
        self.Xn = torch.empty_like(self.X)
        self.x_i, self.z_i, self.l_i = td(p.x_i[lo:hi]), td(p.z_i[lo:hi]), td(p.l_i[lo:hi])
        self.x_j, self.z_ij, self.l_ij = td(p.x_j[lo:hi]), td(p.z_ij[lo:hi]), td(p.l_ij[lo:hi])
        self.z_ji, self.l_ji = td(p.z_ji[lo:hi]), td(p.l_ji[lo:hi])
        self.c = td(p.c[lo:hi])
        self.PzT = td(p.Pz.T)
        self.Ts = td(shift_T(p))
        n_loc, m = hi - lo, p.tb.m
        self.LAM = torch.empty((n_loc, m), dtype=torch.float64, device=dev)
        self.F = torch.empty(n_loc, dtype=torch.float64, device=dev)
        self.ST = torch.empty(n_loc, dtype=torch.int32, device=dev)
        self.IT = torch.empty(n_loc, dtype=torch.int32, device=dev)
        self.LB, self.UB = td(p.tb.lbg), td(p.tb.ubg)
        self.res = torch.zeros((n_loc, 3), dtype=torch.float64, device=dev)
        self.P = torch.empty((n_loc, p.tb.n_par), dtype=torch.float64, device=dev)
        self.blocks = [(off, shape[0], shape[1], T) for (_, _, off, shape, T)
                       in p.father.shifted_entries()]
        self.time_prev = 0.
        self.history = []
        self.alpha, self.c_res_p = 1., None      # Nesterov state
        # on GPUs the exchange runs inside the C ABI (omg_admm_exchange_x / omg_admm_zl_update_dist:
        # NCCL all-gather + index kernel + residual all-reduce, one stream, no host round trip);
        # the torch.distributed exchange above serves the gloo CPU tests
        self.comm = None
        self._par_t = None
        self._tf_t = None
        if dev.type == 'cuda' and not bool(problem.options.get('nesterov_acceleration')):
            self.comm = b200.AdmmComm(rank, world, dev.index, group)
            self.nghb_d = torch.as_tensor(np.ascontiguousarray(problem.nghb[lo:hi], dtype=np.int32), device=dev)
            self.back_d = torch.as_tensor(np.ascontiguousarray(problem.back[lo:hi], dtype=np.int32), device=dev)
            self.res_total = torch.zeros(3, dtype=torch.float64, device=dev)

    # ------------------------------------------------------------------
    def _pack_parameters(self, t):
        """Host builds the constant part; consensus parameters are written on
        the device (they never leave it)."""
        p, torch = self.pr, self.torch
        if self._par_t != t:            # the host part only changes with the time
            host = np.tile(p.pack_parameters(t), (self.formations, 1))[self.lo:self.hi]
            self._P_host = torch.from_numpy(np.ascontiguousarray(host)).to(self.dev)
            self._par_t = t
        self.P.copy_(self._P_host)
        off, a = p.par_off, p.upd_label
        n_loc, nsh, nn = self.hi - self.lo, p.nsh, p.n_nghb
        self.P[:, off[(a, 'z_i')]:off[(a, 'z_i')] + nsh] = self.z_i
        self.P[:, off[(a, 'z_ji')]:off[(a, 'z_ji')] + nsh * nn] = self.z_ji.reshape(n_loc, -1)
        self.P[:, off[(a, 'l_i')]:off[(a, 'l_i')] + nsh] = self.l_i
        self.P[:, off[(a, 'l_ji')]:off[(a, 'l_ji')] + nsh * nn] = self.l_ji.reshape(n_loc, -1)

    def _shift_over_knot(self):
        L = self.pr.L
        Ts = self.Ts
        for name in ('x_i', 'z_i', 'l_i', 'x_j', 'z_ij', 'l_ij', 'z_ji', 'l_ji'):
            a = getattr(self, name)
            setattr(self, name, (a.reshape(-1, L) @ Ts.T).reshape(a.shape).contiguous())
        self.solver.shift_batch_device(self.X, self.blocks)

    def dual_update(self, t, fetch=True):
        """One ADMM iteration at (relative) time t; returns (p_res, d_res, c_res) -- or, with
        fetch=False on the native path, nothing: the residuals stay on the device
        (``self.res_total``) and the iteration needs no host synchronisation."""
        p, torch = self.pr, self.torch
        if (t > 0. and int(np.round(self.time_prev / p.knot_time, 6)) <
                int(np.round(t / p.knot_time, 6))):
            self._shift_over_knot()
        self.time_prev = t
        # x-update: one batched NLP solve for all local agents
        self._pack_parameters(t)
        self.solver.solve_batch_device(self.X, self.P, self.LB, self.UB, self.Xn, self.LAM,
                                       self.F, self.ST, self.IT)
        self.X, self.Xn = self.Xn, self.X
        self.x_i = self.X[:, p.x_off:p.x_off + p.nsh].contiguous()
        if self._tf_t != t:
            Tf, Tb = p.first_knot_transforms(t)
            self._Tf_d = torch.tensor(Tf, dtype=torch.float64, device=self.dev)
            self._Tb_d = torch.tensor(Tb, dtype=torch.float64, device=self.dev)
            self._tf_t = t
        Tf_d, Tb_d = self._Tf_d, self._Tb_d
        if self.comm is not None:
            # exchange 1, consensus kernel, residual all-reduce, exchange 2: all inside the C ABI
            self.comm.exchange_x(self.nghb_d, self.x_i, self.x_j)
            self.comm.zl_update(self.PzT, self.c, Tf_d, Tb_d, p.options['rho'], self.x_i, self.x_j,
                                self.z_i, self.z_ij, self.l_i, self.l_ij, self.res, p.L,
                                self.nghb_d, self.back_d, self.z_ji, self.l_ji, self.res_total)
            if not fetch:
                return None
            tot = self.res_total.cpu().numpy()
            out = (float(np.sqrt(tot[0])), float(np.sqrt(tot[1])), float(tot[2]))
            self.history.append(out)
            return out
        # communicate x
        self.x_j = self.ex.gather_x(self.x_i)
        # z / lambda / residuals
        nesterov = bool(p.options.get('nesterov_acceleration'))
        if nesterov:
            prev = [a.clone() for a in (self.z_i, self.z_ij, self.l_i, self.l_ij)]
        self.b200.admm_zl_update(self.PzT, self.c, Tf_d, Tb_d, p.options['rho'], self.x_i,
                                 self.x_j, self.z_i, self.z_ij, self.l_i, self.l_ij,
                                 self.res, p.L)
        tot = self.ex.allreduce_sum(self.res.sum(0))
        if nesterov:
            # fast ADMM: the combined residual is global (same decision on every rank)
            c_res, eta = float(tot[2]), p.options.get('eta', 0.999)
            if self.c_res_p is None:
                self.c_res_p = c_res / eta
            if (not p.options.get('nesterov_reset')) or c_res <= eta * self.c_res_p:
                alpha_p = self.alpha
                self.alpha = 0.5 * (1. + np.sqrt(1. + 4. * alpha_p**2))
                w = (alpha_p - 1.) / self.alpha
                for name, old in zip(('z_i', 'z_ij', 'l_i', 'l_ij'), prev):
                    if p.options.get('AMA') and name.startswith('z'):
                        continue            # AMA extrapolates the multipliers only (admm.py:527-541)
                    a = getattr(self, name)
                    a.add_(a - old, alpha=w)
                self.c_res_p = c_res
            else:
                self.alpha = 1.
                for name, old in zip(('z_i', 'z_ij', 'l_i', 'l_ij'), prev):
                    getattr(self, name).copy_(old)
                self.c_res_p = self.c_res_p / eta
        # communicate z, l
        self.z_ji, self.l_ji = self.ex.gather_zl(self.z_ij, self.l_ij)
        tot = tot.cpu().numpy()
        out = (float(np.sqrt(tot[0])), float(np.sqrt(tot[1])), float(tot[2]))
        self.history.append(out)
        return out

    def status(self):
        return self.ST.cpu().numpy(), self.IT.cpu().numpy()

    def formation_residuals(self):
        """(formations, 3) primal / dual / combined residual of each copy from the per-agent
        contributions of the last iteration (all ranks; a host read)."""
        res = self.res
        if self.ex.world > 1:
            res = self.ex._all_gather(res)
        tot = res.reshape(self.formations, -1, 3).sum(1).cpu().numpy()
        return np.stack([np.sqrt(tot[:, 0]), np.sqrt(tot[:, 1]), tot[:, 2]], axis=1)


class _Tiled(object):
    """The arrays of a formation problem repeated for F side-by-side copies (views the runner
    reads once at construction); everything else is the problem's."""

    def __init__(self, problem, F, spread):
        self._p = problem
        N = problem.N
        for name in ('X', 'x_i', 'z_i', 'l_i', 'x_j', 'z_ij', 'l_ij', 'z_ji', 'l_ji', 'c'):
            a = np.asarray(getattr(problem, name))
            setattr(self, name, np.tile(a, (F,) + (1,) * (a.ndim - 1)))
        if spread:
            for f in range(1, F):
                rng = np.random.RandomState(f)
                self.X[f * N:(f + 1) * N] *= 1. + spread * rng.uniform(-1., 1., self.X[:N].shape)
        off = (np.arange(F) * N).repeat(N)[:, None]
        self.nghb = np.tile(np.asarray(problem.nghb), (F, 1)) + off
        self.back = np.tile(np.asarray(problem.back), (F, 1))

    def __getattr__(self, name):
        return getattr(self._p, name)


def shift_T(problem):
    """Knot-crossing transformation of the shared blocks (identity for a RendezVous)."""
    if hasattr(problem, 'shared_shift_T'):
        return problem.shared_shift_T()
    from ..basics.spline_extra import shiftoverknot_T
    return shiftoverknot_T(problem.basis)


class FormationDDRunner(object):
    """Runs ``FormationPoint2pointDualDecomposition`` (problems/dualdecomposition.py) on this
    rank's GPU.  One iteration = reference ``DDProblem.dual_update`` (dualdecomposition.py:279-314):

        init_step     knot shift of x_i, x_j, z_ij, l_ij, l_ji and of the NLP's variables
        update_xz     ONE batched NLP solve (omg_solve_batch): own trajectory + neighbour copies
        communicate   x_j <- neighbours' x_i                    [NCCL all-gather, C ABI]
        update_l      l_ij += rho (x_j - z_ij), residual ||Tf (x_j - z_ij)||^2   (elementwise, device)
        communicate   l_ji <- neighbours' l_ij                  [NCCL all-gather, C ABI]
    """

    def __init__(self, problem, rank=0, world=1, group=None, device=None):
        import torch
        from ..solver import b200
        self.torch, self.b200 = torch, b200
        self.pr = p = problem
        self.solver = problem.solver
        self.ex = AgentExchange(p.N, p.nghb, p.back, rank, world, group)
        lo, hi = self.ex.lo, self.ex.hi
        self.lo, self.hi = lo, hi
        dev = device if isinstance(device, torch.device) else \
            torch.device('cuda', self.solver.device if device is None else device)
        self.dev = dev
        td = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, device=dev)
        self.X = td(p.X[lo:hi])
        self.Xn = torch.empty_like(self.X)
        self.x_i, self.x_j, self.z_ij = td(p.x_i[lo:hi]), td(p.x_j[lo:hi]), td(p.z_ij[lo:hi])
        self.l_ij, self.l_ji = td(p.l_ij[lo:hi]), td(p.l_ji[lo:hi])
        n_loc, m = hi - lo, p.tb.m
        self.LAM = torch.empty((n_loc, m), dtype=torch.float64, device=dev)
        self.F = torch.empty(n_loc, dtype=torch.float64, device=dev)
        self.ST = torch.empty(n_loc, dtype=torch.int32, device=dev)
        self.IT = torch.empty(n_loc, dtype=torch.int32, device=dev)
        self.LB, self.UB = td(p.tb.lbg), td(p.tb.ubg)
        self.P = torch.empty((n_loc, p.tb.n_par), dtype=torch.float64, device=dev)
        self.blocks = [(off, shape[0], shape[1], T) for (_, _, off, shape, T) in p.father.shifted_entries()]
        self.Ts = td(shift_T(p))
        self.time_prev = 0.
        self.history = []
        self._par_t = self._tf_t = None
        self.comm = None
        if dev.type == 'cuda':
            self.comm = b200.AdmmComm(rank, world, dev.index, group)
            nn = p.n_nghb
            self.nghb_d = torch.as_tensor(np.ascontiguousarray(p.nghb[lo:hi], dtype=np.int32), device=dev)
            # rows of the all-gathered l_ij, seen as (N * nn, nsh): what neighbour j holds for agent i
            rows = (p.nghb[lo:hi] * nn + p.back[lo:hi]).reshape(-1, 1)
            self.lrow_d = torch.as_tensor(np.ascontiguousarray(rows, dtype=np.int32), device=dev)

    def _pack_parameters(self, t):
        p, torch = self.pr, self.torch
        if self._par_t != t:
            host = p.pack_parameters(t)[self.lo:self.hi]
            self._P_host = torch.from_numpy(np.ascontiguousarray(host)).to(self.dev)
            self._par_t = t
        self.P.copy_(self._P_host)
        off, a = p.par_off, p.upd_label
        n_loc, w = self.hi - self.lo, p.nsh * p.n_nghb
        self.P[:, off[(a, 'l_ij')]:off[(a, 'l_ij')] + w] = self.l_ij.reshape(n_loc, -1)
        self.P[:, off[(a, 'l_ji')]:off[(a, 'l_ji')] + w] = self.l_ji.reshape(n_loc, -1)

    def _shift_over_knot(self):
        L, Ts, p = self.pr.L, self.Ts, self.pr
        for name in ('x_i', 'x_j', 'z_ij', 'l_ij', 'l_ji'):
            a = getattr(self, name)
            setattr(self, name, (a.reshape(-1, L) @ Ts.T).reshape(a.shape).contiguous())
        self.solver.shift_batch_device(self.X, self.blocks)
        self.X[:, p.z_off:p.z_off + p.nsh * p.n_nghb] = self.z_ij.reshape(self.X.shape[0], -1)

    def dual_update(self, t):
        """One dual decomposition iteration at (relative) time t; returns the primal residual."""
        p, torch = self.pr, self.torch
        if (t > 0. and int(np.round(self.time_prev / p.knot_time, 6)) < int(np.round(t / p.knot_time, 6))):
            self._shift_over_knot()
        self.time_prev = t
        self._pack_parameters(t)
        self.solver.solve_batch_device(self.X, self.P, self.LB, self.UB, self.Xn, self.LAM,
                                       self.F, self.ST, self.IT)
        self.X, self.Xn = self.Xn, self.X
        n_loc, nn, nsh = self.X.shape[0], p.n_nghb, p.nsh
        st = self.ST.cpu().numpy()
        bad = np.nonzero(st == 2)[0]
        if len(bad):
            # Restoration_Failed (the cold xz-update of an agent can end there): these instances go
            # once more through the host call, which adds the feasibility phase and the re-solve
            # (solver/b200.py: solve_batch) -- what IPOPT's restoration does inside the same nlpsol call
            idx = torch.as_tensor(bad, device=self.dev)
            r = self.solver.solve_batch(self.Xn[idx].cpu().numpy(), self.P[idx].cpu().numpy())
            self.X[idx] = torch.tensor(r['x'], dtype=torch.float64, device=self.dev)
            self.ST[idx] = torch.tensor(r['status'], dtype=torch.int32, device=self.dev)
            self.IT[idx] = torch.tensor(r['iters'], dtype=torch.int32, device=self.dev)
        self.x_i = self.X[:, p.x_off:p.x_off + nsh].contiguous()
        self.z_ij = self.X[:, p.z_off:p.z_off + nsh * nn].reshape(n_loc, nn, nsh).contiguous()
        if self.comm is not None:
            self.comm.exchange_x(self.nghb_d, self.x_i, self.x_j)
        else:
            self.x_j = self.ex.gather_x(self.x_i)
        if self._tf_t != t:
            Tf, _ = p.first_knot_transforms(t)
            self._Tf_d = torch.tensor(Tf, dtype=torch.float64, device=self.dev)
            self._tf_t = t
        d = self.x_j - self.z_ij
        self.l_ij = (self.l_ij + p.options['rho'] * d).contiguous()
        e = d.reshape(-1, p.L) @ self._Tf_d.T
        tot = self.ex.allreduce_sum((e * e).sum().reshape(1))
        if self.comm is not None:
            flat_in = self.l_ij.reshape(n_loc * nn, nsh)
            flat_out = self.l_ji.reshape(n_loc * nn, 1, nsh)
            self.comm.exchange_x(self.lrow_d, flat_in, flat_out)
        else:
            _, self.l_ji = self.ex.gather_zl(self.l_ij, self.l_ij)
        out = float(np.sqrt(float(tot[0])))
        self.history.append(out)
        return out

    def status(self):
        return self.ST.cpu().numpy(), self.IT.cpu().numpy()
