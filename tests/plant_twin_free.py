"""The numpy twin of omg_closed_loop_step_free: plant_twin_ext's plant step per instance, on the basis
rows of that instance's own motion time.  Instance b reads T_b = X[b, t_index], takes the rows of
BSplineBasis and its derivatives (divided by T_b^d) at s * sample_time / T_b for
s = 0..n_samp[b], and runs plant_step with its own n_samp and, with the disturbance, its own
n_traj (0: no disturbance).  An instance with n_samp[b] = 0 keeps the values it came with."""
import numpy as np

import plant_twin_ext as tw


def rows(basis, T, sample_time, n_samp, n_der=4):
    """[n_der, n_samp + 1, L]: the basis and its derivatives 1..n_der-1 (divided by T^d) at
    s * sample_time / T."""
    tau = sample_time * np.arange(n_samp + 1) / T
    out = [basis.eval_basis(tau)]
    for d in range(1, n_der):
        Bd, Pd = basis.derivative(d)
        out.append(Bd.eval_basis(tau).dot(Pd) / T**d)
    return np.array(out)


def plant_step_free(model, X, block, t_index, n_samp, sample_time, plant_x, plant_u, out, step, seed=0,
                    time_constant=None, disturbance_spec=None):
    """The four outputs of omg_closed_loop_step_free, starting from ``out`` (numpy copies of what the
    output buffers held).  block = (offset, L, columns, degree, knots); disturbance_spec =
    (fc, mean, stdev, n_traj [B])."""
    from omg_tools_b200.basics.spline import BSplineBasis
    off, L, nc, degree, knots = block
    basis = BSplineBasis(knots, degree)
    n_der = min(4, degree + 1)
    res = [np.array(o, dtype=float, copy=True) for o in out]
    for b in range(X.shape[0]):
        if n_samp[b] == 0:
            continue
        T = X[b, t_index]
        R = rows(basis, T, sample_time, int(n_samp[b]), n_der)
        spec = None
        if disturbance_spec is not None and disturbance_spec[3][b] > 0:
            fc, mean, stdev, n_traj = disturbance_spec
            spec = (fc, mean, stdev, int(n_traj[b]))
        r = tw.plant_step(model, X[b:b + 1, off:off + nc * L], L, R[0], R[1], sample_time, plant_x[b:b + 1],
                          plant_u[b:b + 1], step, seed=seed, time_constant=time_constant, disturbance_spec=spec,
                          instances=[b], higher=R[2:])
        for o, v in zip(res, r):
            o[b] = v[0]
    return res
