"""The numpy twin of omg_closed_loop_step_fleet (omg_tools_b200/csrc/omg_b200.cu): the plant step
of tests/plant_twin_ext.py for every vehicle of a fleet, vehicle v reading its input splines at
its own column offset of x and drawing its noise as signals v * n_input + j of the instance."""
import numpy as np

import plant_twin as tw
import plant_twin_ext as twx


def disturbance(seed, step, inst, sig0, n_sig, n_traj, fc, mean, stdev):
    """Filtered input disturbance [n_sig, n_traj] of signals sig0 .. sig0 + n_sig - 1."""
    from scipy.signal import butter, filtfilt
    b, a = butter(3, fc, 'low')
    return np.array([filtfilt(b, a, mean[k] + stdev[k] * tw.normals(seed, step, inst, sig0 + k, n_traj))
                     for k in range(n_sig)])


def plant_step(model, X, offsets, L, R, dt, plant_x, plant_u, step, seed=0,
               time_constant=None, disturbance_spec=None, instances=None):
    """The four outputs [B, n_veh, ·] of omg_closed_loop_step_fleet for every instance b of X [B, n]
    (global instance ids ``instances``, default 0..B-1); R = [n_der, n_samp + 1, L]."""
    B, nv = plant_x.shape[:2]
    ni = plant_u.shape[2]
    n_samp = R.shape[1] - 1
    inst = np.arange(B) if instances is None else np.asarray(instances)
    res = [np.zeros_like(plant_x), np.zeros_like(plant_u), np.zeros_like(plant_x), np.zeros_like(plant_u)]
    f = lambda x, u: twx.ode(model, x, u)
    for b in range(B):
        for v, off in enumerate(offsets):
            U = twx.planned_inputs(model, X[b, off:], L, R[0], R[1], ni, R[2:])
            A = U.copy()
            if disturbance_spec is not None:
                fc, mean, stdev, n_traj = disturbance_spec
                A = A + disturbance(seed, step, inst[b], v * ni, ni, n_traj, fc, mean, stdev)[:, :n_samp + 1].T
            if time_constant is not None:
                tau = time_constant
                A = tw.rk4(lambda u, c: (c - u) / tau, plant_u[b, v], A, dt)
            res[0][b, v] = tw.rk4(f, plant_x[b, v], A, dt)[-1]
            res[1][b, v] = A[-1]
            res[2][b, v] = tw.rk4(f, plant_x[b, v], U, dt)[-1]
            res[3][b, v] = U[-1]
    return res
