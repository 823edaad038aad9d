"""numpy restatement of omg_closed_loop_step (omg_tools_b200/csrc/omg_b200.cu): the
closed-loop plant step of execution/batch_mpc.py, written from the reference's
Vehicle.simulate / predict / add_disturbance (vehicle.py:302-337, 359-449).

- The white noise comes from the same counter-based generator: Philox4x32-10 keyed by the seed,
  counter (sample pair, signal, instance, MPC step), two 52-bit uniforms per block, Box-Muller.
  The uniforms are bit-identical to the kernel's; the normals differ by the last bits of log,
  cos and sin.
- The filter is scipy.signal.filtfilt itself, on butter(3, fc), over the whole stored
  trajectory (n_traj samples), as the reference filters it.
- RK4 and the first-order lag follow the kernel's rule: the linearly interpolated input
  (u_i; (u_i + u_i+1)/2 at both midpoints; u_i+1) of the reference's interp1d."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """ctr: uint64 array [..., 4] of 32-bit words; key: (k0, k1).  Returns [..., 4] (uint64)."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(10):
        if r:
            k0, k1 = np.uint64((int(k0) + W0) & MASK), np.uint64((int(k1) + W1) & MASK)
        p0, p1 = np.uint64(M0) * c[0], np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, axis=-1)


def uniforms(seed, step, inst, sig, n):
    """(u1, u2) of the ceil(n/2) Philox blocks of one series, in (0, 1)."""
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    npair = (n + 1) // 2
    ctr = np.zeros((npair, 4), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3] = np.arange(npair), sig, inst, step
    c = philox4x32_10(ctr, (seed & MASK, seed >> 32))
    s32, s12 = np.uint64(32), np.uint64(12)
    m1 = ((c[:, 0] << s32) | c[:, 1]) >> s12
    m2 = ((c[:, 2] << s32) | c[:, 3]) >> s12
    return (m1.astype(np.float64) + 0.5) * 2.0**-52, (m2.astype(np.float64) + 0.5) * 2.0**-52


def normals(seed, step, inst, sig, n):
    u1, u2 = uniforms(seed, step, inst, sig, n)
    r, w = np.sqrt(-2.0 * np.log(u1)), 6.283185307179586 * u2
    return np.stack([r * np.cos(w), r * np.sin(w)], axis=1).reshape(-1)[:n]


def disturbance(seed, step, inst, n_sig, n_traj, fc, mean, stdev):
    """Filtered input disturbance [n_sig, n_traj] (reference add_disturbance)."""
    from scipy.signal import butter, filtfilt
    b, a = butter(3, fc, 'low')
    return np.array([filtfilt(b, a, mean[k] + stdev[k] * normals(seed, step, inst, k, n_traj))
                     for k in range(n_sig)])


def planned_inputs(model, coeffs, L, R0, R1, n_input):
    """Planned input samples [n_samp+1, n_input] of one instance (splines2signals): ds/dt for
    the integrator model, thrust and angular rates from f~, q_phi, q_theta for Quadrotor3D."""
    col = lambda c: coeffs[c * L:(c + 1) * L]
    if model == 1:
        f, qp, qt = R0.dot(col(0)), R0.dot(col(1)), R0.dot(col(2))
        dqp, dqt = R1.dot(col(1)), R1.dot(col(2))
        ep, et = 1. + qp * qp, 1. + qt * qt
        return np.c_[f * (ep * et), 2. * dqp / ep, 2. * dqt / et]
    return np.array([R1.dot(col(c)) for c in range(n_input)]).T


def ode(model, x, u, g=9.81):
    if model == 1:
        phi, theta = x[6], x[7]
        return np.array([x[3], x[4], x[5], u[0] * np.sin(theta) * np.cos(phi), -u[0] * np.sin(phi),
                         -g + u[0] * np.cos(phi) * np.cos(theta), u[1], u[2]])
    return np.array(u, dtype=float)


def rk4(f, x, U, dt):
    """RK4 over the samples U [ns+1, ...] on their linear interpolation; returns the samples."""
    out = [np.array(x, dtype=float)]
    for i in range(U.shape[0] - 1):
        um = 0.5 * (U[i] + U[i + 1])
        k1 = f(x, U[i])
        k2 = f(x + 0.5 * dt * k1, um)
        k3 = f(x + 0.5 * dt * k2, um)
        k4 = f(x + dt * k3, U[i + 1])
        x = x + (dt / 6.0) * (k1 + 2.0 * k2 + 2.0 * k3 + k4)
        out.append(x)
    return np.array(out)


def plant_step(model, X, L, R0, R1, dt, plant_x, plant_u, step, seed=0,
               time_constant=None, disturbance_spec=None, instances=None):
    """The four outputs of omg_closed_loop_step for every instance b of X [B, n] (global
    instance ids ``instances``, default 0..B-1).  disturbance_spec = (fc, mean, stdev, n_traj)."""
    B = X.shape[0]
    ni = plant_u.shape[1]
    n_samp = R0.shape[0] - 1
    inst = np.arange(B) if instances is None else np.asarray(instances)
    res = [np.zeros_like(plant_x), np.zeros_like(plant_u), np.zeros_like(plant_x), np.zeros_like(plant_u)]
    for b in range(B):
        U = planned_inputs(model, X[b], L, R0, R1, ni)
        A = U.copy()
        if disturbance_spec is not None:
            fc, mean, stdev, n_traj = disturbance_spec
            A = A + disturbance(seed, step, inst[b], ni, n_traj, fc, mean, stdev)[:, :n_samp + 1].T
        if time_constant is not None:
            tau = time_constant
            lagf = lambda u, c: (c - u) / tau
            A = rk4(lagf, plant_u[b], A, dt)
        res[0][b] = rk4(lambda x, u: ode(model, x, u), plant_x[b], A, dt)[-1]
        res[1][b] = A[-1]
        res[2][b] = rk4(lambda x, u: ode(model, x, u), plant_x[b], U, dt)[-1]
        res[3][b] = U[-1]
    return res
