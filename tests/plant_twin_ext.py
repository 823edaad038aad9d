"""The numpy twin of omg_closed_loop_step (tests/plant_twin.py) for every vehicle model of
omg_closed_loop_step_der: plant_twin's generator, filter, RK4 and lag rules, with the planned
inputs and the ODEs of the planar Quadrotor (model 2), Dubins (3), HolonomicOrient (4) and
SimpleQuadrotor3D (5) added, written from the vehicles' splines2signals and ode.  Models 0 and 1
are plant_twin's own."""
import numpy as np

import plant_twin as tw

G = 9.81


def planned_inputs(model, coeffs, L, R0, R1, n_input, higher=None):
    """Planned input samples [n_samp+1, n_input] of one instance (splines2signals): (v, omega)
    for Dubins, (x', y', theta') for HolonomicOrient, and the quadrotors' inputs from the second
    and third derivatives higher = [R2, R3] of the position splines."""
    col = lambda c: coeffs[c * L:(c + 1) * L]
    if model == 2:                      # quadrotor.py
        (ddx, ddy), (dddx, dddy) = [[R.dot(col(c)) for c in range(2)] for R in higher[:2]]
        ay = ddy + G
        return np.c_[np.sqrt(ddx**2 + ay**2), (dddx * ay - ddx * dddy) / (ay**2 + ddx**2)]
    if model == 3:                      # dubins.py
        vt, tg, dtg = R0.dot(col(0)), R0.dot(col(1)), R1.dot(col(1))
        return np.c_[vt * (1 + tg**2), 2 * dtg / (1 + tg**2)]
    if model == 4:                      # holonomicorient.py
        tg = R0.dot(col(2))
        return np.c_[R1.dot(col(0)), R1.dot(col(1)), 2 * R1.dot(col(2)) / (1 + tg**2)]
    if model == 5:                      # quadrotor3d_simple.py
        (ddx, ddy, ddz), (dddx, dddy, dddz) = [[R.dot(col(c)) for c in range(3)] for R in higher[:2]]
        az = ddz + G
        u1 = np.sqrt(ddx**2 + ddy**2 + az**2)
        u2 = (-dddy * (ddx**2 + az**2) + ddy * (ddx * dddx + dddz * az)) / \
            ((ddx**2 + ddy**2 + az**2) * np.sqrt(ddx**2 + az**2))
        return np.c_[u1, u2, (az * dddx - ddx * dddz) / (az**2 + ddx**2)]
    return tw.planned_inputs(model, coeffs, L, R0, R1, n_input)


def ode(model, x, u):
    if model == 5:                      # Quadrotor3D's ODE
        return tw.ode(1, x, u, G)
    if model == 2:
        return np.array([x[2], x[3], u[0] * np.sin(x[4]), u[0] * np.cos(x[4]) - G, u[1]])
    if model == 3:
        return np.array([u[0] * np.cos(x[2]), u[0] * np.sin(x[2]), u[1]])
    return tw.ode(model, x, u, G)       # 0, 1, and 4 (integrator)


def plant_step(model, X, L, R0, R1, dt, plant_x, plant_u, step, seed=0,
               time_constant=None, disturbance_spec=None, instances=None, higher=None):
    """plant_twin.plant_step for every model; higher = the rows of derivatives 2 and 3."""
    B = X.shape[0]
    ni = plant_u.shape[1]
    n_samp = R0.shape[0] - 1
    inst = np.arange(B) if instances is None else np.asarray(instances)
    res = [np.zeros_like(plant_x), np.zeros_like(plant_u), np.zeros_like(plant_x), np.zeros_like(plant_u)]
    f = lambda x, u: ode(model, x, u)
    for b in range(B):
        U = planned_inputs(model, X[b], L, R0, R1, ni, higher)
        A = U.copy()
        if disturbance_spec is not None:
            fc, mean, stdev, n_traj = disturbance_spec
            A = A + tw.disturbance(seed, step, inst[b], ni, n_traj, fc, mean, stdev)[:, :n_samp + 1].T
        if time_constant is not None:
            tau = time_constant
            A = tw.rk4(lambda u, c: (c - u) / tau, plant_u[b], A, dt)
        res[0][b] = tw.rk4(f, plant_x[b], A, dt)[-1]
        res[1][b] = A[-1]
        res[2][b] = tw.rk4(f, plant_x[b], U, dt)[-1]
        res[3][b] = U[-1]
    return res
