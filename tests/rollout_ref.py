"""Float64 reference for DHRobot.rollout / Robot.rollout: classical RK4 under a zero-order-hold torque, with the
sensitivities chained through the four stages from a reference accel_derivatives (rne_derivs_ref for DH arms,
tree_derivs_ref for trees), and, for trees, the complex step of the whole discrete map, which gives A_k and B_k without
the composition formula.  Every function works on a batch: x (N, 2n), tau (N, n)."""
import numpy as np

import rne_derivs_ref as dref
import tree_derivs_ref as tref


def step(accel, x, tau, dt):
    """One RK4 step of x = [q; qd] (dtype-generic: runs on complex numbers when accel does)."""
    n = tau.shape[1]
    f = lambda y: np.concatenate([y[:, n:], accel(y[:, :n], y[:, n:], tau)], axis=1)  # noqa: E731
    k1 = f(x)
    k2 = f(x + dt / 2 * k1)
    k3 = f(x + dt / 2 * k2)
    k4 = f(x + dt * k3)
    return x + dt / 6 * (k1 + 2 * k2 + 2 * k3 + k4)


def chained_step(accel, accel_derivs, x, tau, dt):
    """(x_{k+1}, A_k, B_k) with dk_i/dx = J_f(x_i) (I + c_i dt dk_{i-1}/dx), dk_i/dtau = J_f(x_i) c_i dt dk_{i-1}/dtau +
    [0; M^-1(x_i)], J_f = [[0, I], [dqdd_dq, dqdd_dqd]]."""
    N, n = tau.shape
    I = np.eye(2 * n)
    ks, dxs, dts = [], [], []
    for c in (0.0, 0.5, 0.5, 1.0):
        xs = x if not ks else x + c * dt * ks[-1]
        Sx = I if not ks else I + c * dt * dxs[-1]
        St = np.zeros((N, 2 * n, n)) if not ks else c * dt * dts[-1]
        aq, aqd, at = accel_derivs(xs[:, :n], xs[:, n:], tau)
        J = np.zeros((N, 2 * n, 2 * n))
        J[:, :n, n:] = np.eye(n)
        J[:, n:, :n], J[:, n:, n:] = aq, aqd
        ks.append(np.concatenate([xs[:, n:], accel(xs[:, :n], xs[:, n:], tau)], axis=1))
        dxs.append(J @ Sx)
        dts.append(J @ St + np.concatenate([np.zeros((N, n, n)), at], axis=1))
    w = (1, 2, 2, 1)
    xn = x + dt / 6 * sum(wi * k for wi, k in zip(w, ks))
    A = I + dt / 6 * sum(wi * d for wi, d in zip(w, dxs))
    B = dt / 6 * sum(wi * d for wi, d in zip(w, dts))
    return xn, A, B


def rollout(model, q0, qd0, tau, dt, sensitivities=True):
    """model = (accel, accel_derivs); q0, qd0 (N, n); tau (N, K, n).  Returns q, qd (N, K+1, n) and A (N, K, 2n, 2n),
    B (N, K, 2n, n) (None without sensitivities)."""
    accel, accel_derivs = model
    n = q0.shape[1]
    x = np.concatenate([q0, qd0], axis=1).astype(np.float64)
    xs, As, Bs = [x], [], []
    for k in range(tau.shape[1]):
        if sensitivities:
            x, A, B = chained_step(accel, accel_derivs, x, tau[:, k], dt)
            As.append(A)
            Bs.append(B)
        else:
            x = step(accel, x, tau[:, k], dt)
        xs.append(x)
    X = np.stack(xs, axis=1)
    if not sensitivities:
        return X[..., :n], X[..., n:], None, None
    return X[..., :n], X[..., n:], np.stack(As, axis=1), np.stack(Bs, axis=1)


def dh(L, mdh, grav):
    """The model of a packed DH link table; grav = MINUS the robot's gravity, as the kernels take it.  The derivatives are
    Richardson differences of the oracle's accel (rne_derivs_ref): relative accuracy about 1e-8."""
    return (lambda q, qd, t: dref.accel(L, mdh, grav, q, qd, t),
            lambda q, qd, t: dref.accel_derivatives(L, mdh, grav, q, qd, t))


def tree(desc, gravity):
    """The model of a tree description; gravity = the robot's gravity.  Complex-step derivatives, exact to rounding."""
    def accel(q, qd, t):
        return np.stack([tref.accel(desc, q[i], qd[i], t[i], gravity) for i in range(len(q))])

    def accel_derivs(q, qd, t):
        d = [tref.accel_derivatives(desc, q[i], qd[i], t[i], gravity) for i in range(len(q))]
        return tuple(np.stack([x[j] for x in d]) for j in range(3))

    return accel, accel_derivs


def complex_step(accel, x, tau, dt, h=1e-30):
    """(A, B) of one RK4 step, (N, 2n, 2n) and (N, 2n, n), by the complex step of the whole map (accel must run on complex
    numbers, as tree(...)[0] does)."""
    N, n = tau.shape
    A = np.empty((N, 2 * n, 2 * n))
    B = np.empty((N, 2 * n, n))
    for j in range(2 * n):
        e = np.zeros(2 * n, dtype=complex)
        e[j] = 1j * h
        A[:, :, j] = step(accel, x + e, tau.astype(complex), dt).imag / h
    for j in range(n):
        e = np.zeros(n, dtype=complex)
        e[j] = 1j * h
        B[:, :, j] = step(accel, x.astype(complex), tau + e, dt).imag / h
    return A, B
