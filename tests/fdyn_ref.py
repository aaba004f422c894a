"""Reference side of the device forward-dynamics integrator (k_fdyn behind DHRobot.fdyn / Robot.fdyn).

The reference is scipy's RK45 stepped exactly as oracle.fdyn steps it (DynamicsMixin.fdyn restated: one accepted step
per `step()`, the start state first, `interp1d` onto `np.arange(0, T, dt)` when `dt` is given), with the oracle's
accel on the right-hand side.  Besides (t, q, qd) it reports what the solver did -- function evaluations, accepted and
rejected steps, the accepted step sizes -- so a test can show that a case really exercises rejection, the max_step
clamp or a given first step.

RK45 spends one evaluation at t0 and one in its initial step selection, then six per attempted step (five stages and
the derivative at the new point), so attempts = (nfev - 2) / 6, or (nfev - 1) / 6 when `first_step` is given.
"""
from collections import namedtuple

import numpy as np
from scipy import integrate, interpolate

from oracle import oracle as orc

Run = namedtuple("Run", "t q qd nfev accepted rejected steps")


def rk45(rhs, y0, T, solver_args=None, dt=None):
    """Integrate y' = rhs(t, y) over [0, T].  Returns (t, y, nfev, accepted, rejected, steps); y is (len(t), len(y0))."""
    sa = dict(solver_args or {})
    y0 = np.asarray(y0, dtype=np.float64)
    integ = integrate.RK45(rhs, t0=0.0, y0=y0, t_bound=T, **sa)
    tl, yl, steps = [0], [y0], []
    while integ.status == "running":
        integ.step()
        if integ.status == "failed":
            raise RuntimeError("integration completed with failed status ")
        steps.append(integ.t - integ.t_old)
        tl.append(integ.t)
        yl.append(integ.y)
    ta, ya = np.array(tl), np.array(yl)
    attempts, rest = divmod(integ.nfev - (1 if sa.get("first_step") is not None else 2), 6)
    assert rest == 0, integ.nfev
    if dt is not None:
        tnew = np.arange(0, T, dt)
        ta, ya = tnew, interpolate.interp1d(ta, ya, axis=0)(tnew)
    return ta, ya, integ.nfev, len(steps), attempts - len(steps), np.array(steps)


def fdyn(accel, n, T, q0, qd0=None, torque=None, solver_args=None, dt=None):
    """accel(q, qd, tau) -> qdd; torque(t, q, qd) -> tau or None for zero torque.  The state is x = [q, qd]."""
    q0 = np.asarray(q0, dtype=np.float64).reshape(n)
    qd0 = np.zeros(n) if qd0 is None else np.asarray(qd0, dtype=np.float64).reshape(n)

    def f(t, x):
        q, qd = x[:n], x[n:]
        tau = np.zeros(n) if torque is None else np.asarray(torque(t, q, qd), dtype=np.float64)
        return np.r_[qd, accel(q, qd, tau)]

    t, x, nfev, acc, rej, steps = rk45(f, np.r_[q0, qd0], T, solver_args, dt)
    return Run(t, x[:, :n], x[:, n:], nfev, acc, rej, steps)


def dh_gravity(robot, gravity=None):
    """The robot's gravity seen from its base frame: the DH recursion has no base transform, so the gravity vector is
    rotated into the base frame instead (reference DHRobot.rne)."""
    g = np.asarray(robot.gravity if gravity is None else gravity, dtype=np.float64).reshape(3)
    return np.asarray(robot.base.A, dtype=np.float64)[:3, :3].T @ g


def dh_rne(robot):
    """rne_fn(q, qd, qdd, gravity) of a DH / MDH robot on the oracle's recursion (which takes MINUS the gravity)."""
    n, mdh, L = robot.n, int(robot.mdh), robot._pack_rne()
    return lambda q, qd, qdd, g: orc.rne(n, mdh, L, -np.asarray(g, dtype=np.float64), q, qd, qdd)  # noqa: E731


def dh_accel(robot, gravity=None):
    rne, n, g = dh_rne(robot), robot.n, dh_gravity(robot, gravity)
    return lambda q, qd, tau: orc.dyn_accel(rne, n, q, qd, tau, g)[0]  # noqa: E731


def tree_rne(robot):
    tree = robot.tree_description()
    return lambda q, qd, qdd, g: orc.tree_rne(tree, q, qd, qdd, g)  # noqa: E731


def tree_accel(robot, gravity=None):
    rne, n = tree_rne(robot), robot.n
    g = np.asarray(robot.gravity if gravity is None else gravity, dtype=np.float64).reshape(3)
    return lambda q, qd, tau: orc.dyn_accel(rne, n, q, qd, tau, g)[0]  # noqa: E731


def max_cond(rne, n, q):
    """The largest condition number of the joint-space inertia matrix over the states q (k, n)."""
    return float(np.linalg.cond(orc.dyn_inertia(rne, n, np.atleast_2d(q))).max())


def keeps_velocity_signs(qd):
    """True when no joint velocity is zero or changes sign along the trajectory qd (k, n): the Coulomb friction term
    jumps at qd = 0, and an adaptive integrator crossing it chatters with tiny steps (so does the reference)."""
    s = np.sign(qd[0])
    return bool((s != 0).all() and (np.sign(qd) == s).all())
