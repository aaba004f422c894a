"""Float64 reference for DHRobot.rne_derivatives / accel_derivatives: Richardson-extrapolated central differences
(4th order in the step) of the oracle's rne and of accel built on it, plus the robots and states the tests share.

Compare only at states whose joint rates are all at least 0.1 in magnitude: the Coulomb friction step at qd = 0 must not
fall inside a stencil."""
import numpy as np

import dyn_ref as D
from oracle import oracle as orc

H = 1e-3  # the error of the extrapolated difference is O(H^4) from truncation plus O(eps / H) from rounding


def ddx(f, x, h=H):
    """Jacobian (N, m, n) of f: (N, n) -> (N, m) at x (N, n), [r, i, k] = d f_i / d x_k: column k is
    (4 D(h/2) - D(h)) / 3 with D(s) the central difference in x[:, k]."""
    x = np.asarray(x, dtype=np.float64)
    cols = []
    for k in range(x.shape[1]):
        e = np.zeros(x.shape[1])
        e[k] = 1.0
        d = lambda s: (f(x + s * e) - f(x - s * e)) / (2 * s)  # noqa: E731
        cols.append((4 * d(h / 2) - d(h)) / 3)
    return np.stack(cols, axis=-1)


def rne(L, mdh, grav, q, qd, qdd, fext=None):
    """tau (N, n) from the oracle; grav is the vector handed to the kernel (minus the robot's gravity)."""
    return orc.rne(len(L) // 24, mdh, L, grav, q, qd, qdd, fext)


def inertia(L, mdh, q):
    """M (N, n, n) in the layout of DHRobot.inertia: row i = rne(q, 0, e_i) without gravity (Dynamics.py:752-758)."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    N, n = q.shape
    z = np.zeros((N, n))
    M = np.empty((N, n, n))
    for i in range(n):
        e = np.zeros((N, n))
        e[:, i] = 1.0
        M[:, i, :] = rne(L, mdh, np.zeros(3), q, z, e)
    return M


def accel(L, mdh, grav, q, qd, torque):
    """qdd = M^-1 (torque - rne(q, qd, 0)) over rows, as oracle.dyn_accel (Dynamics.py:490-503)."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    h = rne(L, mdh, grav, q, qd, np.zeros_like(q))
    return np.linalg.solve(inertia(L, mdh, q), (np.atleast_2d(torque) - h)[..., None])[..., 0]


def rne_derivatives(L, mdh, grav, q, qd, qdd, fext=None):
    """(dtau_dq, dtau_dqd), each (N, n, n)."""
    return (ddx(lambda x: rne(L, mdh, grav, x, qd, qdd, fext), q),
            ddx(lambda x: rne(L, mdh, grav, q, x, qdd, fext), qd))


def mdh_prismatic_first(L, mdh):
    return bool(mdh) and np.asarray(L).reshape(-1, 24)[0, 4] != 0


def accel_derivatives(L, mdh, grav, q, qd, torque):
    """(dqdd_dq, dqdd_dqd, dqdd_dtau), each (N, n, n): differences of accel.

    An MDH arm with a prismatic first joint keeps ne.c's treatment of that joint, under which inertia(q) is not
    symmetric and accel is not the inverse of rne; there the operation is defined by its formula, -M^-1 dtau_dx at
    qdd* and M^-1, and that is what is returned (dtau_dx from differences of rne)."""
    if mdh_prismatic_first(L, mdh):
        Minv = np.linalg.inv(inertia(L, mdh, q))
        iq, iqd = rne_derivatives(L, mdh, grav, q, qd, accel(L, mdh, grav, q, qd, torque))
        return -Minv @ iq, -Minv @ iqd, Minv
    return (ddx(lambda x: accel(L, mdh, grav, x, qd, torque), q),
            ddx(lambda x: accel(L, mdh, grav, q, x, torque), qd),
            ddx(lambda x: accel(L, mdh, grav, q, qd, x), torque))


def friction(L, qd):
    """Joint friction torque -(G^2 B qd + |G| Tc(qd)) (N, n), Tc+ for qd > 0, Tc- for qd < 0 (Link.friction)."""
    T = np.asarray(L).reshape(-1, 24)
    G, B, tcp, tcm = T[:, 20], T[:, 21], T[:, 22], T[:, 23]
    tc = np.where(qd > 0, tcp, 0.0) + np.where(qd < 0, tcm, 0.0)
    return -(G * G * B * qd + np.abs(G) * tc)


def viscous(L):
    """G^2 B per joint: the friction part of the diagonal of dtau_dqd."""
    T = np.asarray(L).reshape(-1, 24)
    return T[:, 20] ** 2 * T[:, 21]


def robot(n, mdh, prismatic, friction_on, seed, profile="gen"):
    """A packed link table from dyn_ref.robot with the fields the joint variable replaces set to 0 (theta of a revolute
    joint, d of a prismatic one), so that it round-trips through DHRobot._pack_rne."""
    T = np.asarray(D.robot(n, mdh, profile, prismatic, friction_on, seed)).reshape(-1, 24).copy()
    T[T[:, 4] == 0, 2] = 0.0
    T[T[:, 4] != 0, 3] = 0.0
    return T.ravel()


def dhrobot(L, mdh):
    """The DHRobot of a packed link table."""
    import b2kin as rtb

    links = []
    for l in np.asarray(L).reshape(-1, 24):
        links.append(rtb.DHLink(alpha=l[0], a=l[1], theta=l[2], d=l[3], sigma=int(l[4]), offset=l[5], mdh=bool(mdh), m=l[6],
                                r=l[7:10], I=l[10:19].reshape(3, 3), Jm=l[19], G=l[20], B=l[21], Tc=l[22:24]))
    r = rtb.DHRobot(links)
    assert np.array_equal(r._pack_rne(), np.asarray(L)), "link table does not round-trip"
    return r


def revolute_first(L):
    """The same table with joint 1 made revolute (d = 0.2): an MDH arm whose prismatic joints are not the first."""
    T = np.asarray(L).reshape(-1, 24).copy()
    T[0, 2:5] = 0.0, 0.2, 0
    return T.ravel()


def states(L, N, seed):
    """(q, qd, qdd, torque) float64 (N, n): q in [-pi, pi] (prismatic q in [-0.5, 0.5]), 0.1 <= |qd| <= 2."""
    rng = np.random.default_rng(seed)
    pris = np.asarray(L).reshape(-1, 24)[:, 4] != 0
    n = len(pris)
    q = np.where(pris, rng.uniform(-0.5, 0.5, (N, n)), rng.uniform(-np.pi, np.pi, (N, n)))
    qd = rng.choice([-1.0, 1.0], (N, n)) * rng.uniform(0.1, 2.0, (N, n))
    return q, qd, rng.normal(size=(N, n)), 10 * rng.normal(size=(N, n))
