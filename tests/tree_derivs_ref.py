"""Reference for the derivatives of tree-robot dynamics (Robot.rne_derivatives / accel_derivatives).

`rne` restates oracle.tree_rne -- the numpy transcription of the reference's Robot.rne -- with every array in the dtype
of its inputs, so that it also runs on complex numbers.  tau is analytic in q and qd, so the complex step
Im tau(x + i h e_k) / h with h = 1e-30 is its derivative exact to rounding, with no step size to trade against
cancellation.  The forward mode is the one oracle.dyn_accel defines, differentiated by hand: qdd* = M^-1 (torque - bias),
d qdd* / dx = -M^-1 d rne(q, qd, qdd*) / dx with qdd* held fixed, d qdd* / d torque = M^-1.
"""
import numpy as np

from oracle import oracle as orc

H = 1e-30


def _skew(v):
    z = v[0] * 0
    return np.array([[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]])


def _joint_T(axis, eta):
    c, s = np.cos(eta), np.sin(eta)
    T = np.eye(4, dtype=np.result_type(eta, np.float64))
    if axis == 0:
        T[1:3, 1:3] = [[c, -s], [s, c]]
    elif axis == 1:
        T[0, 0], T[0, 2], T[2, 0], T[2, 2] = c, s, -s, c
    elif axis == 2:
        T[0:2, 0:2] = [[c, -s], [s, c]]
    else:
        T[axis - 3, 3] = eta
    return T


def _inv_Ad(T):
    """Ad(T^-1) without a matrix inverse (T is a rigid transform; np.linalg.inv is not complex-step safe in general)."""
    R, p = T[:3, :3], T[:3, 3]
    Ri = R.T
    A = np.zeros((6, 6), dtype=T.dtype)
    A[:3, :3] = Ri
    A[:3, 3:] = _skew(-Ri @ p) @ Ri
    A[3:, 3:] = Ri
    return A


def _crm(v):
    X = np.zeros((6, 6), dtype=v.dtype)
    X[:3, :3] = _skew(v[3:]); X[:3, 3:] = _skew(v[:3]); X[3:, 3:] = _skew(v[3:])
    return X


def rne(tree, q, qd, qdd, gravity):
    """One state: tau (n,) in group order, as oracle.tree_rne computes it, in the dtype of q / qd / qdd."""
    n = len(tree["parent"])
    dt = np.result_type(q, qd, qdd, np.float64)
    a_grav = np.zeros(6, dtype=dt)
    a_grav[:3] = -np.asarray(gravity, dtype=np.float64)
    Q = np.zeros(n, dtype=dt)
    Xup, v, a, f = [None] * n, [None] * n, [None] * n, [None] * n
    for j in range(n):
        ji = tree["jindex"][j]
        s = np.array(orc._AXIS_S[tree["axis"][j]], dtype=np.float64)
        eta = -q[ji] if tree["flip"][j] else q[ji]
        T = np.asarray(tree["C"][j], dtype=np.float64) @ _joint_T(tree["axis"][j], eta)
        Xup[j] = _inv_Ad(T)
        vJ = s * qd[ji]
        pa = tree["parent"][j]
        if pa < 0:
            v[j] = vJ.astype(dt)
            a[j] = Xup[j] @ a_grav + s * qdd[ji]
        else:
            v[j] = Xup[j] @ v[pa] + vJ
            a[j] = Xup[j] @ a[pa] + s * qdd[ji] + _crm(v[j]) @ vJ
        I = np.asarray(tree["I6"][j], dtype=np.float64)
        f[j] = I @ a[j] + (-_crm(v[j]).T) @ (I @ v[j])
    for j in reversed(range(n)):
        Q[j] = np.sum(f[j] * np.array(orc._AXIS_S[tree["axis"][j]]))
        pa = tree["parent"][j]
        if pa >= 0:
            f[pa] = f[pa] + Xup[j].T @ f[j]
    return Q


def rne_derivatives(tree, q, qd, qdd, gravity):
    """(dtau_dq, dtau_dqd), each (n, n) with [i, k] = d tau_i / d x_k, by complex step."""
    q, qd, qdd = (np.asarray(x, dtype=np.float64) for x in (q, qd, qdd))
    n = q.shape[0]
    dq, dqd = np.zeros((n, n)), np.zeros((n, n))
    for k in range(n):
        e = np.zeros(n, dtype=complex)
        e[k] = 1j * H
        dq[:, k] = rne(tree, q + e, qd, qdd, gravity).imag / H
        dqd[:, k] = rne(tree, q, qd + e, qdd, gravity).imag / H
    return dq, dqd


def inertia(tree, q):
    """M as oracle.dyn_inertia builds it: row i = rne(q, 0, e_i, gravity 0)."""
    n = len(q)
    z = np.zeros(n)
    return np.stack([rne(tree, q, z, np.eye(n)[i], np.zeros(3)) for i in range(n)])


def accel(tree, q, qd, torque, gravity):
    """oracle.dyn_accel for one state."""
    n = len(q)
    return np.linalg.solve(inertia(tree, q), torque - rne(tree, q, qd, np.zeros(n), gravity))


def accel_derivatives(tree, q, qd, torque, gravity):
    """(dqdd_dq, dqdd_dqd, dqdd_dtau) at qdd* = accel(q, qd, torque), each (n, n)."""
    qdd = accel(tree, q, qd, torque, gravity)
    Mi = np.linalg.inv(inertia(tree, q))
    dq, dqd = rne_derivatives(tree, q, qd, qdd, gravity)
    return -Mi @ dq, -Mi @ dqd, Mi


def richardson(f, x, k, h=1e-3):
    """d f / d x_k by Richardson-extrapolated central differences (error O(h^4))."""
    def central(hh):
        e = np.zeros_like(x)
        e[k] = hh
        return (f(x + e) - f(x - e)) / (2 * hh)
    return (4 * central(h / 2) - central(h)) / 3
