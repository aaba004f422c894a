"""Reference for the dynamics regressor of tree robots (Robot.rne_regressor, regressor_gram, identify).

Robot.rne is linear in the groups' spatial inertias, so column 10k + c of Y is tree_derivs_ref.rne (the restatement of
oracle.tree_rne) with group k's I6 set to the basis matrix of parameter c and every other group's to zero.  Parameters
per group, in the group order of tau: [m, hx, hy, hz, Ixx, Iyy, Izz, Ixy, Iyz, Ixz] of I6 = [[m E, -[h]x], [[h]x, Ib]].
"""
import numpy as np

import tree_derivs_ref as TR

_IB = [(0, 0), (1, 1), (2, 2), (0, 1), (1, 2), (0, 2)]


def basis(c):
    """The 6x6 spatial inertia of a unit value of parameter c, every other parameter 0."""
    I6 = np.zeros((6, 6))
    if c == 0:
        I6[:3, :3] = np.eye(3)
    elif c <= 3:
        S = TR._skew(np.eye(3)[c - 1])
        I6[:3, 3:], I6[3:, :3] = -S, S
    else:
        a, b = _IB[c - 4]
        I6[3 + a, 3 + b] = I6[3 + b, 3 + a] = 1.0
    return I6


def group_parameters(I6):
    I6 = np.asarray(I6, dtype=np.float64)
    return np.array([I6[0, 0], I6[5, 1], I6[3, 2], I6[4, 0]] + [I6[3 + a, 3 + b] for a, b in _IB])


def dynamic_parameters(tree):
    return np.concatenate([group_parameters(I6) for I6 in tree["I6"]])


def rigid_body_inertia(rng, m=None):
    """A full rigid-body spatial inertia: mass m, centre of mass c, a random positive-definite rotational inertia Ic
    about c (not a point mass), moved to the frame origin."""
    m = rng.uniform(0.3, 3) if m is None else m
    c = rng.uniform(-0.3, 0.3, 3)
    A = rng.normal(size=(3, 3)) * 0.2
    Ic = A @ A.T + 0.01 * np.eye(3)
    S = TR._skew(m * c)
    I6 = np.zeros((6, 6))
    I6[:3, :3] = m * np.eye(3)
    I6[:3, 3:], I6[3:, :3] = -S, S
    I6[3:, 3:] = Ic + m * (c @ c * np.eye(3) - np.outer(c, c))
    return I6


def below(tree, i):
    """below[k]: group k is group i or hangs below it."""
    n = len(tree["parent"])
    out = [False] * n
    for k in range(n):
        out[k] = k == i or (tree["parent"][k] >= 0 and out[tree["parent"][k]])
    return np.array(out)


def regressor(tree, q, qd, qdd, gravity):
    """Y (n, 10n) of one state, 10n calls of the restated rne."""
    n = len(tree["parent"])
    Y = np.zeros((n, 10 * n))
    zero = [np.zeros((6, 6))] * n
    for k in range(n):
        for c in range(10):
            I6 = list(zero)
            I6[k] = basis(c)
            Y[:, 10 * k + c] = TR.rne(dict(tree, I6=I6), q, qd, qdd, gravity)
    return Y
