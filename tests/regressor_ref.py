"""Float64 reference for DHRobot.rne_regressor / regressor_gram / identify, built from the oracle's rne alone.

Without a tip wrench rne is linear in the 14 parameters of each link (DESIGN f-16), so column 14i + k of Y is rne on a
link table whose only nonzero dynamics are those of link i, chosen so that its parameter vector is the unit vector e_k:
  m          m = 1, r = 0, I = 0
  m r_a      m = 1, r = e_a, I = -(E - e_a e_a^T) (so I_o = 0), minus the m column
  I_o entry  m = 0, I = the symmetric unit matrix of that entry
  Jm, B, Tc+, Tc-   that friction parameter 1, the link's G kept
Every other link has m = 0, r = 0, I = 0 and no friction; the kinematics and G of every link are kept."""
import numpy as np

import rne_derivs_ref as R
from oracle import oracle as orc

# (row, col) pairs of the six inertia entries, in the order Ixx, Iyy, Izz, Ixy, Iyz, Ixz
I_ENTRIES = ((0, 0), (1, 1), (2, 2), (0, 1), (1, 2), (0, 2))


def unit_tables(L):
    """The 14 n link tables of the columns of Y, in column order, and the column to subtract (or None) for each."""
    T = np.asarray(L, dtype=np.float64).reshape(-1, 24)
    n = len(T)
    base = T.copy()
    base[:, 6:20] = 0.0  # m, r, I, Jm
    base[:, 21:24] = 0.0  # B, Tc+, Tc-
    tables, minus = [], []
    for i in range(n):
        col0 = 14 * i
        t = base.copy(); t[i, 6] = 1.0
        tables.append(t); minus.append(None)
        for a in range(3):
            t = base.copy(); t[i, 6] = 1.0; t[i, 7 + a] = 1.0
            e = np.zeros(3); e[a] = 1.0
            t[i, 10:19] = (-(np.eye(3) - np.outer(e, e))).ravel()
            tables.append(t); minus.append(col0)
        for (r, c) in I_ENTRIES:
            t = base.copy()
            U = np.zeros((3, 3)); U[r, c] = U[c, r] = 1.0
            t[i, 10:19] = U.ravel()
            tables.append(t); minus.append(None)
        for f in (19, 21, 22, 23):
            t = base.copy(); t[i, f] = 1.0
            tables.append(t); minus.append(None)
    return [t.ravel() for t in tables], minus


def regressor(L, mdh, grav, q, qd, qdd):
    """Y (N, n, 14n) from 14n calls of the oracle's rne."""
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    tables, minus = unit_tables(L)
    cols = [orc.rne(q.shape[1], mdh, t, grav, q, qd, qdd) for t in tables]
    cols = [c - cols[m] if m is not None else c for c, m in zip(cols, minus)]
    return np.stack(cols, axis=-1)


def parameters(L):
    """pi (14n,) of a packed link table, the convention of DHRobot.dynamic_parameters (symmetric part of I)."""
    T = np.asarray(L, dtype=np.float64).reshape(-1, 24)
    out = []
    for l in T:
        m, r, I = l[6], l[7:10], l[10:19].reshape(3, 3)
        Io = 0.5 * (I + I.T) + m * (r @ r * np.eye(3) - np.outer(r, r))
        out += [m, *(m * r), *(Io[a, b] for a, b in I_ENTRIES), l[19], l[21], l[22], l[23]]
    return np.array(out)


def structural_mask(n):
    """True where Y is zero by construction: link i < joint j, and the friction columns of link i in rows j != i."""
    M = np.zeros((n, 14 * n), dtype=bool)
    for j in range(n):
        for i in range(n):
            if i < j:
                M[j, 14 * i:14 * i + 14] = True
            elif i != j:
                M[j, 14 * i + 10:14 * i + 14] = True
    return M


def states(L, N, seed, zeros=True):
    """(q, qd, qdd) float64 (N, n) from rne_derivs_ref.states, with about a fifth of qd exactly 0 when `zeros`."""
    q, qd, qdd, _ = R.states(L, N, seed)
    if zeros:
        qd[np.random.default_rng(seed + 1).random(qd.shape) < 0.2] = 0.0
    return q, qd, qdd
