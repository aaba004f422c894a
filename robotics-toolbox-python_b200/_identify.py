"""Least-squares identification of inertial parameters from the normal equations of a dynamics regressor, shared by
``DHRobot.identify`` and ``Robot.identify``."""
from __future__ import annotations

from collections import namedtuple

import numpy as np

IdentifyResult = namedtuple("IdentifyResult", "pi rank rms")


def solve(G, b, s, keep, eps, rcond, N, n) -> IdentifyResult:
    """The minimum-norm pi of the normal equations G pi = b (G = sum Y^T W Y, b = sum Y^T W tau, s = sum tau^T W tau over N
    rows of n torques): columns outside ``keep`` and zero columns (below 16 ``eps`` of the largest column norm) get 0; the
    rest of G is scaled to unit diagonal, and its eigenvalues below ``rcond`` times the largest are dropped (rank = the
    number kept).  rms = sqrt((s - 2 pi.b + pi.G.pi) / (N n))."""
    # A column at the rounding level of the compute type is a zero column: a structurally zero term that the link
    # constants (cos(pi/2) = 6e-17) or cancelling products leave a few ulps off 0 would otherwise become a unit
    # column after the scaling below.  The cut, 16 eps of the largest column norm (2e-6 in float32), sits well
    # below real columns: on Puma560 inertial columns are 4e-5 of the armature columns (G^2 qdd).
    keep = keep & (np.diag(G) > (16 * eps) ** 2 * np.max(np.diag(G), initial=0.0))
    pi = np.zeros(G.shape[0])
    rank = 0
    if keep.any():
        Gk, bk = G[np.ix_(keep, keep)], b[keep]
        d = 1.0 / np.sqrt(np.diag(Gk))
        lam, V = np.linalg.eigh(d[:, None] * Gk * d[None, :])
        use = lam > rcond * lam[-1]
        rank = int(use.sum())
        pi[keep] = d * (V[:, use] @ ((V[:, use].T @ (d * bk)) / lam[use]))
    res = s - 2 * pi @ b + pi @ G @ pi
    return IdentifyResult(pi, rank, float(np.sqrt(max(res, 0.0) / max(N * n, 1))))
