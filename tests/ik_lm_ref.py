"""High-precision reference of one step of the batched LM / NR / GN inverse-kinematics solvers (csrc/b2k_ik.cuh).

For a chain with dense jindex (an ``oracle.Chain``), a joint vector q, a target Tep and the weights We (unit, a 0/1 mask or
general), ``step`` returns ``(e, E, dq)``:

* e = the angle-axis error of the compiled reference (``orc.angle_axis``) at the fp64 pose, E = 1/2 e^T We e;
* J = ``Chain.jacob0(q)`` in fp64 (FK and J are pinned to the compiled reference elsewhere);
* dq solved in mpmath at 40 digits:
    LM (chan / wampler / sugihara)  (J^T We J + wn I)^-1 J^T We e,  wn = lambda E | lambda | E + lambda
    NR                              V diag(s / (s^2 + d^2)) U^T e on the unweighted J (NR weighs only E)
    GN                              the minimum-norm least-squares solution of diag(sqrt we) J dq = diag(sqrt we) e,
                                    singular values below eps * max(6, n) * s_max counted as zero (as the oracle does).

``cond`` gives the condition number of the system each step solves (the normal matrix of LM; (s_max^2 + d^2) /
(s_min^2 + d^2) over the min(n, weighted rows) singular values for NR / GN), which is what the kernels' accuracy
depends on.
``rand_q`` restates the counter-based restart draw of the kernels (``ik_rand_q``) on ``orc.rand_u01``.
"""
from __future__ import annotations

import mpmath as mp
import numpy as np

from oracle import oracle as orc

DPS = 40
EPS = 2.220446049250313e-16
METHODS = ("chan", "wampler", "sugihara", "nr", "gn")
UNIT = np.ones(6)


def error(C, q, Tep, we=UNIT):
    """(e, E) at q: the compiled reference's angle-axis error and E = 1/2 e^T We e (oracle order of summation)."""
    Te = C.fkine(np.asarray(q, dtype=np.float64)[None])[0]
    e = orc.angle_axis(Te, np.asarray(Tep, dtype=np.float64))
    E = 0.0
    for k in range(6):
        E += e[k] * we[k] * e[k]
    return e, 0.5 * E


def _weighted(J, e, method, we):
    ws = np.sqrt(np.maximum(we, 0.0)) if method == "gn" else np.ones(6)
    return ws[:, None] * J, ws * e


def dq_of(J, e, E, method, lam, we=UNIT):
    """The step for a given fp64 J (6, n), e (6) and E, in mpmath; returned as fp64."""
    n = J.shape[1]
    with mp.workdps(DPS):
        if method in ("chan", "wampler", "sugihara"):
            wn = {"chan": mp.mpf(lam) * mp.mpf(E), "wampler": mp.mpf(lam), "sugihara": mp.mpf(E) + mp.mpf(lam)}[method]
            Jm = mp.matrix(J.tolist())
            W = mp.diag([mp.mpf(float(w)) for w in we])
            A = Jm.T * W * Jm + wn * mp.eye(n)
            g = Jm.T * W * mp.matrix(e.tolist())
            try:
                x = mp.lu_solve(A, g)
            except ZeroDivisionError:  # singular normal matrix: the kernels abandon such a search
                return np.full(n, np.nan)
            return np.array([float(x[i]) for i in range(n)])
        Jw, ew = _weighted(J, e, method, we)
        # The SVD through the eigenvectors of the smaller Gram matrix (40 digits leave ~20 for its singular values):
        # n < 6: Jw^T Jw = V S^2 V^T and dq = sum_i v_i (v_i . Jw^T ew) / (s_i^2 + d^2);
        # n >= 6: Jw Jw^T = U S^2 U^T and dq = Jw^T sum_i u_i (u_i . ew) / (s_i^2 + d^2).
        A = mp.matrix(Jw.tolist())
        rowform = n >= 6
        G = A * A.T if rowform else A.T * A
        lam2, Q = mp.eigsy(G)
        r = G.rows
        s = [mp.sqrt(max(lam2[i], 0)) for i in range(r)]
        b = mp.matrix(ew.tolist()) if rowform else A.T * mp.matrix(ew.tolist())
        d2 = mp.mpf(lam) ** 2 if method == "nr" else mp.mpf(0)
        thr = mp.mpf(EPS) * max(6, n) * max(s) if method == "gn" else mp.mpf(-1)
        x = mp.matrix(r, 1)
        for i in range(r):
            if not s[i] > thr or s[i] ** 2 + d2 == 0:
                continue
            t = sum(Q[a, i] * b[a] for a in range(r)) / (s[i] ** 2 + d2)
            for a in range(r):
                x[a] += Q[a, i] * t
        if rowform:
            x = A.T * x
        return np.array([float(x[i]) for i in range(n)])


def step(C, q, Tep, method, lam, we=UNIT):
    """(e, E, dq) of one solver step at q (see the module docstring)."""
    we = np.asarray(we, dtype=np.float64)
    e, E = error(C, q, Tep, we)
    J = C.jacob0(np.asarray(q, dtype=np.float64)[None])[0]
    return e, E, dq_of(J, e, E, method, lam, we)


def cond(J, E, method, lam, we=UNIT):
    """Condition number of the system the step solves, in fp64 (only used to pick the rows a tolerance applies to)."""
    we = np.asarray(we, dtype=np.float64)
    n = J.shape[1]
    if method in ("chan", "wampler", "sugihara"):
        wn = {"chan": lam * E, "wampler": lam, "sugihara": E + lam}[method]
        return float(np.linalg.cond(J.T @ (we[:, None] * J) + wn * np.eye(n)))
    Jw, _ = _weighted(J, np.zeros(6), method, we)
    # no truncation here: the kernels solve the full-rank system of min(n, weighted rows) singular values, so a row whose
    # weighted rows are dependent is ill-conditioned for them even where the minimum-norm step is well defined
    k = min(n, int((np.abs(Jw).sum(axis=1) > 0).sum()) if method == "gn" else 6)
    s = np.linalg.svd(Jw, compute_uv=False)[:max(k, 1)]
    d2 = lam * lam if method == "nr" else 0.0
    lo = s.min() ** 2 + d2
    return float((s.max() ** 2 + d2) / lo) if lo > 0 else np.inf


def rand_q(qlim_l, qlim_h, seed, row, search):
    """The restart draw of search `search` of problem row `row` (fp64; ik_rand_q / oracle rand_q)."""
    out = np.empty(len(qlim_l))
    for i in range(len(qlim_l)):
        r = 2.0 * orc.rand_u01(seed, row, search, i) - 1.0
        out[i] = (r + 1.0) * ((qlim_h[i] - qlim_l[i]) / 2.0) + qlim_l[i]
    return out
