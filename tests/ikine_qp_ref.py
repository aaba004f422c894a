"""Per-row numpy restatement of the reference's Python IK solver loop with the quadratic-programming step (IK_QP).

IKSolver._solve (the Python semantics: step, then test the pre-step error, wrap with floor-modulo, reject results
outside the joint limits) with the step DESIGN (f-11) restates, at the pre-step q:

    e = angle-axis error of fkine(q) against Tep (unweighted),  E = 1/2 e^T We e,  J = jacob0(q)
    minimise 1/2 kj |dq|^2 + 1/2 w |s|^2 + c^T dq   subject to  J dq + s = e,   w = ks / sum|e|
    c = -jacobm(q) / km  (km > 0),  and with kq > 0 at most one velocity-damper row per joint:
        -dq_i <= ((q_i - l_i) - ps) / ((pi_i - ps) kq)   if q_i - l_i <= pi_i
         dq_i <= ((h_i - q_i) - ps) / ((pi_i - ps) kq)   if h_i - q_i <= pi_i   (wins when both hold)
    q <- q + dq

Eliminating s leaves  min 1/2 dq^T H dq - r^T dq,  H = kj I + w J^T J,  r = w J^T e - c,  under one-sided bounds on
single coordinates.  `qp_bounded` solves that exactly with a primal active-set method (a different algorithm from the
kernel's), so the two are independent.  Pose and Jacobian come from the oracle's chain, jacobm from oracle.hessian +
oracle.jacobm, restarts from oracle.rand_u01 keyed by (seed, row, search, joint) like the kernel's.
"""
import math

import numpy as np

from oracle import oracle as orc


def damper(q, ql, qh, kq, ps, pi):
    """(sign, bound) per joint: sign * dq_i <= bound; sign 0 = no row.  The upper-limit row wins when both hold."""
    n = len(q)
    sgn, bnd = np.zeros(n), np.zeros(n)
    if not kq > 0:
        return sgn, bnd
    for i in range(n):
        dl, dh = q[i] - ql[i], qh[i] - q[i]
        if dh <= pi[i]:
            sgn[i], bnd[i] = 1.0, (dh - ps) / (pi[i] - ps) / kq
        elif dl <= pi[i]:
            sgn[i], bnd[i] = -1.0, (dl - ps) / (pi[i] - ps) / kq
    return sgn, bnd


def qp_bounded(H, r, sgn, bnd, tol=1e-13):
    """argmin 1/2 x^T H x - r^T x  subject to  sgn_i x_i <= bnd_i (rows with sgn_i = 0 are free); H SPD.
    Primal active set (Nocedal & Wright, Algorithm 16.3) from the projection of 0 onto the bounds."""
    n = len(r)
    con = sgn != 0
    W = con & (bnd < 0)  # 0 violates these rows: start on their bounds
    x = np.where(W, sgn * bnd, 0.0)
    for _ in range(20 * n + 20):
        f = ~W
        xn = x.copy()
        if f.any():
            xn[f] = np.linalg.solve(H[np.ix_(f, f)], r[f] - H[np.ix_(f, W)] @ x[W])
        p = xn - x
        if np.abs(p).max() <= tol * (1.0 + np.abs(x).max()):
            g = H @ x - r
            mu = -sgn * g  # multiplier of sgn_i x_i <= bnd_i
            neg = W & (mu < -tol * (1.0 + np.abs(r).max()))
            if not neg.any():
                return x
            W[np.flatnonzero(neg)[np.argmin(mu[neg])]] = False
            continue
        alpha, block = 1.0, -1
        for i in np.flatnonzero(con & f):
            sp = sgn[i] * p[i]
            if sp > 0:
                a = (bnd[i] - sgn[i] * x[i]) / sp
                if a < alpha:
                    alpha, block = max(a, 0.0), i
        x = x + alpha * p
        if block >= 0:
            x[block] = sgn[block] * bnd[block]
            W[block] = True
    raise RuntimeError("qp_bounded: no convergence")


def jacobm_term(J):
    """ETS.jacobm with all six axes, from the base-frame Jacobian J (6, n): (n,)"""
    return orc.jacobm(J, orc.hessian(J))[:, 0]


def qp_problem(J, e, q, ql, qh, kj, ks, kq, km, ps, pi):
    """(H, r, sgn, bnd, w) of one step"""
    n = J.shape[1]
    w = ks / np.sum(np.abs(e))
    c = -jacobm_term(J) / km if km > 0 else np.zeros(n)
    H = kj * np.eye(n) + w * J.T @ J
    r = w * J.T @ e - c
    sgn, bnd = damper(q, ql, qh, kq, ps, pi)
    return H, r, sgn, bnd, w


def step(J, e, q, ql, qh, kj, ks, kq, km, ps, pi):
    """dq of one QP step (0 where sum|e| = 0)"""
    if np.sum(np.abs(e)) == 0:
        return np.zeros(J.shape[1])
    H, r, sgn, bnd, _ = qp_problem(J, e, q, ql, qh, kj, ks, kq, km, ps, pi)
    return qp_bounded(H, r, sgn, bnd)


def rand_q(seed, row, search, ql, qh):
    q = np.empty(len(ql))
    for i in range(len(ql)):
        r = 2.0 * orc.rand_u01(seed, row, search, i) - 1.0
        q[i] = (r + 1.0) * ((qh[i] - ql[i]) / 2.0) + ql[i]
    return q


def wrap(q):
    w = np.fmod(q + math.pi, 2 * math.pi)
    w = np.where(w < 0, w + 2 * math.pi, w)
    return w - math.pi


def solve_row(C, T, q0, ilimit, slimit, tol, joint_limits, we, seed, row, kj=1.0, ks=1.0, kq=0.0, km=0.0, ps=0.0,
              pi=0.3):
    """IKSolver._solve with the QP step for one target: (q, success, iterations, searches, residual)."""
    n = C.n
    ql, qh = C.qlim_l, C.qlim_h
    pi = np.full(n, float(pi)) if np.ndim(pi) == 0 else np.asarray(pi, dtype=np.float64)
    we = np.ones(6) if we is None else np.asarray(we, dtype=np.float64)
    total = 0
    E = 0.0
    q = None
    for search in range(slimit):
        q = np.array(q0, dtype=np.float64) if (search == 0 and q0 is not None) else rand_q(seed, row, search, ql, qh)
        i = 0
        while i < ilimit:
            i += 1
            e = orc.angle_axis(C.fkine(q)[0], T)
            E = 0.5 * float(e @ (we * e))
            J = C.jacob0(q)[0]
            try:
                dq = step(J, e, q, ql, qh, kj, ks, kq, km, ps, pi)
            except (np.linalg.LinAlgError, RuntimeError):
                break
            if not np.isfinite(dq).all():
                break
            q = q + dq
            if E < tol:
                q = wrap(q)
                valid = bool(((q >= ql) & (q <= qh)).all())
                if not valid and joint_limits:
                    break
                return q, 1, total + i, search + 1, E
        total += i
    return q, 0, total, slimit, E


def solve(C, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, joint_limits=True, we=None, seed=0, rng_per_row=False,
          rows=None, **qp):
    """solve_row over the rows of Tep (or the subset `rows`): arrays (q, success, iterations, searches, residual).
    rng_per_row defaults to False, as ETS.ikine_QP passes it."""
    Tep = np.asarray(Tep, dtype=np.float64).reshape(-1, 4, 4)
    rows = np.arange(Tep.shape[0]) if rows is None else np.asarray(rows)
    q0 = None if q0 is None else np.broadcast_to(np.asarray(q0, dtype=np.float64).reshape(-1, C.n), (Tep.shape[0], C.n))
    out = [solve_row(C, Tep[r], None if q0 is None else q0[r], ilimit, slimit, tol, joint_limits, we, seed,
                     int(r) if rng_per_row else 0, **qp) for r in rows]
    return (np.array([o[0] for o in out]), np.array([o[1] for o in out], dtype=np.int32),
            np.array([o[2] for o in out], dtype=np.int32), np.array([o[3] for o in out], dtype=np.int32),
            np.array([o[4] for o in out]))
