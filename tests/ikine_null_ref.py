"""Per-row numpy restatement of the reference's Python IK solver loop with its null-space terms.

IKSolver._solve (the Python semantics: step, then test the pre-step error, wrap with floor-modulo), the steps of
IK_LM (chan / wampler / sugihara), IK_NR and IK_GN, and IKSolver._calc_qnull / _null_Σ as DESIGN (f-7) restates them:

    q <- q + (dq_solver + qnull),   qnull = (I - pinv(J) J) g,   g = [kq > 0] sigma(q) / kq + [km > 0] jacobm(q) / km

Pose and Jacobian come from the oracle's chain (orc.Chain.fkine / jacob0), the manipulability Jacobian from
oracle.hessian + oracle.jacobm, the projector from np.linalg.pinv, and the restart draws from oracle.rand_u01 keyed by
(seed, row, search, joint) like the kernel's.
"""
import math

import numpy as np

from oracle import oracle as orc

METHODS = {"chan": 0, "wampler": 1, "sugihara": 2, "nr": 3, "gn": 4}


def sigma(q, ql, qh, ps, pi):
    """_null_Σ with the reference's final sign: pushes a joint away from a limit it is within pi of."""
    s = np.zeros(len(q))
    for i in range(len(q)):
        if q[i] - ql[i] <= pi[i]:
            s[i] = ((q[i] - ql[i]) - pi[i]) ** 2 / (ps - pi[i]) ** 2
        if qh[i] - q[i] <= pi[i]:
            s[i] = -(((qh[i] - q[i]) - pi[i]) ** 2) / (ps - pi[i]) ** 2
    return s


def jacobm_term(J):
    """ETS.jacobm with all six axes, from the base-frame Jacobian J (6, n): (n,)"""
    return orc.jacobm(J, orc.hessian(J))[:, 0]


def qnull(J, q, ql, qh, kq, km, ps, pi):
    """_calc_qnull: (I - pinv(J) J) g"""
    n = J.shape[1]
    g = np.zeros(n)
    if kq > 0:
        g += sigma(q, ql, qh, ps, pi) / kq
    if km > 0:
        g += jacobm_term(J) / km
    if not (kq > 0 or km > 0):
        return g
    return (np.eye(n) - np.linalg.pinv(J) @ J) @ g


def _step(J, e, E, we, k, method):
    n = J.shape[1]
    if method <= 2:
        wn = k * E if method == 0 else (k if method == 1 else E + k)
        return np.linalg.solve(J.T @ (we[:, None] * J) + wn * np.eye(n), J.T @ (we * e))
    if method == 3:
        if k > 0:  # damped pseudo-inverse of the compiled NR step (pinv_damping)
            return J.T @ np.linalg.solve(J @ J.T + k * k * np.eye(6), e)
        return np.linalg.pinv(J) @ e
    w = np.sqrt(we)
    return np.linalg.pinv(w[:, None] * J) @ (w * e)


def step(J, e, E, we, k, method):
    """The solver's own update dq; None where numpy raises LinAlgError or the step is not finite (a search that has
    run off to inf / nan: the oracle's loop and the kernel abandon it there)."""
    try:
        dq = _step(J, e, E, we, k, method)
    except np.linalg.LinAlgError:
        return None
    return dq if np.isfinite(dq).all() else None


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


def solve_row(C, T, q0, ilimit, slimit, tol, joint_limits, we, k, method, seed, row, kq=0.0, km=0.0, ps=0.0, pi=0.3):
    """IKSolver._solve for one target: (q, success, iterations, searches, residual)."""
    n = C.n
    ql, qh = C.qlim_l, C.qlim_h
    pi = np.full(n, float(pi)) if np.ndim(pi) == 0 else np.asarray(pi, dtype=np.float64)
    we = np.ones(6) if we is None else np.asarray(we, dtype=np.float64)
    meth = METHODS[method] if isinstance(method, str) else int(method)
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
            dq = step(J, e, E, we, k, meth)
            if dq is None:
                break
            try:
                qn = qnull(J, q, ql, qh, kq, km, ps, pi)
            except np.linalg.LinAlgError:  # numpy's SVD gives up on a non-finite J: the search is abandoned
                break
            q = q + (dq + qn)
            if E < tol:
                q = wrap(q)
                valid = bool(((q >= ql) & (q <= qh)).all())
                if not valid and joint_limits:
                    break
                return q, 1, total + i, search + 1, E
        total += i
    return q, 0, total, slimit, E


def solve(C, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, joint_limits=True, we=None, k=1.0, method="chan", seed=0,
          rng_per_row=True, rows=None, **null):
    """solve_row over the rows of Tep (or the subset `rows`): arrays (q, success, iterations, searches, residual)."""
    Tep = np.asarray(Tep, dtype=np.float64).reshape(-1, 4, 4)
    rows = np.arange(Tep.shape[0]) if rows is None else np.asarray(rows)
    q0 = None if q0 is None else np.broadcast_to(np.asarray(q0, dtype=np.float64).reshape(-1, C.n), (Tep.shape[0], C.n))
    out = [solve_row(C, Tep[r], None if q0 is None else q0[r], ilimit, slimit, tol, joint_limits, we, k, method, seed,
                     int(r) if rng_per_row else 0, **null) for r in rows]
    return (np.array([o[0] for o in out]), np.array([o[1] for o in out], dtype=np.int32),
            np.array([o[2] for o in out], dtype=np.int32), np.array([o[3] for o in out], dtype=np.int32),
            np.array([o[4] for o in out]))
