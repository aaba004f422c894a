"""Float64 restatement of the static-force methods (DHRobot.gravjac, pay, paycap, friction).  Test infrastructure only.

The reference's Dynamics.py is not available, so the quantities are restated from their definitions, per row, on link
frames built with oracle.chains.dh_A (T_0 = base, T_k = T_{k-1} A_k(q_k)):
- joint j (0-based) turns about / slides along z of T_j (standard DH) or T_{j+1} (modified DH), through its origin, with
  sign -1 for a flipped joint; a point p moves with column  s z x (p - o) | s z  (revolute) or  s z | 0  (prismatic);
- gravjac: tau = -sum_i J_ci^T m_i g with pc_i = T_{i+1} r_i, and J0 = the columns at the tool point T_n tool;
- pay: -J^T W with J = J0 (frame 0) or blkdiag(R^T, R^T) J0 (frame 1, R the end-effector rotation);
- paycap: the issue's piecewise formula on tau_B = gravjac tau and tau_P = pay(w / |w|);
- friction: -(G^2 B qd + |G| Tc(qd)), the actuator terms of ne.c.
The tests pin these to the oracle (dyn_gravload, Chain.jacob0, rne with fext, rne minus its friction-free twin).
Link tables are the 24-double layout of oracle.chains.pack_rne.
"""
import numpy as np

from oracle import chains as ch


def links_of(n, L, flips=None):
    """24-double link table -> the link dicts of oracle.chains (flip per joint from `flips`)."""
    Lk = np.asarray(L, dtype=np.float64).reshape(n, 24)
    out = []
    for j, l in enumerate(Lk):
        out.append(dict(alpha=l[0], a=l[1], theta=l[2], d=l[3], sigma=int(l[4]), offset=l[5], m=l[6], r=l[7:10].copy(),
                        I=l[10:19].reshape(3, 3).copy(), Jm=l[19], G=l[20], B=l[21], Tc=l[22:24].copy(),
                        flip=bool(flips[j]) if flips is not None else False))
    return out


def _row(links, mdh, q, base, tool, g):
    n = len(links)
    T = [np.eye(4) if base is None else np.asarray(base, dtype=np.float64)]
    for j, l in enumerate(links):
        T.append(T[-1] @ ch.dh_A(l, float(q[j]), mdh))
    Te = T[n] if tool is None else T[n] @ tool
    pe = Te[:3, 3]
    pc = [(T[i + 1] @ np.append(links[i]["r"], 1.0))[:3] for i in range(n)]

    def column(j, p):
        F = T[j + 1] if mdh else T[j]
        z, o = F[:3, 2], F[:3, 3]
        s = -1.0 if links[j].get("flip", False) else 1.0
        if links[j].get("sigma", 0):
            return np.concatenate([s * z, np.zeros(3)])
        return np.concatenate([s * np.cross(z, p - o), s * z])

    J0 = np.stack([column(j, pe) for j in range(n)], axis=1)
    tau = np.zeros(n)
    for j in range(n):
        for i in range(j, n):
            tau[j] -= column(j, pc[i])[:3] @ (links[i]["m"] * g)
    return tau, J0, Te[:3, :3]


def gravjac(links, mdh, q, gravity, base=None, tool=None):
    """-> tau (N,n), J0 (N,6,n)"""
    q = np.atleast_2d(q)
    g = np.asarray(gravity, dtype=np.float64)
    res = [_row(links, mdh, qk, base, tool, g)[:2] for qk in q]
    return np.stack([r[0] for r in res]), np.stack([r[1] for r in res])


def jacobe(links, mdh, q, base=None, tool=None):
    """(N,6,n): blkdiag(R^T, R^T) J0"""
    q = np.atleast_2d(q)
    out = []
    for qk in q:
        _, J0, R = _row(links, mdh, qk, base, tool, np.zeros(3))
        out.append(np.vstack([R.T @ J0[:3], R.T @ J0[3:]]))
    return np.stack(out)


def pay(links, mdh, W, q, frame, base=None, tool=None):
    """-J^T W, (N,n); W (6,) or (N,6)"""
    q = np.atleast_2d(q)
    J = jacobe(links, mdh, q, base, tool) if frame == 1 else gravjac(links, mdh, q, np.zeros(3), base, tool)[1]
    W = np.broadcast_to(np.asarray(W, dtype=np.float64), (q.shape[0], 6))
    return -np.einsum("nkj,nk->nj", J, W)


def paycap(links, mdh, w, tauR, frame, q, gravity, base=None, tool=None):
    """-> wmax (N,n), joint (N,)"""
    q = np.atleast_2d(q)
    w = np.broadcast_to(np.asarray(w, dtype=np.float64), (q.shape[0], 6))
    nrm = np.linalg.norm(w, axis=1)
    zero = nrm == 0
    wh = w / np.where(zero, 1.0, nrm)[:, None]
    tauB = gravjac(links, mdh, q, gravity, base, tool)[0]
    tauP = pay(links, mdh, wh, q, frame, base, tool)
    tauR = np.asarray(tauR, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        wmax = np.where(tauP > 0, (tauR[:, 0] - tauB) / tauP, np.where(tauP < 0, (tauR[:, 1] - tauB) / tauP, np.inf))
    joint = np.argmin(wmax, axis=1).astype(np.int32)
    wmax[zero] = np.nan
    joint[zero] = -1
    return wmax, joint


def friction(links, qd):
    qd = np.atleast_2d(qd)
    G = np.array([l["G"] for l in links])
    Bv = np.array([l["B"] for l in links])
    Tc = np.array([l["Tc"] for l in links])
    tc = np.where(qd > 0, Tc[:, 0], np.where(qd < 0, Tc[:, 1], 0.0))
    return -(G * G * Bv * qd + np.abs(G) * tc)


# the worked paycap case: a planar 2R standard-DH arm, q = 0, a downward unit force in the world frame
PLANAR_2R = [dict(a=1.0, alpha=0.0, m=2.0, r=np.array([-0.5, 0.0, 0.0])), dict(a=0.5, alpha=0.0, m=1.0, r=np.array([-0.25, 0.0, 0.0]))]
PLANAR_2R_CASE = dict(w=[0, -1, 0, 0, 0, 0], tauR=[[30, -30], [5, -5]], frame=0, q=[0.0, 0.0], gravity=[0, -9.81, 0],
                      tauB=[22.0725, 2.4525], tauP=[1.5, 0.5], wmax=[5.285, 5.095], joint=1)
