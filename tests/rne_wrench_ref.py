"""Float64 references for DHRobot.rne(..., base_wrench=True).  Test infrastructure only.

- `rne_wrench`: a batched numpy restatement of the oracle's ne.c recursion (oracle_kin.c rne_one), operation for
  operation, that also returns the base wrench.  Its tau is pinned to the oracle's rne by the tests; its wbase is the
  recursion's own f_1, n_1 carried into frame 0: [R_1 f_1, R_1 n_1] for standard DH (n_1 is about O_0) and
  [R_1 f_1, R_1 n_1 + p*_1 x R_1 f_1] for modified DH (n_1 is about O_1).
- `momentum_balance`: an independent prediction of the same wrench from link poses alone (Newton-Euler for the whole
  robot): f_0 = dP/dt - M g_b + R_n f_tip, n_0 = dH_O0/dt - sum m_i p_ci x g_b + R_n n_tip + p_n x R_n f_tip, with P and
  H_O0 from finite differences along q(t) = q + qd t + qdd t^2 / 2.
- `virtual_joint_tree`: the same links behind six massless joints (tx, ty, tz, Rx, Ry, Rz) as a rigid-body tree for the
  oracle's spatial-vector recursion; at zero virtual coordinates their six torques are the base wrench.

L is the 24-double link table, grav the vector handed to the recursion (MINUS the gravity in frame 0), as for orc.rne.
"""
import numpy as np

from oracle import chains as ch
from oracle import oracle as orc


def _links(n, L):
    return np.asarray(L, dtype=np.float64).reshape(n, 24)


def _rot(mdh, st, ct, sa, ca):
    """Link rotation (frame j in frame j-1): Rz(theta) Rx(alpha) for DH, Rx(alpha) Rz(theta) for MDH; (N,3,3)."""
    R = np.zeros(st.shape + (3, 3))
    if not mdh:
        R[:, 0] = np.stack([ct, -ca * st, sa * st], -1)
        R[:, 1] = np.stack([st, ca * ct, -sa * ct], -1)
        R[:, 2] = np.stack([np.zeros_like(st), np.full_like(st, sa), np.full_like(st, ca)], -1)
    else:
        R[:, 0] = np.stack([ct, -st, np.zeros_like(st)], -1)
        R[:, 1] = np.stack([st * ca, ca * ct, np.full_like(st, -sa)], -1)
        R[:, 2] = np.stack([st * sa, ct * sa, np.full_like(st, ca)], -1)
    return R


def _mul(R, v):
    return np.einsum("nij,nj->ni", R, v)


def _tmul(R, v):
    return np.einsum("nji,nj->ni", R, v)


def _geometry(n, mdh, L, q):
    """Per link: R (N,3,3), p* (N,3), prismatic flag."""
    Lk = _links(n, L)
    q = np.atleast_2d(np.asarray(q, dtype=np.float64))
    N = q.shape[0]
    R, ps, pris = [], [], []
    for j in range(n):
        alpha, A, theta, D, sigma, offset = Lk[j, :6]
        p = int(sigma) != 0
        th = np.full(N, theta) if p else q[:, j] + offset
        d = q[:, j] + offset if p else np.full(N, D)
        sa, ca = np.sin(alpha), np.cos(alpha)
        R.append(_rot(mdh, np.sin(th), np.cos(th), sa, ca))
        ps.append(np.stack([np.full(N, A), (-d if mdh else d) * sa, d * ca], -1))
        pris.append(p)
    return R, ps, pris


def rne_wrench(n, mdh, L, grav, q, qd, qdd, fext=None):
    """(tau (N,n), wbase (N,6)) of the ne.c recursion for every row."""
    Lk = _links(n, L)
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    N = q.shape[0]
    R, ps, pris = _geometry(n, mdh, L, q)
    g = np.broadcast_to(np.asarray(grav, dtype=np.float64), (N, 3))
    fx = np.zeros(6) if fext is None else np.asarray(fext, dtype=np.float64).reshape(6)
    f_tip, n_tip = np.broadcast_to(fx[:3], (N, 3)), np.broadcast_to(fx[3:], (N, 3))
    z = np.zeros((N, 3))
    w, wd, acc, abar = [None] * n, [None] * n, [None] * n, [None] * n
    for j in range(n):
        qdv, qddv = z.copy(), z.copy()
        qdv[:, 2], qddv[:, 2] = qd[:, j], qdd[:, j]
        rc = Lk[j, 7:10]
        if mdh:
            if not pris[j]:
                if j == 0:
                    w[j], wd[j], t1 = qdv, qddv, g
                else:
                    t1 = _tmul(R[j], w[j - 1])
                    w[j] = t1 + qdv
                    wd[j] = np.cross(t1, qdv) + _tmul(R[j], wd[j - 1]) + qddv
                    t1 = np.cross(wd[j - 1], ps[j]) + np.cross(w[j - 1], np.cross(w[j - 1], ps[j])) + acc[j - 1]
                acc[j] = _tmul(R[j], t1)
            elif j == 0:  # sic, ne.c:187-204
                w[j], wd[j], acc[j] = qdv, qddv, np.array(g)
            else:
                w[j] = _tmul(R[j], w[j - 1])
                wd[j] = _tmul(R[j], wd[j - 1])
                t1 = np.cross(wd[j - 1], ps[j]) + np.cross(w[j - 1], np.cross(w[j - 1], ps[j])) + acc[j - 1]
                acc[j] = _tmul(R[j], t1) + 2.0 * np.cross(_tmul(R[j], w[j - 1]), qdv) + qddv
        else:
            if not pris[j]:
                w[j] = _tmul(R[j], qdv if j == 0 else w[j - 1] + qdv)
                wd[j] = _tmul(R[j], qddv if j == 0 else wd[j - 1] + qddv + np.cross(w[j - 1], qdv))
                acc[j] = (np.cross(wd[j], ps[j]) + np.cross(w[j], np.cross(w[j], ps[j]))
                          + _tmul(R[j], g if j == 0 else acc[j - 1]))
            else:
                if j == 0:
                    w[j], wd[j] = z.copy(), z.copy()
                    acc[j] = _tmul(R[j], qddv + g)
                else:
                    w[j], wd[j] = _tmul(R[j], w[j - 1]), _tmul(R[j], wd[j - 1])
                    acc[j] = _tmul(R[j], qddv + acc[j - 1])
                acc[j] = (acc[j] + np.cross(wd[j], ps[j]) + 2.0 * np.cross(w[j], _tmul(R[j], qdv))
                          + np.cross(w[j], np.cross(w[j], ps[j])))
        abar[j] = np.cross(wd[j], rc) + np.cross(w[j], np.cross(w[j], rc)) + acc[j]
    f, nn = [None] * n, [None] * n
    for j in reversed(range(n)):
        m, rc = Lk[j, 6], Lk[j, 7:10]
        I = Lk[j, 10:19].reshape(3, 3)
        Nv = wd[j] @ I + np.cross(w[j], w[j] @ I)  # column-major read of I (vmath.c mat_vect_mult)
        F = m * abar[j]
        if mdh:
            if j == n - 1:
                f[j], t1 = f_tip + F, n_tip
            else:
                Rf = _mul(R[j + 1], f[j + 1])
                f[j] = Rf + F
                t1 = _mul(R[j + 1], nn[j + 1]) + np.cross(ps[j + 1], Rf)
            nn[j] = t1 + np.cross(rc, F) + Nv
        else:
            t1 = np.cross(ps[j] + rc, F)
            if j != n - 1:
                f[j] = F + _mul(R[j + 1], f[j + 1])
                t1 = t1 + _mul(R[j + 1], np.cross(_tmul(R[j + 1], ps[j]), f[j + 1]) + nn[j + 1])
            else:
                f[j] = F + f_tip
                t1 = t1 + np.cross(ps[j], f_tip) + n_tip
            nn[j] = t1 + Nv
    tau = np.empty((N, n))
    for j in range(n):
        Jm, G, B, Tcp, Tcm = Lk[j, 19:24]
        zax = np.array([0.0, 0.0, 1.0]) if mdh else R[j][:, 2, :]  # R_j^T z0 = the third row of R_j
        t = np.sum((f[j] if pris[j] else nn[j]) * zax, -1)
        t = t + G * G * Jm * qdd[:, j] + G * G * B * qd[:, j]
        tau[:, j] = t + abs(G) * (np.where(qd[:, j] > 0, Tcp, 0.0) + np.where(qd[:, j] < 0, Tcm, 0.0))
    f0 = _mul(R[0], f[0])
    n0 = _mul(R[0], nn[0])
    if mdh:
        n0 = n0 + np.cross(ps[0], f0)
    return tau, np.concatenate([f0, n0], -1)


# ------------------------------------------------------------------ whole-robot momentum balance
def _kinematics(n, mdh, L, q):
    """Link frames in frame 0: R (N,n,3,3), origins (N,n,3), centres of mass (N,n,3)."""
    Lk = _links(n, L)
    R, ps, _ = _geometry(n, mdh, L, q)
    N = R[0].shape[0]
    Ra, pa = np.broadcast_to(np.eye(3), (N, 3, 3)), np.zeros((N, 3))
    Rs, Os, Cs = [], [], []
    for j in range(n):
        step = ps[j] if mdh else _mul(R[j], ps[j])  # frame j's origin in frame j-1
        pa = pa + _mul(Ra, step)
        Ra = Ra @ R[j]
        Rs.append(Ra), Os.append(pa), Cs.append(pa + _mul(Ra, np.broadcast_to(Lk[j, 7:10], (N, 3))))
    return np.stack(Rs, 1), np.stack(Os, 1), np.stack(Cs, 1)


def _momenta(n, mdh, L, q, qd, qdd, t, d):
    """Linear momentum P and angular momentum about O_0, H, at time t of q(t) = q + qd t + qdd t^2 / 2."""
    Lk = _links(n, L)
    path = lambda s: q + qd * s + 0.5 * qdd * s * s  # noqa: E731
    R, _, c = _kinematics(n, mdh, L, path(t))
    Rp, _, cp = _kinematics(n, mdh, L, path(t + d))
    Rm, _, cm = _kinematics(n, mdh, L, path(t - d))
    v = (cp - cm) / (2 * d)
    W = ((Rp - Rm) / (2 * d)) @ R.transpose(0, 1, 3, 2)  # skew(omega)
    om = 0.5 * np.stack([W[..., 2, 1] - W[..., 1, 2], W[..., 0, 2] - W[..., 2, 0], W[..., 1, 0] - W[..., 0, 1]], -1)
    m = Lk[:, 6][None, :, None]
    I = Lk[:, 10:19].reshape(n, 3, 3)
    Iw = np.einsum("nkij,kjl,nkml,nkm->nki", R, I, R, om)  # R I R^T omega
    return (m * v).sum(1), (np.cross(c, m * v) + Iw).sum(1)


def momentum_balance(n, mdh, L, g_b, q, qd, qdd, fext=None, h=1e-3, d=1e-5):
    """(f_0, n_0) = the wrench the base must exert on link 1 (frame 0, moment about O_0); g_b the gravity in frame 0."""
    Lk = _links(n, L)
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    # five-point central differences in t (truncation O(h^4)); the momenta themselves from central differences in d
    PH = {k: _momenta(n, mdh, L, q, qd, qdd, k * h, d) for k in (-2, -1, 1, 2)}
    ddt = lambda i: (PH[-2][i] - 8 * PH[-1][i] + 8 * PH[1][i] - PH[2][i]) / (12 * h)  # noqa: E731
    Rn, On, c = _kinematics(n, mdh, L, q)
    m = Lk[:, 6]
    g_b = np.asarray(g_b, dtype=np.float64)
    f0 = ddt(0) - m.sum() * g_b
    n0 = ddt(1) - np.cross((m[None, :, None] * c).sum(1), g_b)
    if fext is not None:
        fx = np.asarray(fext, dtype=np.float64).reshape(6)
        Rf = _mul(Rn[:, -1], np.broadcast_to(fx[:3], (q.shape[0], 3)))
        f0 = f0 + Rf
        n0 = n0 + _mul(Rn[:, -1], np.broadcast_to(fx[3:], (q.shape[0], 3))) + np.cross(On[:, -1], Rf)
    return np.concatenate([f0, n0], -1)


def at_rest(n, mdh, L, g_b, q):
    """Closed form for qd = qdd = 0 and no tip wrench: f_0 = -M g_b, n_0 = -sum m_i p_ci x g_b."""
    m = _links(n, L)[:, 6]
    _, _, c = _kinematics(n, mdh, L, np.atleast_2d(q))
    g_b = np.asarray(g_b, dtype=np.float64)
    return np.concatenate([np.broadcast_to(-m.sum() * g_b, (c.shape[0], 3)), -np.cross((m[None, :, None] * c).sum(1), g_b)], -1)


# ------------------------------------------------------------------ six virtual joints in front of the links
def _rz(t):
    return ch.trotz(t)


def virtual_joint_tree(n, mdh, L):
    """A rigid-body tree (orc.tree_rne's form) of six massless joints tx, ty, tz, Rx, Ry, Rz followed by the n links,
    each link with its full spatial inertia (mass, centre of mass and rotational inertia) in its joint frame."""
    Lk = _links(n, L)
    parent = list(range(-1, 5))
    axis = [3, 4, 5, 0, 1, 2]
    Cs = [np.eye(4)] * 6
    I6 = [np.zeros((6, 6))] * 6
    prev_tail = np.eye(4)
    for j in range(n):
        alpha, A, theta, D, sigma, offset = Lk[j, :6]
        pris = int(sigma) != 0
        if not mdh:
            pre = _rz(theta) @ ch.transl(0, 0, offset) if pris else _rz(offset)
            post = (ch.transl(A, 0, 0) if pris else ch.transl(0, 0, D) @ ch.transl(A, 0, 0)) @ ch.trotx(alpha)
        else:
            pre = ch.trotx(alpha) @ ch.transl(A, 0, 0) @ (_rz(theta) @ ch.transl(0, 0, offset) if pris else _rz(offset))
            post = np.eye(4) if pris else ch.transl(0, 0, D)
        Cs.append(prev_tail @ pre)
        axis.append(5 if pris else 2)
        parent.append(5 + j)
        m, r, I = Lk[j, 6], Lk[j, 7:10], Lk[j, 10:19].reshape(3, 3)
        Rp = post[:3, :3]
        S = orc.spatial_inertia(m, Rp @ r + post[:3, 3])
        S[3:, 3:] += Rp @ I @ Rp.T
        I6.append(S)
        prev_tail = post
    k = n + 6
    return dict(parent=parent, axis=axis, flip=[0] * k, jindex=list(range(k)), C=Cs, I6=I6)


def tree_wrench(n, mdh, L, q, qd, qdd, gravity):
    """The six virtual-joint torques at zero virtual coordinates; gravity = the robot's gravity in frame 0."""
    q, qd, qdd = (np.atleast_2d(np.asarray(x, dtype=np.float64)) for x in (q, qd, qdd))
    z = np.zeros((q.shape[0], 6))
    Q = orc.tree_rne(virtual_joint_tree(n, mdh, L), np.hstack([z, q]), np.hstack([z, qd]), np.hstack([z, qdd]), gravity)
    return Q[:, :6]


# ------------------------------------------------------------------ test robots
def random_links(rng, n, mdh, prismatic=False):
    """Arm with structural zeros, non-zero rotational inertia (symmetric), actuator terms; with `prismatic` about every
    other joint is translational."""
    links = []
    for k in range(n):
        alpha = rng.choice([0.0, np.pi / 2, -np.pi / 2, np.pi, rng.uniform(-1, 1)])
        I6 = rng.uniform(0.01, 0.5, 3).tolist() + (rng.uniform(-0.01, 0.01, 3) * rng.integers(0, 2, 3)).tolist()
        links.append(dict(d=float(rng.choice([0.0, rng.uniform(-0.5, 0.5)])), a=float(rng.choice([0.0, rng.uniform(-0.5, 0.5)])),
                          alpha=float(alpha), offset=float(rng.choice([0.0, rng.uniform(-1, 1)])),
                          I=I6, r=(rng.uniform(-0.3, 0.3, 3) * rng.integers(0, 2, 3)).tolist(), m=float(rng.uniform(0.1, 5)),
                          Jm=float(rng.choice([0.0, 2e-4])), G=float(rng.choice([0.0, -60.0, 100.0])),
                          B=float(rng.choice([0.0, 1e-3])), Tc=[float(rng.choice([0.0, 0.3])), float(rng.choice([0.0, -0.4]))]))
        if prismatic and (k % 2 == 1 or rng.random() < 0.3):
            links[-1].update(sigma=1, theta=float(rng.choice([0.0, np.pi / 2, rng.uniform(-1, 1)])))
    return links


def robots():
    """(name, n, mdh, L, physical): Puma560, UR10, the MDH Panda and random DH / MDH tables with n = 1..10, some with
    prismatic joints.  physical = False for MDH with a prismatic first joint: the recursion keeps ne.c's quirk there
    (base acceleration taken over unrotated, joint rate put into w), so the physical identities do not hold."""
    rng = np.random.default_rng(2024)
    out = [("puma560", 6, 0, ch.pack_rne(ch.puma560_links()), True), ("ur10", 6, 0, ch.pack_rne(ch.ur10_links()), True),
           ("panda_mdh", 7, 1, ch.pack_rne(ch.panda_mdh_links(), mdh=True), True)]
    for n in range(1, 11):
        for mdh in (0, 1):
            out.append((f"rand_n{n}_{'mdh' if mdh else 'dh'}", n, mdh, ch.pack_rne(random_links(rng, n, mdh), mdh=bool(mdh)), True))
    for k, (n, mdh) in enumerate([(4, 0), (5, 1), (3, 0), (6, 1), (1, 0)]):
        links = random_links(rng, n, mdh, prismatic=True)
        if k == 2:
            links[0].update(sigma=1, theta=0.3)  # prismatic first joint, standard DH: physical
        out.append((f"prismatic{k}_n{n}_{'mdh' if mdh else 'dh'}", n, mdh, ch.pack_rne(links, mdh=bool(mdh)),
                    not (mdh and int(links[0].get("sigma", 0)))))
    links = random_links(rng, 3, 1, prismatic=True)
    links[0].update(sigma=1, theta=0.2)
    out.append(("prismatic_first_mdh_n3", 3, 1, ch.pack_rne(links, mdh=True), False))
    return out
