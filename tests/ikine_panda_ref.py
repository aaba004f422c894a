"""Restatement of DHRobot.ikine_panda -- the closed-form inverse kinematics of a Panda-type 7R arm at a given q7 -- in
numpy, one row per pose, step by step as DESIGN (f-17) states it: fold base, tool and the last link at theta7, elbow from
the distance O6-O2, wrist from the elbow triangle, then ZYZ Euler angles of the shoulder rotation.  Test infrastructure
only: test_ikine_panda_cpu.py pins it by round trips through the oracle's modified-DH forward kinematics and by the
configuration predicates of config_of; test_gpu_ikine_panda.py checks the device against it.

Every function takes the robot's MDH table as `dh` = (7, 4) rows of (d, a, alpha, offset), link k being
Rx(alpha_k) Tx(a_k) Rz(theta_k) Tz(d_k), and the robot's base and tool.
"""
import numpy as np

from ikine_a_ref import code_of, dh_table, fk, letters_of, random_se3, tr2eul, wrap  # noqa: F401  (re-exported)
from oracle import chains

EPS = np.finfo(np.float64).eps
# |C / rho| up to 1 + BAND eps and |p| up to h + BAND eps |v| count as reached (and are clamped): on-boundary rows reach
# the boundary only up to rounding (DESIGN f-17 gives the measured overshoot)
BAND = 64


def link(theta, d, a, alpha):
    """(N,4,4) modified-DH link transforms Rx(alpha) Tx(a) Rz(theta) Tz(d)"""
    theta = np.atleast_1d(np.asarray(theta, dtype=np.float64))
    ct, st, ca, sa = np.cos(theta), np.sin(theta), np.cos(alpha), np.sin(alpha)
    A = np.zeros(theta.shape + (4, 4))
    A[:, 0, 0], A[:, 0, 1], A[:, 0, 3] = ct, -st, a
    A[:, 1, 0], A[:, 1, 1], A[:, 1, 2], A[:, 1, 3] = st * ca, ct * ca, -sa, -sa * d
    A[:, 2, 0], A[:, 2, 1], A[:, 2, 2], A[:, 2, 3] = st * sa, ct * sa, ca, ca * d
    A[:, 3, 3] = 1
    return A


def fold(dh, base, tool, T, q7):
    """W = (base Rx(alpha1) Tx(a1))^-1 T (A7(theta7) tool)^-1 = A2 ... A6 with the first link's joint rotation and d1
    left in, so that W is frame 6 in the frame whose origin O1 lies d1 below O2 on the first axis"""
    d, a, alpha, off = dh.T
    T = np.asarray(T, dtype=np.float64).reshape(-1, 4, 4)
    q7 = np.broadcast_to(np.asarray(q7, dtype=np.float64), T.shape[:1])
    head = base @ link(0.0, 0.0, a[0], alpha[0])[0]
    with np.errstate(invalid="ignore"):
        return np.linalg.inv(head) @ T @ np.linalg.inv(link(q7 + off[6], d[6], a[6], alpha[6]) @ tool)


def _solve(dh, base, tool, T, q7, config):
    """-> theta (N,6) of joints 1..6 before offsets, ok (N,), and the margins (1 - |C/rho|, 1 - |p/h|, |sin theta2|, h)"""
    code = code_of(config) if isinstance(config, str) else int(config)
    right, down, flip = code & 1, (code >> 1) & 1, (code >> 2) & 1
    d, a, alpha, off = dh.T
    T = np.asarray(T, dtype=np.float64).reshape(-1, 4, 4)
    q7 = np.broadcast_to(np.asarray(q7, dtype=np.float64), T.shape[:1])
    W = fold(dh, base, tool, T, q7)
    R, p = W[:, :3, :3], W[:, :3, 3]
    O2 = np.array([0.0, 0.0, d[0]])
    d3, a4, a5, d5 = d[2], a[3], a[4], d[4]
    with np.errstate(invalid="ignore", divide="ignore"):
        # v = O6 -> O2 in frame 6
        v = np.einsum("nij,ni->nj", R, O2 - p)
        vx, vy, vz = v[:, 0], v[:, 1], v[:, 2]
        h = np.hypot(vx, vy)
        tiny = 16 * EPS * np.linalg.norm(v, axis=-1)
        axis6 = h <= tiny  # O2 on joint 6's axis: theta6 is free, psi = 0 and the wrist equation reads p = 0
        psi = np.where(axis6, 0.0, np.arctan2(vy, vx))
        # 1. elbow
        A, B = -a4 * a5 - d3 * d5, a4 * d5 - d3 * a5
        rho, phi = np.hypot(A, B), np.arctan2(B, A)
        cr = (a4 ** 2 + d3 ** 2 + a5 ** 2 + d5 ** 2 - (v * v).sum(-1)) / 2 / rho
        ok = np.isfinite(q7) & (np.abs(cr) <= 1 + BAND * EPS)
        th4 = phi + (-1.0 if down else 1.0) * np.arccos(np.clip(cr, -1, 1))
        c4, s4 = np.cos(th4), np.sin(th4)
        # 2. the triangle in frame 4: O4 -> O2 is (gx, gy), O4 -> O6 is (a5, d5)
        r = -a4 * c4 - d3 * s4 - a5
        pw = a4 * s4 - d3 * c4 - d5
        # 3. wrist: v_x s6 + v_y c6 = p, theta6 + psi = asin(p / h) = atan2(p, w) with w = c5 r = sqrt(h^2 - p^2) =
        # sqrt(r^2 - v_z^2), taken from the smaller squares; |r| at rounding puts O2 on joint 5's axis (theta5 free)
        axis5 = np.abs(r) <= tiny
        ps = np.where(axis6, 0.0, pw / h)
        ok &= np.abs(pw) - h <= BAND * EPS * np.linalg.norm(v, axis=-1)
        w2 = np.where(np.abs(r) < h, (r - vz) * (r + vz), (h - pw) * (h + pw))
        asn = np.where(axis6, 0.0, np.arctan2(pw, np.sqrt(np.maximum(w2, 0.0))))
        th6 = (np.pi - asn if flip else asn) - psi
        c6, s6 = np.cos(th6), np.sin(th6)
        # 4. theta5, 0 where O2 lies on joint 5's axis
        vu = vx * c6 - vy * s6
        sg = np.where(r >= 0, 1.0, -1.0)
        th5 = np.where(axis5, 0.0, np.arctan2(sg * vz, sg * vu))
        # 5. shoulder: R3 = R(W) R(A6)^T R(A5)^T R(A4)^T = Rz(theta1) Ry(theta2) Rz(theta3), tr2eul with its singular rule
        Rt = lambda k, th: link(th, 0.0, 0.0, alpha[k])[:, :3, :3].transpose(0, 2, 1)  # noqa: E731
        R3 = R @ Rt(5, th6) @ Rt(4, th5) @ Rt(3, th4)
        e = tr2eul(R3, flip=not right)
    theta = np.concatenate([e, np.stack([th4, th5, th6], -1)], -1)
    return theta, ok, (1 - np.abs(cr), 1 - np.abs(ps), np.abs(np.sin(e[:, 1])), h)


def ikine_panda(dh, base, tool, T, q7, config):
    """-> q (N,7), joints 1..6 wrapped into [-pi, pi) and q[:, 6] = q7 as given, ok (N,) bool; rows out of reach get NaN"""
    theta, ok, _ = _solve(dh, base, tool, T, q7, config)
    q7 = np.broadcast_to(np.asarray(q7, dtype=np.float64), ok.shape)
    q = np.concatenate([wrap(theta - dh[:6, 3]), q7[:, None]], -1)
    q[~ok] = np.nan
    return q, ok


def margins(dh, base, tool, T, q7, config):
    """Per row of the solution in `config`: 1 - |C/rho| (elbow), 1 - |p/h| (wrist), |sin theta2| (shoulder) and h, the
    distance of O2 from joint 6's axis -- the distances to the branch boundaries and the degenerate wrist"""
    return _solve(dh, base, tool, T, q7, config)[2]


def frames(dh, q):
    """(N,8,4,4) link frames 0 .. 7 of the bare chain (no base, no tool, offsets applied)"""
    d, a, alpha, off = dh.T
    th = np.atleast_2d(q) + off
    F = [np.broadcast_to(np.eye(4), (th.shape[0], 4, 4))]
    for k in range(7):
        F.append(F[-1] @ link(th[:, k], d[k], a[k], alpha[k]))
    return np.stack(F, 1)


def config_code(dh, q):
    """The configuration a joint vector satisfies, as a code (bit 0 = r, bit 1 = d, bit 2 = f), from the link frames:
    r iff sin(theta2) >= 0; u iff ((O2 - O4) x (O6 - O4)) . z4 >= 0; n iff (O2 - O6) . x5 >= 0"""
    q = np.atleast_2d(q)
    F = frames(dh, q)
    O2, O4, O6 = F[:, 2, :3, 3], F[:, 4, :3, 3], F[:, 6, :3, 3]
    right = np.sin(q[:, 1] + dh[1, 3]) >= 0
    up = (np.cross(O2 - O4, O6 - O4) * F[:, 4, :3, 2]).sum(-1) >= 0
    near = ((O2 - O6) * F[:, 5, :3, 0]).sum(-1) >= 0
    return right.astype(int) | (~up).astype(int) << 1 | (~near).astype(int) << 2


def config_of(dh, q):
    """config_code as letters, one string per row"""
    return [letters_of(c) for c in config_code(dh, q)]


def fk_mdh(robot, q):
    """base A1 ... A7 tool through the oracle's modified-DH link transform (oracle.chains.dh_A), one row at a time"""
    Ls = [dict(d=l.d, a=l.a, alpha=l.alpha, offset=l.offset) for l in robot.links]
    out = []
    for row in np.atleast_2d(q):
        T = robot._base.copy()
        for L, qj in zip(Ls, row):
            T = T @ chains.dh_A(L, qj, mdh=True)
        out.append(T @ robot._tool)
    return np.array(out)


def random_robot(rtb, rng):
    """A random modified-DH 7R arm of the Panda pattern: alpha2 .. alpha6 = (-pi/2, pi/2, pi/2, -pi/2, pi/2), a2 = a3 =
    a6 = 0, d2 = d4 = d6 = 0, both signs of d3, a4, a5 and d5, everything else random -- a1, alpha1, d1, a7, alpha7,
    d7, the offsets, a base and a tool included"""
    h = np.pi / 2
    sgn = lambda: rng.choice([-1, 1])  # noqa: E731
    d = [rng.uniform(0.1, 0.5), 0.0, rng.uniform(0.1, 0.5) * sgn(), 0.0, rng.uniform(0.1, 0.5) * sgn(), 0.0, rng.uniform(-0.2, 0.2)]
    a = [rng.uniform(-0.2, 0.2), 0.0, 0.0, rng.uniform(0.02, 0.2) * sgn(), rng.uniform(0.02, 0.2) * sgn(), 0.0,
         rng.uniform(-0.2, 0.2)]
    alpha = [rng.uniform(-np.pi, np.pi), -h, h, h, -h, h, rng.uniform(-np.pi, np.pi)]
    off = rng.uniform(-np.pi, np.pi, 7)
    links = [rtb.RevoluteMDH(d=d[j], a=a[j], alpha=alpha[j], offset=off[j]) for j in range(7)]
    return rtb.DHRobot(links, name="panda-pattern", base=random_se3(rng), tool=random_se3(rng, 0.1))
