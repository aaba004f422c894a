"""Restatement of DHRobot.ikine_ur -- the closed-form inverse kinematics of a UR-type 6R arm -- in numpy, one row per
pose, step by step as DESIGN (f-15) states it: fold base, tool and the last link's constant part, shoulder, wrist from the
first axis, then the planar three-link problem of the parallel axes 2, 3 and 4.  Test infrastructure only:
test_ikine_ur_cpu.py pins it by round trips through the oracle's forward kinematics and by the configuration predicates
of config_of; test_gpu_ikine_ur.py checks the device against it.

Every function takes the robot's DH table as `dh` = (6, 4) rows of (d, a, alpha, offset), and the robot's base and tool.
"""
import numpy as np

from ikine_a_ref import code_of, dh_table, fk, letters_of, random_se3, wrap  # noqa: F401  (re-exported for the tests)

EPS = np.finfo(np.float64).eps
# |c3| up to 1 + ELBOW_BAND eps counts as reached (and is clamped to 1): a straight elbow, such as UR10's qz and qr, gives
# c3 = 1 up to the rounding of the fold and of X^2 + Y^2
ELBOW_BAND = 64


def _rx(alpha):
    c, s = np.cos(alpha), np.sin(alpha)
    return np.array([[1, 0, 0, 0], [0, c, -s, 0], [0, s, c, 0], [0, 0, 0, 1.0]])


def fold(dh, base, tool, T):
    """T' = base^-1 T tool^-1 Tt^-1 with Tt = transl(a6, 0, d6) Rx(alpha6), so that T' = A1 ... A5 Rz(theta6)"""
    d, a, alpha, _ = dh.T
    Tt = np.eye(4)
    Tt[0, 3], Tt[2, 3] = a[5], d[5]
    return np.linalg.inv(base) @ np.asarray(T, dtype=np.float64).reshape(-1, 4, 4) @ np.linalg.inv(Tt @ _rx(alpha[5]) @ tool)


def _solve(dh, base, tool, T, config):
    """-> theta (N,6) before offsets, ok (N,), and the margins (1 - |c3|, |sin theta5|, r - |D|, |X|)"""
    code = code_of(config) if isinstance(config, str) else int(config)
    right, down, flip = code & 1, (code >> 1) & 1, (code >> 2) & 1
    d, a, _, _ = dh.T
    W = fold(dh, base, tool, T)
    xp, yp, zp, p = W[:, :3, 0], W[:, :3, 1], W[:, :3, 2], W[:, :3, 3]
    D = d[1] + d[2] + d[3]
    r = np.hypot(p[:, 0], p[:, 1])
    zero = np.zeros_like(r)
    with np.errstate(invalid="ignore", divide="ignore"):
        # 1. shoulder: p . z1 = D
        ok = np.abs(D) <= r
        s = np.arcsin(D / r)
        th1 = np.arctan2(p[:, 1], p[:, 0]) + (s if right else np.pi - s)
        c1, s1 = np.cos(th1), np.sin(th1)
        x1, z1 = np.stack([c1, s1, zero], -1), np.stack([s1, -c1, zero], -1)
        # 2. wrist: z1 in the tool-side frame is (s5 c6, -s5 s6, c5)
        u, v, w = (xp * z1).sum(-1), (yp * z1).sum(-1), (zp * z1).sum(-1)
        sg = -1.0 if flip else 1.0
        th5 = np.arctan2(sg * np.hypot(u, v), w)
        sing = (np.abs(u) < 10 * EPS) & (np.abs(v) < 10 * EPS)
        th6 = np.where(sing, 0.0, np.arctan2(-sg * v, sg * u))
        c5, s5, c6, s6 = np.cos(th5), np.sin(th5), np.cos(th6), np.sin(th6)
        # 3. the planar problem in the plane normal to z1
        O4 = p + d[4] * (s6[:, None] * xp + c6[:, None] * yp)
        X, Y = (O4 * x1).sum(-1), O4[:, 2] - d[0]
        x4 = c5[:, None] * (c6[:, None] * xp - s6[:, None] * yp) - s5[:, None] * zp
        th234 = np.arctan2(x4[:, 2], (x4 * x1).sum(-1))
        # 4. elbow
        c3 = (X * X + Y * Y - a[1] ** 2 - a[2] ** 2) / (2 * a[1] * a[2])
        ok &= np.abs(c3) <= 1 + ELBOW_BAND * EPS
        sx = np.where(X >= 0, 1.0, -1.0)
        th3 = (1.0 if down else -1.0) * sx * np.sign(a[1] * a[2]) * np.arccos(np.clip(c3, -1, 1))
        th2 = np.arctan2(Y, X) - np.arctan2(a[2] * np.sin(th3), a[1] + a[2] * np.cos(th3))
        th4 = th234 - th2 - th3
    theta = np.stack([th1, th2, th3, th4, th5, th6], -1)
    return theta, ok, (1 - np.abs(c3), np.abs(np.sin(th5)), r - abs(D), np.abs(X))


def ikine_ur(dh, base, tool, T, config):
    """-> q (N,6) wrapped into [-pi, pi), ok (N,) bool; rows that are out of reach get NaN"""
    theta, ok, _ = _solve(dh, base, tool, T, config)
    q = wrap(theta - dh[:, 3])
    q[~ok] = np.nan
    return q, ok


def margins(dh, base, tool, T, config):
    """Per row of the solution in `config`: 1 - |c3| (elbow), |sin theta5| (wrist), r - |D| (shoulder) and |X| (the
    elbow letter's sign(X)) -- the distances to the branch boundaries"""
    return _solve(dh, base, tool, T, config)[2]


def config_code(dh, q):
    """The configuration a joint vector satisfies, as a code (bit 0 = r, bit 1 = d, bit 2 = f), in the frame of link 1:
    r iff O5 . x1 = X + d5 sin(theta234) >= 0; u iff the elbow O3 lies above the shoulder-O4 line, sign(X) (X a2 s2 -
    Y a2 c2) > 0 with X = a2 c2 + a3 c23, Y = a2 s2 + a3 s23; n iff sin(theta5) >= 0"""
    d, a, _, off = dh.T
    th = np.atleast_2d(q) + off
    t2, t23, t234 = th[:, 1], th[:, 1] + th[:, 2], th[:, 1] + th[:, 2] + th[:, 3]
    X = a[1] * np.cos(t2) + a[2] * np.cos(t23)
    Y = a[1] * np.sin(t2) + a[2] * np.sin(t23)
    right = X + d[4] * np.sin(t234) >= 0
    up = np.where(X >= 0, 1.0, -1.0) * (X * a[1] * np.sin(t2) - Y * a[1] * np.cos(t2)) > 0
    near = np.sin(th[:, 4]) >= 0
    return right.astype(int) | (~up).astype(int) << 1 | (~near).astype(int) << 2


def config_of(dh, q):
    """config_code as letters, one string per row"""
    return [letters_of(c) for c in config_code(dh, q)]


def random_robot(rtb, rng):
    """A random standard-DH 6R arm of the UR pattern: alpha = (pi/2, 0, 0, pi/2, -pi/2, any), a1 = a4 = a5 = 0, a2 and a3
    of either sign, d2 and d3 nonzero, everything else random -- offsets, d6 / a6 / alpha6, a base and a tool included"""
    h = np.pi / 2
    d = [rng.uniform(0.1, 0.5), rng.uniform(0.05, 0.2) * rng.choice([-1, 1]), rng.uniform(0.05, 0.2) * rng.choice([-1, 1]),
         rng.uniform(-0.2, 0.2), rng.uniform(0.05, 0.2) * rng.choice([-1, 1]), rng.uniform(0, 0.2)]
    a = [0.0, rng.uniform(0.2, 0.7) * rng.choice([-1, 1]), rng.uniform(0.2, 0.7) * rng.choice([-1, 1]), 0.0, 0.0,
         rng.uniform(-0.1, 0.1)]
    alpha = [h, 0.0, 0.0, h, -h, rng.uniform(-np.pi, np.pi)]
    off = rng.uniform(-np.pi, np.pi, 6)
    links = [rtb.RevoluteDH(d=d[j], a=a[j], alpha=alpha[j], offset=off[j]) for j in range(6)]
    return rtb.DHRobot(links, name="ur-pattern", base=random_se3(rng), tool=random_se3(rng, 0.1))
