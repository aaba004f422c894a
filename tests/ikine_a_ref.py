"""Restatement of DHRobot.ikine_a -- the closed-form inverse kinematics of a Puma-type 6R arm that the reference
implements as DHRobot.ikine_6s (Puma560.ikine_a) -- in numpy, one row per pose, step by step as DESIGN (f-6) states
it: wrist centre, shoulder, elbow, then tr2eul of the wrist rotation.  Test infrastructure only:
test_ikine_a_cpu.py pins it by round trips through the oracle's forward kinematics and by the configuration
predicates of config_of; test_gpu_ikine_a.py checks the device against it.

Every function takes the robot's DH table as `dh` = (6, 4) rows of (d, a, alpha, offset), and the robot's base and tool.
"""
import numpy as np

from oracle import oracle as orc

EPS = np.finfo(np.float64).eps
LETTERS = ("lr", "ud", "nf")


def dh_table(robot):
    return np.array([[l.d, l.a, l.alpha, l.offset] for l in robot.links], dtype=np.float64)


def code_of(config):
    """"lun" -> 0 ... "rdf" -> 7: bit 0 = r, bit 1 = d, bit 2 = f"""
    return int("r" in config) | (int("d" in config) << 1) | (int("f" in config) << 2)


def letters_of(code):
    return "".join(pair[(code >> k) & 1] for k, pair in enumerate(LETTERS))


def wrap(x):
    return np.mod(x + np.pi, 2 * np.pi) - np.pi


def fk(robot, q):
    """the oracle's forward kinematics of the robot's ETS (base, offsets and tool included)"""
    return orc.Chain(robot.ets().describe()).fkine(np.atleast_2d(q))


def _link(theta, d, a, alpha):
    """(N,4,4) standard DH link transforms Rz(theta) Tz(d) Tx(a) Rx(alpha)"""
    ct, st, ca, sa = np.cos(theta), np.sin(theta), np.cos(alpha), np.sin(alpha)
    A = np.zeros(theta.shape + (4, 4))
    A[:, 0] = np.stack([ct, -st * ca, st * sa, a * ct], -1)
    A[:, 1] = np.stack([st, ct * ca, -ct * sa, a * st], -1)
    A[:, 2, 1], A[:, 2, 2], A[:, 2, 3], A[:, 3, 3] = sa, ca, d, 1
    return A


def _rx(alpha):
    c, s = np.cos(alpha), np.sin(alpha)
    return np.array([[1, 0, 0, 0], [0, c, -s, 0], [0, s, c, 0], [0, 0, 0, 1.0]])


def tr2eul(R, flip=False):
    """R = Rz(phi) Ry(theta) Rz(psi) -> (phi, theta, psi), (N,3,3) -> (N,3); flip picks the other phi (theta < 0)"""
    sing = (np.abs(R[:, 0, 2]) < 10 * EPS) & (np.abs(R[:, 1, 2]) < 10 * EPS)
    phi = np.arctan2(-R[:, 1, 2], -R[:, 0, 2]) if flip else np.arctan2(R[:, 1, 2], R[:, 0, 2])
    phi = np.where(sing, 0.0, phi)
    sp, cp = np.where(sing, 0.0, np.sin(phi)), np.where(sing, 1.0, np.cos(phi))
    theta = np.arctan2(cp * R[:, 0, 2] + sp * R[:, 1, 2], R[:, 2, 2])
    psi = np.arctan2(-sp * R[:, 0, 0] + cp * R[:, 1, 0], -sp * R[:, 0, 1] + cp * R[:, 1, 1])
    return np.stack([phi, theta, psi], -1)


def ikine_a(dh, base, tool, T, config):
    """-> q (N,6) wrapped into [-pi, pi), ok (N,) bool; rows that are out of reach get NaN"""
    code = code_of(config) if isinstance(config, str) else int(config)
    right, down, flip = code & 1, (code >> 1) & 1, (code >> 2) & 1
    d, a, alpha, off = dh.T
    T = np.asarray(T, dtype=np.float64).reshape(-1, 4, 4)
    N = T.shape[0]
    # 1. wrist centre
    Tt = np.eye(4)
    Tt[0, 3], Tt[2, 3] = a[5], d[5]
    Tt = Tt @ _rx(alpha[5])
    W = np.linalg.inv(base) @ T @ np.linalg.inv(Tt @ tool)  # base^-1 T tool^-1 Tt^-1
    Px, Py, Pz = W[:, 0, 3], W[:, 1, 3], W[:, 2, 3]
    Z, D, r = Pz - d[0], d[1] + d[2], np.hypot(Px, Py)
    with np.errstate(invalid="ignore", divide="ignore"):
        # 2. shoulder
        ok = np.abs(D) <= r
        s = np.arcsin(D / r)
        th1 = np.arctan2(Py, Px) + (s if right else np.pi - s)
        # 3. elbow
        V = Px * np.cos(th1) + Py * np.sin(th1)
        c = (a[1] ** 2 + V ** 2 + Z ** 2 - a[2] ** 2 - d[3] ** 2) / (2 * a[1] * np.sqrt(V ** 2 + Z ** 2))
        ok &= np.isfinite(c) & (np.abs(c) <= 1)
        # a2 < 0 mirrors the upper arm: without the sign of a2, "u" would put the elbow below the shoulder-wrist line
        n2 = (-1 if down else 1) * (1 if right else -1) * np.sign(a[1])
        th2 = np.arctan2(Z, V) + n2 * np.arccos(c)
        # 4. forearm
        num = np.cos(th2) * V + np.sin(th2) * Z - a[1]
        den = np.cos(th2) * Z - np.sin(th2) * V
        th3 = np.arctan2(a[2], d[3]) - np.arctan2(num, den)
        # 5. wrist: R = R(A1 A2 A3)^T R(W), ZYZ Euler angles
        A123 = _link(th1, d[0], a[0], alpha[0]) @ _link(th2, d[1], a[1], alpha[1]) @ _link(th3, d[2], a[2], alpha[2])
        R = A123[:, :3, :3].transpose(0, 2, 1) @ W[:, :3, :3]
        e = tr2eul(R, bool(flip))
        if alpha[3] > 0:
            e[:, 1] = -e[:, 1]
    theta = np.concatenate([np.stack([th1, th2, th3], -1), e], -1)
    q = wrap(theta - off)
    q[~ok] = np.nan
    return q.reshape(N, 6), ok


def config_code(dh, q):
    """The configuration a joint vector satisfies, as a code (bit 0 = r, bit 1 = d, bit 2 = f): r iff V(q) > 0, u iff
    the elbow is above the shoulder-wrist line (sign(V) (V a2 s2 - Z a2 c2) > 0), n iff sign(alpha4) sin(theta5) < 0"""
    d, a, alpha, off = dh.T
    th = np.atleast_2d(q) + off
    c2, s2, c23, s23 = np.cos(th[:, 1]), np.sin(th[:, 1]), np.cos(th[:, 1] + th[:, 2]), np.sin(th[:, 1] + th[:, 2])
    V = a[1] * c2 + a[2] * c23 - d[3] * s23
    Z = a[1] * s2 + a[2] * s23 + d[3] * c23
    right = V > 0
    up = np.sign(V) * (V * a[1] * s2 - Z * a[1] * c2) > 0
    noflip = np.sign(alpha[3]) * np.sin(th[:, 4]) < 0
    return right.astype(int) | (~up).astype(int) << 1 | (~noflip).astype(int) << 2


def config_of(dh, q):
    """config_code as letters, one string per row"""
    return [letters_of(c) for c in config_code(dh, q)]


def margins(dh, base, tool, T, config):
    """Per row: |c| of the elbow, |sin theta5| and r - |D| -- the distances to the branch boundaries"""
    q, ok = ikine_a(dh, base, tool, T, config)
    d, a, alpha, off = dh.T
    T = np.asarray(T, dtype=np.float64).reshape(-1, 4, 4)
    Tt = np.eye(4)
    Tt[0, 3], Tt[2, 3] = a[5], d[5]
    W = np.linalg.inv(base) @ T @ np.linalg.inv(Tt @ _rx(alpha[5]) @ tool)
    Px, Py, Pz = W[:, 0, 3], W[:, 1, 3], W[:, 2, 3]
    Z, r = Pz - d[0], np.hypot(Px, Py)
    th1 = q[:, 0] + off[0]
    V = Px * np.cos(th1) + Py * np.sin(th1)
    with np.errstate(invalid="ignore", divide="ignore"):
        c = (a[1] ** 2 + V ** 2 + Z ** 2 - a[2] ** 2 - d[3] ** 2) / (2 * a[1] * np.sqrt(V ** 2 + Z ** 2))
    return np.abs(c), np.abs(np.sin(q[:, 4] + off[4])), r - abs(d[1] + d[2])


def random_se3(rng, scale=0.3):
    """a random rigid transform: rotation from a normalised quaternion, translation up to `scale`"""
    w, x, y, z = rng.normal(size=4)
    n = np.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    T = np.eye(4)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                 [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                 [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]
    T[:3, 3] = rng.uniform(-scale, scale, 3)
    return T


def random_robot(rtb, rng, wrist_sign):
    """A random standard-DH 6R arm of the Puma pattern: alpha = (pi/2, 0, -pi/2, s pi/2, -s pi/2, any), a1 = a4 = a5 = 0,
    d5 = 0, everything else random -- offsets, d6 / a6 / alpha6, a base and a tool included"""
    h = np.pi / 2
    d = [rng.uniform(0.2, 0.8), rng.uniform(-0.2, 0.2), rng.uniform(-0.2, 0.2), rng.uniform(0.2, 0.6), 0.0, rng.uniform(0, 0.2)]
    a = [0.0, rng.uniform(0.2, 0.6) * rng.choice([-1, 1]), rng.uniform(-0.1, 0.1), 0.0, 0.0, rng.uniform(-0.1, 0.1)]
    alpha = [h, 0.0, -h, wrist_sign * h, -wrist_sign * h, rng.uniform(-np.pi, np.pi)]
    off = rng.uniform(-np.pi, np.pi, 6)
    links = [rtb.RevoluteDH(d=d[j], a=a[j], alpha=alpha[j], offset=off[j]) for j in range(6)]
    return rtb.DHRobot(links, name="pattern", base=random_se3(rng), tool=random_se3(rng, 0.1))
