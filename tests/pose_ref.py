"""High-precision restatement of the pose-representation kernels: b2k_jacob0_analytical, b2k_p_servo_rpy and b2k_ctraj
(b2k_pose.cu) and the angle-axis pose error of b2k_angle_axis / b2k_p_servo (ik_angle_axis, b2k_ik.cuh).

Test infrastructure only.  Every function restates the definition the kernel implements -- spatialmath's tr2rpy,
tr2eul, rotvelxform(inverse=True) and quaternion slerp, and _angle_axis of ik.cpp -- and evaluates it in mpmath at 50
digits on exactly the numbers the kernel received: fp64 inputs, or the fp32-rounded ones for fp32 runs.  The branch
predicates use the kernel's constant and dtype (10 eps of the dtype for the gimbal bands of rpy and ZYZ, ln < 1e-9 /
1e-6 in trlog, ln < 1e-6 in angle-axis), so that a row on either side of a threshold is compared with the branch the
kernel is specified to take.  test_pose_ref_cpu.py pins this module against the oracle and by identities;
test_gpu_pose_edges.py checks the kernels against it.

Rotations are 3x3 nested lists of mpf (exact) or numpy arrays (converted exactly, element by element).
"""
import mpmath
import numpy as np

M = mpmath.MPContext()
M.dps = 50

EPS = {np.float64: 2.0 ** -52, np.float32: 2.0 ** -23}
REPS = ("rpy/xyz", "rpy/zyx", "eul", "exp")  # the kernel's representation codes 0..3


def _dt(dt):
    return np.dtype(dt).type


def band(dt):
    """the half-width of the gimbal bands of tr2rpy / tr2eul: 10 eps of the dtype (r_eps, b2k_common.cuh)"""
    return 10 * EPS[_dt(dt)]


def trlog_cut(dt):
    """rot_to_exp treats ln = |vex(R - R^T)| below this as theta in {0, pi}: (real)1e-9 * (1 or 1000)"""
    return float(np.float64(1e-9)) if _dt(dt) == np.float64 else float(np.float32(1e-9) * np.float32(1000))


def mpm(R):
    """3x3 (or the rotation part of a 4x4) -> nested lists of mpf, exactly"""
    return [[M.mpf(float(R[i][j])) for j in range(3)] for i in range(3)]


def to_np(R):
    return np.array([[float(x) for x in r] for r in R])


def mul(A, B):
    return [[M.fsum(A[i][k] * B[k][j] for k in range(3)) for j in range(3)] for i in range(3)]


def tp(A):
    return [[A[j][i] for j in range(3)] for i in range(3)]


# ------------------------------------------------------------------ constructing rotations
def rot(axis, angle):
    """Rot(k, angle) = I + sin(angle) [k]x + (1 - cos(angle)) [k]x^2, k = axis / |axis|"""
    k = [M.mpf(a) for a in axis]
    n = M.sqrt(M.fsum(a * a for a in k))
    kx, ky, kz = (a / n for a in k)
    s, c = M.sin(angle), M.cos(angle)
    K = [[0, -kz, ky], [kz, 0, -kx], [-ky, kx, 0]]
    K2 = mul(K, K)
    return [[(1 if i == j else 0) + s * K[i][j] + (1 - c) * K2[i][j] for j in range(3)] for i in range(3)]


def rotx(a):
    return rot((1, 0, 0), a)


def roty(a):
    return rot((0, 1, 0), a)


def rotz(a):
    return rot((0, 0, 1), a)


def rpy2r(roll, pitch, yaw, order):
    """'zyx': Rz(yaw) Ry(pitch) Rx(roll); 'xyz': Rx(yaw) Ry(pitch) Rz(roll)"""
    if order == "zyx":
        return mul(rotz(yaw), mul(roty(pitch), rotx(roll)))
    return mul(rotx(yaw), mul(roty(pitch), rotz(roll)))


def eul2r(phi, theta, psi):
    return mul(rotz(phi), mul(roty(theta), rotz(psi)))


def exp2r(v):
    th = M.sqrt(M.fsum(x * x for x in v))
    return rot(v, th) if th != 0 else [[M.mpf(int(i == j)) for j in range(3)] for i in range(3)]


def pose(R, t=(0, 0, 0), dt=np.float64):
    """4x4 homogeneous transform of the (mpmath) rotation R and translation t, rounded to dt"""
    T = np.eye(4)
    T[:3, :3] = to_np(R)
    T[:3, 3] = [float(x) for x in t]
    return T.astype(dt)


# ------------------------------------------------------------------ rotation -> representation (the kernel's branches)
def tr2rpy(R, order="zyx", dt=np.float64):
    """spatialmath tr2rpy -> (roll, pitch, yaw); inside the band |(|R20| or |R02|) - 1| < 10 eps: roll := 0"""
    R = mpm(R) if isinstance(R, np.ndarray) else R
    b = band(dt)
    if order == "zyx":
        if abs(abs(R[2][0]) - 1) < b:
            yaw = -M.atan2(R[0][1], R[0][2]) if R[2][0] < 0 else M.atan2(-R[0][1], -R[0][2])
            return [M.mpf(0), -M.asin(max(min(R[2][0], 1), -1)), yaw]
        return [M.atan2(R[2][1], R[2][2]), M.atan2(-R[2][0], M.sqrt(R[0][0] ** 2 + R[1][0] ** 2)), M.atan2(R[1][0], R[0][0])]
    if abs(abs(R[0][2]) - 1) < b:
        yaw = M.atan2(R[2][1], R[1][1]) if R[0][2] > 0 else -M.atan2(R[1][0], R[2][0])
        return [M.mpf(0), M.asin(max(min(R[0][2], 1), -1)), yaw]
    return [-M.atan2(R[0][1], R[0][0]), M.atan2(R[0][2], M.sqrt(R[0][0] ** 2 + R[0][1] ** 2)), -M.atan2(R[1][2], R[2][2])]


def tr2eul(R, dt=np.float64):
    """spatialmath tr2eul, R = Rz(phi) Ry(theta) Rz(psi), theta >= 0; phi := 0 when |R02| and |R12| are below 10 eps"""
    R = mpm(R) if isinstance(R, np.ndarray) else R
    b = band(dt)
    if abs(R[0][2]) < b and abs(R[1][2]) < b:
        phi, sp, cp = M.mpf(0), M.mpf(0), M.mpf(1)
    else:
        phi = M.atan2(R[1][2], R[0][2])
        sp, cp = M.sin(phi), M.cos(phi)
    return [phi, M.atan2(cp * R[0][2] + sp * R[1][2], R[2][2]),
            M.atan2(-sp * R[0][0] + cp * R[1][0], -sp * R[0][1] + cp * R[1][1])]


def trlog(R, dt=np.float64):
    """exponential coordinates theta k: atan2(ln, tr - 1) l / ln with l = vex(R - R^T), ln = |l|.  Below the cut
    (trlog_cut) theta is 0 (tr > 0) or pi, with the axis from the diagonal: a_i = sqrt(max((R_ii + 1) / 2, 0)), the
    largest taken positive (the first of equals), the others signed by the off-diagonal entries in its row / column.
    Which a_i is largest is decided on the dtype's own rounding of a_i, as the kernel does."""
    Rn = np.asarray(to_np(R) if isinstance(R, list) else R)
    R = mpm(R) if isinstance(R, np.ndarray) else R
    lx, ly, lz = R[2][1] - R[1][2], R[0][2] - R[2][0], R[1][0] - R[0][1]
    ln = M.sqrt(lx * lx + ly * ly + lz * lz)
    tr = R[0][0] + R[1][1] + R[2][2]
    if ln < trlog_cut(dt):
        if tr > 0:
            return [M.mpf(0)] * 3
        d = _dt(dt)
        ad = [np.sqrt(np.maximum((d(Rn[i, i]) + d(1)) / d(2), d(0))) for i in range(3)]
        a = [M.sqrt(max((R[i][i] + 1) / 2, 0)) for i in range(3)]

        def sgn(i, j):  # copysign: the sign bit of the entry the kernel read, -0.0 included
            return float(np.copysign(1.0, Rn[i, j]))

        if ad[0] >= ad[1] and ad[0] >= ad[2]:
            a[1], a[2] = sgn(0, 1) * a[1], sgn(0, 2) * a[2]
        elif ad[1] >= ad[2]:
            a[0], a[2] = sgn(0, 1) * a[0], sgn(1, 2) * a[2]
        else:
            a[0], a[1] = sgn(0, 2) * a[0], sgn(1, 2) * a[1]
        return [M.pi * x for x in a]
    ang = M.atan2(ln, tr - 1)
    return [ang * lx / ln, ang * ly / ln, ang * lz / ln]


def r2x(R, rep, dt=np.float64):
    if rep == "exp":
        return trlog(R, dt)
    if rep == "eul":
        return tr2eul(R, dt)
    return tr2rpy(R, rep[4:], dt)


def x2r(g, rep):
    if rep == "exp":
        return exp2r(g)
    if rep == "eul":
        return eul2r(*g)
    return rpy2r(g[0], g[1], g[2], rep[4:])


# ------------------------------------------------------------------ angular velocity <-> representation rates
def k2(theta):
    """(1 - x cot x) / theta^2, x = theta / 2: the coefficient of [v]x^2 in A^-1 of the exponential coordinates.
    Evaluated with enough extra digits that the cancellation of 1 - x cot x (~ theta^2 / 12) costs nothing."""
    theta = M.mpf(theta)
    if theta == 0:
        return M.mpf(1) / 12
    with M.extradps(int(2 * max(0, -M.log10(abs(theta)))) + 10):
        x = theta / 2
        return (1 - x * M.cot(x)) / theta ** 2


def k2_series(theta):
    """k2 to theta^6: 1/12 + theta^2/720 + theta^4/30240 + theta^6/1209600 (next term theta^8/47900160)"""
    t2 = M.mpf(theta) ** 2
    return M.mpf(1) / 12 + t2 / 720 + t2 ** 2 / 30240 + t2 ** 3 / 1209600


def _skew(v):
    return [[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]]


def rotvelxform(g, rep):
    """A(gamma): omega = A gamma'.  rpy/zyx: omega = yaw' z + pitch' Rz y + roll' Rz Ry x; rpy/xyz: omega = yaw' x +
    pitch' Rx y + roll' Rx Ry z; eul: omega = phi' z + theta' Rz y + psi' Rz Ry z; exp: A = I + (1 - cos) / th^2 [v]x +
    (th - sin) / th^3 [v]x^2"""
    g = [M.mpf(x) for x in g]
    if rep == "rpy/zyx":
        sb, cb, sg, cg = M.sin(g[1]), M.cos(g[1]), M.sin(g[2]), M.cos(g[2])
        return [[cb * cg, -sg, 0], [cb * sg, cg, 0], [-sb, 0, 1]]
    if rep == "rpy/xyz":
        sb, cb, sg, cg = M.sin(g[1]), M.cos(g[1]), M.sin(g[2]), M.cos(g[2])
        return [[sb, 0, 1], [-cb * sg, cg, 0], [cb * cg, sg, 0]]
    if rep == "eul":
        sp, cp, st, ct = M.sin(g[0]), M.cos(g[0]), M.sin(g[1]), M.cos(g[1])
        return [[0, -sp, cp * st], [0, cp, sp * st], [1, 0, ct]]
    th = M.sqrt(M.fsum(x * x for x in g))
    S = _skew(g)
    S2 = mul(S, S)
    if th == 0:
        return [[M.mpf(int(i == j)) for j in range(3)] for i in range(3)]
    a, b = (1 - M.cos(th)) / th ** 2, (th - M.sin(th)) / th ** 3
    return [[(1 if i == j else 0) + a * S[i][j] + b * S2[i][j] for j in range(3)] for i in range(3)]


def rotvel_inverse(g, rep):
    """A(gamma)^-1 in closed form (rotvelxform(gamma, inverse=True)); exp: I - [v]x / 2 + k2(theta) [v]x^2"""
    g = [M.mpf(x) for x in g]
    if rep == "rpy/zyx":
        sb, cb, sg, cg = M.sin(g[1]), M.cos(g[1]), M.sin(g[2]), M.cos(g[2])
        return [[cg / cb, sg / cb, 0], [-sg, cg, 0], [cg * sb / cb, sg * sb / cb, 1]]
    if rep == "rpy/xyz":
        sb, cb, sg, cg = M.sin(g[1]), M.cos(g[1]), M.sin(g[2]), M.cos(g[2])
        return [[0, -sg / cb, cg / cb], [0, cg, sg], [1, sg * sb / cb, -cg * sb / cb]]
    if rep == "eul":
        sp, cp, st, ct = M.sin(g[0]), M.cos(g[0]), M.sin(g[1]), M.cos(g[1])
        return [[-cp * ct / st, -sp * ct / st, 1], [-sp, cp, 0], [cp / st, sp / st, 0]]
    S = _skew(g)
    S2 = mul(S, S)
    c = k2(M.sqrt(M.fsum(x * x for x in g)))
    return [[(1 if i == j else 0) - S[i][j] / 2 + c * S2[i][j] for j in range(3)] for i in range(3)]


def kappa(g, rep):
    """conditioning of A^-1 and of roll / yaw: max(1, 1/|cos pitch|) (rpy), max(1, 1/|sin theta|) (eul), 1 (exp: A^-1
    is bounded for theta <= pi)"""
    if rep == "exp":
        return 1.0
    d = abs(M.sin(g[1])) if rep == "eul" else abs(M.cos(g[1]))
    return float(max(1, 1 / d)) if d > 0 else np.inf


# ------------------------------------------------------------------ the kernels' operations
def jacob0_analytical(T, J, rep, dt=np.float64):
    """Ja = blkdiag(I, A^-1(Gamma(R))) J row by row for T (N,4,4), J (N,6,n) as the kernel received them.  A^-1 is
    evaluated in mpmath once per distinct rotation; its product with J is taken in extended precision (its rounding is
    far below any bar).  Returns (Ja (N,6,n) float64, kappa (N,))."""
    A, kap = rotvel_inverse_rows(T, rep, dt)
    return apply_rows(A, J), kap


def apply_rows(A, J):
    """blkdiag(I, A) J for A (N,3,3) from rotvel_inverse_rows and J (N,6,n)"""
    out = J.astype(np.float64)
    out[:, 3:] = np.einsum("rij,rjc->ric", A, J[:, 3:].astype(np.longdouble)).astype(np.float64)
    return out


def rotvel_inverse_rows(T, rep, dt=np.float64):
    """A^-1(Gamma(R)) (N,3,3, long double) and kappa (N,) of every row of T (N,4,4)"""
    T = np.asarray(T).reshape(-1, 4, 4)
    R = np.ascontiguousarray(T[:, :3, :3])
    keys, inv = np.unique(R.reshape(len(R), -1).view(np.dtype((np.void, R.dtype.itemsize * 9))), return_inverse=True)
    inv = inv.ravel()
    first = np.zeros(len(keys), dtype=np.int64)
    first[inv[::-1]] = np.arange(len(R))[::-1]
    A = np.empty((len(keys), 3, 3), dtype=np.longdouble)
    kap = np.empty(len(keys))
    for u, i in enumerate(first):
        g = r2x(R[i], rep, dt)
        kap[u] = kappa(g, rep)
        if np.isinf(kap[u]):  # exactly on the singularity: A^-1 does not exist
            A[u] = np.nan
            continue
        Ai = rotvel_inverse(g, rep)
        A[u] = [[np.longdouble(M.nstr(x, 25)) for x in row] for row in Ai]
    return A[inv], kap[inv]


def p_servo_rpy(Te, Tep, gain, threshold, dt=np.float64):
    """e = [Re^T (tp - te); tr2rpy(Re^T Rep, 'zyx')], v = gain .* e, arrived = sum |e| < threshold (with the threshold
    in the dtype).  Tep (N,4,4) or one (4,4).  Returns (v (N,6), arrived (N,), sum |e| (N,), kappa (N,))."""
    Te = np.asarray(Te).reshape(-1, 4, 4)
    Tep = np.broadcast_to(np.asarray(Tep).reshape(-1, 4, 4), Te.shape)
    gain = np.broadcast_to(np.asarray(gain, dtype=np.float64), (6,)).astype(_dt(dt)).astype(np.float64)
    thr = M.mpf(float(_dt(dt)(threshold)))
    N = len(Te)
    v, arrived, tot, kap = np.empty((N, 6)), np.empty(N, dtype=bool), np.empty(N), np.empty(N)
    for r in range(N):
        Ret = tp(mpm(Te[r]))
        d = [M.mpf(float(Tep[r, i, 3])) - M.mpf(float(Te[r, i, 3])) for i in range(3)]
        e = [M.fsum(Ret[i][k] * d[k] for k in range(3)) for i in range(3)]
        g = tr2rpy(mul(Ret, mpm(Tep[r])), "zyx", dt)
        e += g
        s = M.fsum(abs(x) for x in e)
        v[r] = [float(M.mpf(gk) * x) for gk, x in zip(gain, e)]
        arrived[r], tot[r], kap[r] = s < thr, float(s), kappa(g, "rpy/zyx")
    return v, arrived, tot, kap


def angle_axis(Te, Tep, gain=1.0, threshold=0.0, dt=np.float64):
    """_angle_axis (ik.cpp:241-286): e = [tp - te; aa(Rep Re^T)], aa from l = vex(R - R^T), ln = |l|: ln < 1e-6 ->
    0 (tr > 0) or pi/2 (diag(R) + 1), else atan2(ln, tr - 1) l / ln.  v = gain .* e, arrived = sum |e| < threshold.
    Returns (v (N,6), arrived (N,), sum |e| (N,), ln (N,))."""
    Te = np.asarray(Te).reshape(-1, 4, 4)
    Tep = np.broadcast_to(np.asarray(Tep).reshape(-1, 4, 4), Te.shape)
    gain = np.broadcast_to(np.asarray(gain, dtype=np.float64), (6,)).astype(_dt(dt)).astype(np.float64)
    thr = M.mpf(float(_dt(dt)(threshold)))
    cut = M.mpf(float(_dt(dt)(1e-6)))
    N = len(Te)
    v, arrived, tot, lns = np.empty((N, 6)), np.empty(N, dtype=bool), np.empty(N), np.empty(N)
    for r in range(N):
        R = mul(mpm(Tep[r]), tp(mpm(Te[r])))
        e = [M.mpf(float(Tep[r, i, 3])) - M.mpf(float(Te[r, i, 3])) for i in range(3)]
        lx, ly, lz = R[2][1] - R[1][2], R[0][2] - R[2][0], R[1][0] - R[0][1]
        ln = M.sqrt(lx * lx + ly * ly + lz * lz)
        tr = R[0][0] + R[1][1] + R[2][2]
        if ln < cut:
            e += [M.mpf(0)] * 3 if tr > 0 else [M.pi / 2 * (R[i][i] + 1) for i in range(3)]
        else:
            ang = M.atan2(ln, tr - 1)
            e += [ang * lx / ln, ang * ly / ln, ang * lz / ln]
        s = M.fsum(abs(x) for x in e)
        v[r] = [float(M.mpf(gk) * x) for gk, x in zip(gain, e)]
        arrived[r], tot[r], lns[r] = s < thr, float(s), float(ln)
    return v, arrived, tot, lns


def r2q(T):
    """host_r2q: the unit quaternion (s, x, y, z) of the rotation part of a 4x4, s >= 0, by the branch on the trace
    and the largest diagonal element, then normalised"""
    R = mpm(T)
    tr = R[0][0] + R[1][1] + R[2][2]
    if tr > 0:
        s = M.sqrt(tr + 1) * 2
        q = [s / 4, (R[2][1] - R[1][2]) / s, (R[0][2] - R[2][0]) / s, (R[1][0] - R[0][1]) / s]
    elif R[0][0] > R[1][1] and R[0][0] > R[2][2]:
        s = M.sqrt(1 + R[0][0] - R[1][1] - R[2][2]) * 2
        q = [(R[2][1] - R[1][2]) / s, s / 4, (R[0][1] + R[1][0]) / s, (R[0][2] + R[2][0]) / s]
    elif R[1][1] > R[2][2]:
        s = M.sqrt(1 + R[1][1] - R[0][0] - R[2][2]) * 2
        q = [(R[0][2] - R[2][0]) / s, (R[0][1] + R[1][0]) / s, s / 4, (R[1][2] + R[2][1]) / s]
    else:
        s = M.sqrt(1 + R[2][2] - R[0][0] - R[1][1]) * 2
        q = [(R[1][0] - R[0][1]) / s, (R[0][2] + R[2][0]) / s, (R[1][2] + R[2][1]) / s, s / 4]
    n = M.sqrt(M.fsum(x * x for x in q)) * (-1 if q[0] < 0 else 1)
    return [x / n for x in q]


def q2r(q):
    w, x, y, z = q
    return [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
            [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
            [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]


def ctraj_dot(T0, T1):
    """q0 . q1 of the two end orientations: its sign picks the shorter arc, and at 0 both arcs are as short"""
    return float(M.fsum(a * b for a, b in zip(r2q(T0), r2q(T1))))


def ctraj(T0, T1, s, other_arc=False):
    """SE3.interp: translation lerp, orientation by slerp along the shorter arc between the quaternions of T0 and T1
    (other_arc: the longer one), s clipped to [0, 1].  T0, T1 (4,4) float64 as the kernel's host receives them, s (N,)
    in the kernel's dtype.  Returns (N,4,4) float64."""
    q0, q1 = r2q(T0), r2q(T1)
    if (M.fsum(a * b for a, b in zip(q0, q1)) < 0) != other_arc:
        q0 = [-x for x in q0]
    th = 2 * M.atan2(M.sqrt(M.fsum((a - b) ** 2 for a, b in zip(q0, q1))), M.sqrt(M.fsum((a + b) ** 2 for a, b in zip(q0, q1))))
    p0 = [M.mpf(float(T0[i, 3])) for i in range(3)]
    p1 = [M.mpf(float(T1[i, 3])) for i in range(3)]
    out = np.zeros((len(s), 4, 4))
    for r, u in enumerate(np.asarray(s)):
        u = min(max(M.mpf(float(u)), 0), 1)
        if th == 0:
            q = q0
        else:
            w0, w1 = M.sin((1 - u) * th) / M.sin(th), M.sin(u * th) / M.sin(th)
            q = [w0 * a + w1 * b for a, b in zip(q0, q1)]
        out[r, :3, :3] = to_np(q2r(q))
        out[r, :3, 3] = [float(a * (1 - u) + u * b) for a, b in zip(p0, p1)]
        out[r, 3, 3] = 1
    return out
