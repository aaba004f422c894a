"""Float64 restatement of planar kinematics (ETS2.eval / jacob0 / jacobe), vectorised over rows.

eval    : base . A_0(q) . A_1(q) ... A_{m-1}(q) . tool, left to right, 3x3 products per row.
jacob0  : the reference's construction: for joint i, dT/dq_i = E_0 . S_i . A_i(q) . E_f (E_0 the product in front of
          the joint, E_f the product behind it with the tool, S_i the generator of the joint's axis, times -1 for a
          flipped joint), read as (dT[:2, 2], (dT[:2, :2] R^T)[1, 0]); no base.
jacobe  : blkdiag(R^T, 1) . jacob0, R the rotation of the pose (tool in, base out).
"""
import numpy as np

_S = {
    "R": np.array([[0.0, -1, 0], [1, 0, 0], [0, 0, 0]]),
    "tx": np.array([[0.0, 0, 1], [0, 0, 0], [0, 0, 0]]),
    "ty": np.array([[0.0, 0, 0], [0, 0, 1], [0, 0, 0]]),
}


def _se2(c, s, x, y):
    N = (np.broadcast(c, s, x, y).shape or (1,))[0]
    A = np.zeros((N, 3, 3))
    A[:, 0, 0] = c
    A[:, 0, 1] = -np.asarray(s)
    A[:, 1, 0] = s
    A[:, 1, 1] = c
    A[:, 0, 2] = x
    A[:, 1, 2] = y
    A[:, 2, 2] = 1.0
    return A


def elem(et, q):
    """(N,3,3) of one ET2 over the rows of q (N, w)"""
    N = q.shape[0]
    if not et.isjoint:
        return np.broadcast_to(et.A(), (N, 3, 3))
    v = q[:, et.jindex] * (-1.0 if et.isflip else 1.0)
    z, o = np.zeros(N), np.ones(N)
    if et.axis == "R":
        return _se2(np.cos(v), np.sin(v), z, z)
    if et.axis == "tx":
        return _se2(o, z, v, z)
    return _se2(o, z, z, v)


def _q2(q):
    return np.atleast_2d(np.asarray(q, dtype=np.float64))


def eval_(ets, q, base=None, tool=None):
    q = _q2(q)
    T = np.broadcast_to(np.eye(3) if base is None else np.asarray(base, float), (q.shape[0], 3, 3))
    for et in ets:
        T = T @ elem(et, q)
    if tool is not None:
        T = T @ np.asarray(tool, float)
    return T


def jacob0(ets, q, tool=None):
    q = _q2(q)
    N = q.shape[0]
    ets = list(ets)
    A = [elem(et, q) for et in ets]
    pre = [np.broadcast_to(np.eye(3), (N, 3, 3))]
    for a in A:
        pre.append(pre[-1] @ a)
    post = [np.broadcast_to(np.eye(3) if tool is None else np.asarray(tool, float), (N, 3, 3))]
    for a in reversed(A):
        post.append(a @ post[-1])
    post = post[::-1]  # post[k] = A_k ... A_{m-1} tool
    R = pre[-1] @ post[-1]
    R = R[:, :2, :2]
    cols = []
    for k, et in enumerate(ets):
        if not et.isjoint:
            continue
        sg = -1.0 if et.isflip else 1.0
        dT = sg * (pre[k] @ _S[et.axis] @ A[k] @ post[k + 1])
        w = (dT[:, :2, :2] @ np.transpose(R, (0, 2, 1)))[:, 1, 0]
        cols.append(np.stack([dT[:, 0, 2], dT[:, 1, 2], w], axis=1))
    return np.stack(cols, axis=2)


def jacobe(ets, q, tool=None):
    q = _q2(q)
    R = eval_(ets, q, tool=tool)[:, :2, :2]
    J = jacob0(ets, q, tool)
    out = J.copy()
    out[:, :2] = np.transpose(R, (0, 2, 1)) @ J[:, :2]
    return out


def random_chain(rng, n, wide=0):
    """A random ETS2 of n joints: every joint kind (R, tx, ty) once n >= 3, flips, 0..2 constants (R(eta), tx, ty,
    SE2) in front of each joint and behind the last, and jindices a permutation of n of the n + wide columns."""
    import b2kin as rtb

    E = rtb.ET2
    kinds = (["R", "tx", "ty"] * n)[:n]
    rng.shuffle(kinds)
    cols = rng.permutation(n + wide)[:n]

    def const():
        k = rng.integers(4)
        if k == 0:
            return E.R(float(rng.uniform(-3, 3)))
        if k == 1:
            return E.tx(float(rng.uniform(-1, 1)))
        if k == 2:
            return E.ty(float(rng.uniform(-1, 1)))
        th = rng.uniform(-3, 3)
        return E.SE2(_se2(np.cos(th), np.sin(th), rng.uniform(-1, 1), rng.uniform(-1, 1))[0])

    ets = []
    for j in range(n):
        ets += [const() for _ in range(rng.integers(3))]
        ets.append(getattr(E, kinds[j])(flip=bool(rng.integers(2)), jindex=int(cols[j])))
    ets += [const() for _ in range(rng.integers(3))]
    return rtb.ETS2(ets)


def random_pose(rng):
    th = rng.uniform(-3, 3)
    return _se2(np.cos(th), np.sin(th), rng.uniform(-1, 1), rng.uniform(-1, 1))[0]
