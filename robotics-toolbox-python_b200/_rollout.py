"""Fixed-step rollout front end shared by DHRobot.rollout and Robot.rollout: argument handling and the call into the
device kernel that integrates an ensemble of trajectories with classical RK4 under a per-step torque sequence and,
on request, returns the exact discrete-time sensitivities A_k, B_k (b2k_rne_rollout / b2k_tree_rollout)."""
from collections import namedtuple

import numpy as np

from . import _buffers as B
from . import _lib

Rollout = namedtuple("rollout", "t q qd A B")


def rollout(robot, entry, handle, kernel_gravity, q0, tau, dt, qd0=None, sensitivities=False, gravity=None, dtype=None):
    """`entry(handle, ...)` is the C entry point of the robot class, `kernel_gravity(gravity)` the gravity vector in
    the convention that entry expects.  Semantics: see DHRobot.rollout."""
    n = robot.n
    if not np.isscalar(dt) or not np.isfinite(dt) or not dt > 0:
        raise ValueError(f"dt must be a positive, finite scalar; got {dt!r}")
    B.check_numeric(q0, "q0")
    B.check_numeric(tau, "tau")
    if qd0 is not None:
        B.check_numeric(qd0, "qd0")
    dt_ = B.pick_dtype(q0, dtype)
    host = not B.is_tensor(q0)
    q0d = B.to_device(q0, dt_)
    taud = B.to_device(tau, dt_)
    if q0d.dim() not in (1, 2) or q0d.shape[-1] != n:
        raise ValueError(f"q0 must have shape ({n},) or (N,{n}); got {tuple(q0d.shape)}")
    if taud.dim() not in (2, 3) or taud.shape[-1] != n or taud.shape[-2] < 1:
        raise ValueError(f"tau must have shape (K,{n}) or (N,K,{n}) with K >= 1; got {tuple(taud.shape)}")
    K = int(taud.shape[-2])
    rows = [q0d.reshape(-1, n)]
    if qd0 is not None:
        qd0d = B.to_device(qd0, dt_)
        if qd0d.dim() not in (1, 2) or qd0d.shape[-1] != n:
            raise ValueError(f"qd0 must have shape ({n},) or (N,{n}); got {tuple(qd0d.shape)}")
        rows.append(qd0d.reshape(-1, n))
    # one trajectory without the N axis only when no input has one
    single = q0d.dim() == 1 and taud.dim() == 2 and (qd0 is None or qd0d.dim() == 1)
    N = max([r.shape[0] for r in rows] + ([taud.shape[0]] if taud.dim() == 3 else []))
    if any(r.shape[0] not in (1, N) for r in rows) or (taud.dim() == 3 and taud.shape[0] != N):
        raise ValueError("q0, qd0 and a per-trajectory tau must have the same number of trajectories N")
    rows = [r.expand(N, n).contiguous() for r in rows]
    q0d, qd0d = rows[0], (rows[1] if qd0 is not None else None)
    taud = taud.contiguous()
    stride = 0 if taud.dim() == 2 else K * n
    q = B.empty((N, K + 1, n), dt_, like=q0d)
    qd = B.empty((N, K + 1, n), dt_, like=q0d)
    A = B.empty((N, K, 2 * n, 2 * n), dt_, like=q0d) if sensitivities else None
    Bm = B.empty((N, K, 2 * n, n), dt_, like=q0d) if sensitivities else None
    g = np.ascontiguousarray(kernel_gravity(gravity), dtype=np.float64)
    _lib.check(entry(handle, B.code(dt_), B.ptr(q0d), B.ptr(qd0d), N, K, float(dt), _lib.dptr(g), B.ptr(taud), stride,
                     B.ptr(q), B.ptr(qd), B.ptr(A), B.ptr(Bm), B.stream_ptr(q0d)))
    outs = [q, qd, A, Bm]
    if host:
        outs = [None if x is None else B.to_host(x) for x in outs]
    if single:
        outs = [None if x is None else x[0] for x in outs]
    return Rollout(np.arange(K + 1) * float(dt), *outs)
