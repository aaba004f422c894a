"""Operational-space dynamics, shared by DHRobot and Robot: the reference's DynamicsMixin.inertia_x, coriolis_x,
gravload_x and accel_x (robot/Dynamics.py, between gravload and itorque).  Per configuration row, with
Ja = jacob0_analytical(q, representation) and Ji = inv(Ja) (pinv=False, n = 6) or pinv(Ja):

    inertia_x   Mx = Ji^T M Ji
    gravload_x  Gx = Ji^T G
    coriolis_x  Cx = Ji^T C Ji - Mx Jad Ji,   Jad = jacob0_dot(q, qd, representation)
    accel_x     qd = Ji xd,  qdd = accel(q, qd, Ja^T w),  xdd = Ja qdd + Jad qd

The producers are the robot's own device methods (jacob0_analytical, jacob0_dot, inertia, coriolis, gravload, accel);
the inverse and the products are one b2k_opspace launch, and accel_x ends with b2k_opspace_xdd.  Every launch is
ordered on the stream of the input's device with no host synchronisation in between.  One configuration (n,) gives
(6,6) / (6,); an (N,n) batch gives (N,6,6) / (N,6); numpy in gives numpy out, a CUDA tensor gives a tensor on its device.
Deviation: inv on a singular Ja raises LinAlgError for one configuration, as numpy does; in a batch the rows whose
elimination met an exactly zero pivot come back as NaN (a kernel cannot raise for one row).
"""
from __future__ import annotations

import numpy as np

from . import _buffers as B
from . import _lib


def _check_inv(robot, pinv, Ji):
    if not pinv and Ji is None and robot.n != 6:
        raise np.linalg.LinAlgError(f"inv needs a square analytical Jacobian; this robot has n = {robot.n} joints (use pinv=True)")


def _prep(robot, q, dtype):
    B.check_numeric(q, "q")
    dt = B.pick_dtype(q, dtype)
    host = not B.is_tensor(q)
    qt = B.to_device(q, dt)
    single = qt.dim() == 1
    qt = qt.reshape(1, -1) if single else qt
    if qt.dim() != 2 or qt.shape[1] != robot.n:
        raise ValueError(f"q must have shape ({robot.n},) or (N,{robot.n}); got {tuple(qt.shape)}")
    return qt.contiguous(), dt, host, single


def _rows(x, name, tail, like, dt):
    """An operand given by the caller, single-row or batched shape -> contiguous (N,)+tail tensor on like's device."""
    B.check_numeric(x, name)
    t = B.to_device(x, dt, device=like.device)
    if t.device != like.device:
        t = t.to(like.device)
    N = like.shape[0]
    if tuple(t.shape) == tuple(tail):
        t = t.reshape((1,) + tuple(tail))
    if tuple(t.shape) != (N,) + tuple(tail):
        raise ValueError(f"{name} must have shape {tuple(tail)} or ({N},) + {tuple(tail)}; got {tuple(t.shape)}")
    return t.contiguous()


_SHAPES = {"Ji": lambda n: (n, 6), "Mx": lambda n: (6, 6), "Cx": lambda n: (6, 6), "Gx": lambda n: (6,), "qd": lambda n: (n,),
           "tau": lambda n: (n,)}


def _launch(n, pinv, like, dt, outs, Ja=None, Ji=None, M=None, C=None, Jd=None, G=None, Mx=None, xd=None, w=None):
    N = like.shape[0]
    res = {k: B.empty((N,) + _SHAPES[k](n), dt, like=like) for k in outs}
    kind = _lib.OPS_PINV if (pinv or Ji is not None) else _lib.OPS_INV
    p = B.ptr
    _lib.check(_lib.lib().b2k_opspace(B.code(dt), n, kind, p(Ja), p(Ji), p(M), p(C), p(Jd), p(G), p(Mx), p(xd), p(w), N,
                                      p(res.get("Ji")), p(res.get("Mx")), p(res.get("Cx")), p(res.get("Gx")), p(res.get("qd")),
                                      p(res.get("tau")), B.stream_ptr(like)))
    return res


def _finish(x, host, single, inverted):
    if single and inverted and np.isnan(B.to_host(x)).any():
        raise np.linalg.LinAlgError("Singular matrix")
    if host:
        x = B.to_host(x)
    return x[0] if single else x


def _ja(robot, qt, representation, dt):
    return robot.jacob0_analytical(qt, representation=representation, dtype=dt).reshape(-1, 6, robot.n).contiguous()


def inertia_x(robot, q, pinv=False, representation="rpy/xyz", Ji=None, dtype=None):
    _check_inv(robot, pinv, Ji)
    qt, dt, host, single = _prep(robot, q, dtype)
    n = robot.n
    Jit = None if Ji is None else _rows(Ji, "Ji", (n, 6), qt, dt)
    Ja = _ja(robot, qt, representation, dt) if Jit is None else None
    M = robot.inertia(qt, dtype=dt)
    out = _launch(n, pinv, qt, dt, ("Mx",), Ja=Ja, Ji=Jit, M=M)["Mx"]
    return _finish(out, host, single, not pinv and Jit is None)


def gravload_x(robot, q, gravity=None, pinv=False, representation="rpy/xyz", Ji=None, dtype=None):
    _check_inv(robot, pinv, Ji)
    qt, dt, host, single = _prep(robot, q, dtype)
    n = robot.n
    Jit = None if Ji is None else _rows(Ji, "Ji", (n, 6), qt, dt)
    Ja = _ja(robot, qt, representation, dt) if Jit is None else None
    G = robot.gravload(qt, gravity=gravity, dtype=dt)
    out = _launch(n, pinv, qt, dt, ("Gx",), Ja=Ja, Ji=Jit, G=G)["Gx"]
    return _finish(out, host, single, not pinv and Jit is None)


def coriolis_x(robot, q, qd, pinv=False, representation="rpy/xyz", J=None, Ji=None, Jd=None, C=None, Mx=None, dtype=None):
    _check_inv(robot, pinv, Ji)
    qt, dt, host, single = _prep(robot, q, dtype)
    n = robot.n
    qdt = _rows(qd, "qd", (n,), qt, dt)
    Jit = None if Ji is None else _rows(Ji, "Ji", (n, 6), qt, dt)
    Ja = None
    if Jit is None:
        Ja = _ja(robot, qt, representation, dt) if J is None else _rows(J, "J", (6, n), qt, dt)
    Jdt = (robot.jacob0_dot(qt, qdt, representation=representation, dtype=dt).reshape(-1, 6, n).contiguous() if Jd is None
           else _rows(Jd, "Jd", (6, n), qt, dt))
    Ct = robot.coriolis(qt, qdt, dtype=dt) if C is None else _rows(C, "C", (n, n), qt, dt)
    Mxt = None if Mx is None else _rows(Mx, "Mx", (6, 6), qt, dt)
    M = robot.inertia(qt, dtype=dt) if Mxt is None else None
    out = _launch(n, pinv, qt, dt, ("Cx",), Ja=Ja, Ji=Jit, M=M, C=Ct, Jd=Jdt, Mx=Mxt)["Cx"]
    return _finish(out, host, single, not pinv and Jit is None)


def accel_x(robot, q, xd, wrench, gravity=None, pinv=False, representation="rpy/xyz", dtype=None):
    _check_inv(robot, pinv, None)
    qt, dt, host, single = _prep(robot, q, dtype)
    n = robot.n
    xdt = _rows(xd, "xd", (6,), qt, dt)
    wt = _rows(wrench, "wrench", (6,), qt, dt)
    Ja = _ja(robot, qt, representation, dt)
    r = _launch(n, pinv, qt, dt, ("qd", "tau"), Ja=Ja, xd=xdt, w=wt)
    qd = r["qd"]
    Jd = robot.jacob0_dot(qt, qd, representation=representation, dtype=dt).reshape(-1, 6, n).contiguous()
    qdd = robot.accel(qt, qd, r["tau"], gravity=gravity, dtype=dt)
    N = qt.shape[0]
    xdd = B.empty((N, 6), dt, like=qt)
    _lib.check(_lib.lib().b2k_opspace_xdd(B.code(dt), n, B.ptr(Ja), B.ptr(qdd), B.ptr(Jd), B.ptr(qd), N, B.ptr(xdd),
                                          B.stream_ptr(qt)))
    return _finish(xdd, host, single, not pinv)
