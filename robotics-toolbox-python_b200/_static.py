"""Static forces: the reference's DynamicsMixin.gravjac, pay, paycap and friction (robot/Dynamics.py), on the device.

gravjac, pay (given q) and paycap are one b2k_gravjac / b2k_pay / b2k_paycap launch each: a lane walks its row's chain
once and never stores the Jacobian it contracts.  pay given J is one b2k_pay_jacobian launch, friction one b2k_friction
launch.  One configuration gives unbatched shapes; numpy in gives numpy out, a CUDA tensor gives a tensor on its device.
"""
from __future__ import annotations

import numpy as np

from . import _buffers as B
from . import _lib


def _stride(W, N, name="W"):
    """Row stride of a wrench argument: (6,) -> 0 (one wrench for every row), (N,6) -> 6."""
    B.check_numeric(W, name)
    shape = tuple(W.shape) if B.is_tensor(W) else np.shape(W)
    if shape == (6,):
        return 0
    if shape == (N, 6):
        return 6
    raise ValueError(f"{name} must have shape (6,) or ({N},6); got {shape}")


def _device_wrench(W, dt, like):
    return B.to_device(W, dt, device=like.device).reshape(-1).contiguous()


def _rows(ets, q, dtype):
    """-> (q (N, width) on the host or device, dtype, host, single); nothing is copied yet."""
    q2, single = ets._qbatch(q)
    return q2, B.pick_dtype(q2, dtype), not B.is_tensor(q2), single


def _out(x, host, single):
    if host:
        x = B.to_host(x)
    return x[0] if single else x


def check_frame(frame):
    if frame not in (0, 1):
        raise ValueError(f"frame must be 0 (world) or 1 (end effector); got {frame!r}")


def pay(ets, W, q=None, J=None, frame=1, dtype=None):
    """tau = -J^T W (N,n) / (n,); J = jacob0 (frame 0) or jacobe (frame 1) of ``ets``, or the given J."""
    check_frame(frame)
    if (q is None) == (J is None):
        raise ValueError("give exactly one of q and J")
    L = _lib.lib()
    if J is not None:
        B.check_numeric(J, "J")
        shape = tuple(J.shape) if B.is_tensor(J) else np.shape(J)
        if len(shape) not in (2, 3) or shape[-2] != 6 or not 1 <= shape[-1] <= _lib.MAX_JOINTS:
            raise ValueError(f"J must be (6,n) or (N,6,n) with n <= {_lib.MAX_JOINTS}; got {shape}")
        single, n = len(shape) == 2, shape[-1]
        N = 1 if single else shape[0]
        stride = _stride(W, N)
        dt = B.pick_dtype(J, dtype)
        Jd = B.to_device(J, dt).reshape(-1, 6, n).contiguous()
        Wd = _device_wrench(W, dt, Jd)
        tau = B.empty((N, n), dt, like=Jd)
        _lib.check(L.b2k_pay_jacobian(B.code(dt), n, B.ptr(Jd), B.ptr(Wd), stride, N, B.ptr(tau), B.stream_ptr(Jd)))
        return _out(tau, not B.is_tensor(J), single)
    q2, dt, host, single = _rows(ets, q, dtype)
    N = q2.shape[0]
    stride = _stride(W, N)
    qd = B.to_device(q2, dt).contiguous()
    Wd = _device_wrench(W, dt, qd)
    tau = B.empty((N, ets.n), dt, like=qd)
    _lib.check(L.b2k_pay(ets._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], B.ptr(Wd), stride, frame, B.ptr(tau), B.stream_ptr(qd)))
    return _out(tau, host, single)


def gravjac(robot, q, gravity=None, dtype=None):
    ets = robot.ets()
    q2, dt, host, single = _rows(ets, q, dtype)
    qd = B.to_device(q2, dt).contiguous()
    N, n = qd.shape[0], robot.n
    g = robot._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
    g = np.ascontiguousarray(g, dtype=np.float64)
    tau = B.empty((N, n), dt, like=qd)
    J0 = B.empty((N, 6, n), dt, like=qd)
    _lib.check(_lib.lib().b2k_gravjac(ets._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(robot._static_mass_table()),
                                      _lib.dptr(g), B.ptr(tau), B.ptr(J0), B.stream_ptr(qd)))
    return _out(tau, host, single), _out(J0, host, single)


def paycap(robot, w, tauR, frame=1, q=None, gravity=None, dtype=None):
    check_frame(frame)
    n = robot.n
    tauR = np.ascontiguousarray(np.asarray(tauR, dtype=np.float64))
    if tauR.shape != (n, 2):
        raise ValueError(f"tauR must have shape ({n},2) (column 0 the largest torque, column 1 the smallest); got {tauR.shape}")
    if q is None:
        raise ValueError("paycap needs q")
    B.check_numeric(w, "w")
    if not B.is_tensor(w):
        w = np.asarray(w, dtype=np.float64)
    ets = robot.ets()
    q2, dt, host, single = _rows(ets, q, dtype)
    N = q2.shape[0]
    stride = _stride(w, N, "w")
    if stride == 0 and not bool((w != 0).any()):
        raise ValueError("w is zero: a payload wrench needs a direction")
    qd = B.to_device(q2, dt).contiguous()
    wd = _device_wrench(w, dt, qd)
    g = robot._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
    g = np.ascontiguousarray(g, dtype=np.float64)
    wmax = B.empty((N, n), dt, like=qd)
    joint = B.empty_i32((N,), like=qd)
    _lib.check(_lib.lib().b2k_paycap(ets._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(robot._static_mass_table()),
                                     _lib.dptr(g), B.ptr(wd), stride, frame, _lib.dptr(tauR), B.ptr(wmax), B.ptr(joint),
                                     B.stream_ptr(qd)))
    wmax, joint = _out(wmax, host, single), _out(joint, host, single)
    if single:
        joint = int(joint)
    return wmax, joint


def friction(robot, qd, dtype=None):
    B.check_numeric(qd, "qd")
    n = robot.n
    dt = B.pick_dtype(qd, dtype)
    host = not B.is_tensor(qd)
    shape = tuple(qd.shape) if B.is_tensor(qd) else np.shape(qd)
    if shape != (n,) and (len(shape) != 2 or shape[1] != n):
        raise ValueError(f"qd must have shape ({n},) or (N,{n}); got {shape}")
    params = np.ascontiguousarray([[l.B, l.G, l.Tc[0], l.Tc[1]] for l in robot.links], dtype=np.float64)
    v = B.to_device(qd, dt).reshape(-1, n).contiguous()
    N = v.shape[0]
    tau = B.empty((N, n), dt, like=v)
    _lib.check(_lib.lib().b2k_friction(B.code(dt), n, _lib.dptr(params), B.ptr(v), N, B.ptr(tau), B.stream_ptr(v)))
    return _out(tau, host, len(shape) == 1)
