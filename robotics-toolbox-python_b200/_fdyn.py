"""Forward-dynamics front end shared by DHRobot.fdyn and Robot.fdyn (reference DynamicsMixin.fdyn, Dynamics.py:185-422,
which every robot class inherits through BaseRobot): argument handling, the scipy route for a Python torque callable,
and the call into the device-resident Dormand-Prince ensemble integrator (b2k_rne_fdyn / b2k_tree_fdyn)."""
import warnings

import numpy as np

from . import _buffers as B
from . import _lib

_EPS = np.finfo(float).eps


def fdyn(robot, entry, handle, kernel_gravity, T, q0, Q=None, Q_args=None, qd0=None, solver="RK45", solver_args=None, dt=None,
         gravity=None, max_steps: int = 4096, dtype=None):
    """`entry(handle, ...)` is the C entry point for this robot class, `kernel_gravity(gravity)` the gravity vector in the
    convention that entry expects.  Semantics: see DHRobot.fdyn."""

    from collections import namedtuple

    n = robot.n
    if not np.isscalar(T):
        raise ValueError("T must be a scalar")
    solver_args = dict(solver_args or {})
    B.check_numeric(q0, "q0")
    if callable(Q):
        from scipy import integrate, interpolate

        q0v = np.asarray(B.to_host(q0) if B.is_tensor(q0) else q0, dtype=np.float64).reshape(n)
        qd0v = np.zeros(n) if qd0 is None else np.asarray(qd0, dtype=np.float64).reshape(n)

        def f(t, x):  # Dynamics._fdyn, Dynamics.py:380-422
            q, qd = x[:n], x[n:]
            tau = np.asarray(Q(robot, t, q, qd, **(Q_args or {})), dtype=np.float64)
            if tau.shape != (n,) or not np.all(np.isreal(tau)):
                raise RuntimeError("torque function must return vector with N real elements")
            return np.r_[qd, robot.accel(q, qd, tau, gravity=gravity)]

        integ = integrate.__dict__[solver](f, t0=0.0, y0=np.r_[q0v, qd0v], t_bound=T, **solver_args)
        tl, xl = [0], [np.r_[q0v, qd0v]]
        while integ.status == "running":
            integ.step()
            if integ.status == "failed":
                raise RuntimeError("integration completed with failed status ")
            tl.append(integ.t)
            xl.append(integ.y)
        ta, xa = np.array(tl), np.array(xl)
        if dt is not None:
            tnew = np.arange(0, T, dt)
            xnew = interpolate.interp1d(ta, xa, axis=0)(tnew)
            return namedtuple("fdyn", "t q qd")(tnew, xnew[:, :n], xnew[:, n:])
        return namedtuple("fdyn", "t q qd")(ta, xa[:, :n], xa[:, n:])
    if solver != "RK45":
        raise ValueError("the device-resident integrator implements RK45 (Dormand-Prince); other solvers need a callable Q")
    unknown = set(solver_args) - {"rtol", "atol", "max_step", "first_step"}
    if unknown:
        raise ValueError(f"unsupported solver_args for the device integrator: {sorted(unknown)}")
    rtol, atol = solver_args.get("rtol", 1e-3), solver_args.get("atol", 1e-6)
    if np.ndim(rtol) or np.ndim(atol):
        raise ValueError("the device integrator takes scalar rtol and atol (one tolerance for every state component)")
    rtol, atol = float(rtol), float(atol)
    if rtol < 100 * _EPS:  # scipy's validate_tol
        warnings.warn(f"At least one element of `rtol` is too small. Setting `rtol = np.maximum(rtol, {100 * _EPS})`.", stacklevel=3)
        rtol = 100 * _EPS
    first_step = solver_args.get("first_step")
    if first_step is not None:  # scipy's validate_first_step; None selects the first step automatically
        if first_step <= 0:
            raise ValueError("`first_step` must be positive.")
        if first_step > abs(T):
            raise ValueError("`first_step` exceeds bounds.")
    dt_ = B.pick_dtype(q0, dtype)
    host = not B.is_tensor(q0)
    q0d = B.to_device(q0, dt_)
    single = q0d.dim() == 1
    q0d = q0d.reshape(-1, n).contiguous()
    nb = q0d.shape[0]
    qd0d = None
    if qd0 is not None:
        qd0d = B.to_device(qd0, dt_).reshape(-1, n)
        qd0d = (qd0d.expand(nb, n) if qd0d.shape[0] == 1 else qd0d).contiguous()
        if qd0d.shape[0] != nb:
            raise ValueError("qd0 must have as many rows as q0")
    mode, tau, tau_rows, kp, kd, qs = 0, None, None, None, None, None
    vec = lambda x, nm: np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n,)))  # noqa: E731
    if Q is None:
        pass
    elif isinstance(Q, tuple) and len(Q) == 4 and Q[0] == "pd":
        mode, kp, kd, qs = 3, vec(Q[1], "kp"), vec(Q[2], "kd"), vec(Q[3], "qstar")
    else:
        B.check_numeric(Q, "Q")
        qa = Q if B.is_tensor(Q) else np.asarray(Q, dtype=np.float64)
        if qa.ndim == 1:
            mode, tau = 1, vec(np.asarray(B.to_host(qa) if B.is_tensor(qa) else qa), "Q")
        else:
            mode, tau_rows = 2, B.to_device(qa, dt_).reshape(nb, n).contiguous()
    g = np.ascontiguousarray(kernel_gravity(gravity), dtype=np.float64)
    grid = dt is not None
    M = len(np.arange(0, T, dt)) if grid else int(max_steps)
    t_out = B.empty((nb, M), dt_, like=q0d)
    q_out = B.empty((nb, M, n), dt_, like=q0d)
    qd_out = B.empty((nb, M, n), dt_, like=q0d)
    cnt = B.empty_i32((nb,), like=q0d)
    stat = B.empty_i32((nb,), like=q0d)
    if not grid:
        for x in (t_out, q_out, qd_out):
            x.fill_(float("nan"))
    _lib.check(entry(
        handle, B.code(dt_), B.ptr(q0d), B.ptr(qd0d), nb, float(T), _lib.dptr(g), mode, _lib.dptr(tau), B.ptr(tau_rows),
        _lib.dptr(kp), _lib.dptr(kd), _lib.dptr(qs), rtol, atol,
        float(solver_args.get("max_step", np.inf)), float(first_step or 0.0), float(dt or 0.0), int(grid), M,
        B.ptr(t_out), B.ptr(q_out), B.ptr(qd_out), B.ptr(cnt), B.ptr(stat), B.stream_ptr(q0d)))
    st = B.to_host(stat)
    if (st & 1).any():
        raise RuntimeError("integration completed with failed status ")  # the reference's message for a failed step
    if (st & 2).any():
        raise RuntimeError(f"more than max_steps = {M} accepted steps; pass dt for a uniform grid or raise max_steps")
    if grid and (B.to_host(cnt) != M).any():  # every grid sample must have been written
        raise RuntimeError(f"the integrator filled {B.to_host(cnt).min()} of the {M} samples of the output grid")
    if single:
        k = int(cnt[0])
        t, q, qd = (B.to_host(x[0, :k]) for x in (t_out, q_out, qd_out))
        return namedtuple("fdyn", "t q qd")(t, q, qd)
    if grid:
        t = np.arange(0, T, dt)
        if host:
            return namedtuple("fdyn", "t q qd")(t, B.to_host(q_out), B.to_host(qd_out))
        return namedtuple("fdyn", "t q qd")(t, q_out, qd_out)
    if host:
        t_out, q_out, qd_out, cnt = (B.to_host(x) for x in (t_out, q_out, qd_out, cnt))
    return namedtuple("fdyn", "t q qd count")(t_out, q_out, qd_out, cnt)
