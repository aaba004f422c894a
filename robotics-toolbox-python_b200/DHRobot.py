"""DH / MDH serial-link robots: kinematics through the compiled ETS chain, inverse dynamics
through the batched RNE kernel.

Mirrors the hot-path part of the reference's ``DHRobot`` (reference
src/roboticstoolbox/robot/DHRobot.py): ``ets()`` 878-918, ``fkine`` 920-979, ``jacobe`` 1066-1140,
``jacob0`` 1142-1198, ``rne`` 1373-1456 with its parameter packing ``_init_rne`` 1340-1361 and
dirty tracking (DHLink.py:24-51), ``ikine_LM`` 2454-2474, and the closed-form ``ikine_6s`` as ``ikine_a``.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np

from . import _buffers as B
from . import _lib
from . import _opspace
from . import _static
from ._se3 import SE3
from .DHLink import DHLink
from .ET import ET
from .ETS import ETS, _mat44
from .IK import IKSolution


class DHRobot:
    def __init__(self, links: List[DHLink], name: str = "", manufacturer: str = "", base=None, tool=None,
                 gravity=None, **kwargs):
        self._rne_ob = None
        if not links or not all(isinstance(l, DHLink) for l in links):
            raise TypeError("links must be a non-empty list of DHLink")
        mdh = {l.mdh for l in links}
        if len(mdh) != 1:
            raise ValueError("Robot has mixed D&H links conventions")
        self.links = list(links)
        for l in self.links:
            l._robot = self
        self.name, self.manufacturer = name, manufacturer
        self._base = np.eye(4) if base is None else _mat44(base, "base")
        self._tool = np.eye(4) if tool is None else _mat44(tool, "tool")
        # reference BaseRobot.py:83 default
        self._gravity = np.array([0.0, 0.0, -9.81]) if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        self._rne_ob = None
        self._dynchanged = False
        self._ets_cache = None
        self._prefix_cache = None
        self._static_mass = None
        self._configs = {}

    # ---- structure
    @property
    def n(self) -> int:
        return len(self.links)

    @property
    def mdh(self) -> int:
        return int(self.links[0].mdh)

    @property
    def base(self) -> SE3:
        return SE3(self._base)

    @base.setter
    def base(self, T):
        self._base = np.eye(4) if T is None else _mat44(T, "base")
        self._ets_cache = None
        self._prefix_cache = None

    @property
    def tool(self) -> SE3:
        return SE3(self._tool)

    @tool.setter
    def tool(self, T):
        self._tool = np.eye(4) if T is None else _mat44(T, "tool")
        self._ets_cache = None
        self._prefix_cache = None

    @property
    def gravity(self) -> np.ndarray:
        return self._gravity

    @gravity.setter
    def gravity(self, g):
        self._gravity = np.asarray(g, dtype=np.float64).reshape(3)
        self.dynchanged()

    @property
    def qlim(self) -> np.ndarray:
        out = np.zeros((2, self.n))
        for j, l in enumerate(self.links):
            if l.qlim is None:
                out[:, j] = (-np.pi, np.pi) if l.isrevolute else (0.0, 1.0)
            else:
                out[:, j] = l.qlim
        return out

    def addconfiguration(self, name, q):
        self._configs[name] = np.asarray(q, dtype=np.float64)
        setattr(self, name, self._configs[name])

    def __len__(self):
        return self.n

    def __iter__(self):
        return iter(self.links)

    # ---- kinematics: reference DHRobot.ets (878-918) then the ETS hot path
    def ets(self) -> ETS:
        if self._ets_cache is None:
            parts = []
            if not np.array_equal(self._base, np.eye(4)):
                parts.append(ETS(ET.SE3(self._base)))
            parts.extend(l.ets for l in self.links)
            if not np.array_equal(self._tool, np.eye(4)):
                parts.append(ETS(ET.SE3(self._tool)))
            self._ets_cache = ETS.from_links(parts)
        return self._ets_cache

    def fkine(self, q, **kwargs) -> SE3:
        """Base and tool incorporated, joint offsets applied (reference DHRobot.fkine 920-979)."""
        return self.ets().fkine(q, **kwargs)

    def eval(self, q, **kwargs):
        return self.ets().eval(q, **kwargs)

    def fkine_all(self, q, old=True, dtype=None):
        """Link frame poses {0} .. {n}: base, base A1, base A1 A2, ... (reference DHRobot.fkine_all, DHRobot.py:1018-1064;
        the tool does not enter, joint offsets do).  (n+1,4,4) for one q, (N,n+1,4,4) for a batch."""
        if self._prefix_cache is None:
            self._prefix_cache = [ETS.from_links([l.ets for l in self.links[:k + 1]]) for k in range(self.n)]
        base = None if np.array_equal(self._base, np.eye(4)) else self._base
        return ETS.eval_frames(self._prefix_cache, q, base=base, dtype=dtype)

    def jacobe(self, q, **kwargs):
        """Jacobian in the end-effector frame (reference DHRobot.jacobe 1066-1140)."""
        return self.ets().jacobe(q, **kwargs)

    def jacob0(self, q, **kwargs):
        """Jacobian in the world frame = tr2jac(T) @ jacobe, base rotation included
        (reference DHRobot.jacob0 1142-1198)."""
        return self.ets().jacob0(q, **kwargs)

    def fkine_jacob0(self, q, **kwargs):
        return self.ets().fkine_jacob0(q, **kwargs)

    # pure functions of the Jacobian (reference DHRobot.py: hessian0 1142-1198 region, manipulability / jacobm /
    # jacob0_dot exercised by tests/test_DHRobot.py:1246-1283), evaluated on the chain's own ETS
    def hessian0(self, q=None, J0=None, **kwargs):
        return self.ets().hessian0(q, J0=J0, **kwargs)

    def hessiane(self, q=None, Je=None, **kwargs):
        return self.ets().hessiane(q, Je=Je, **kwargs)

    def manipulability(self, q=None, J=None, method="yoshikawa", axes="all", **kwargs):
        return self.ets().manipulability(q, J=J, method=method, axes=axes, **kwargs)

    def jacobm(self, q=None, J=None, H=None, axes="all", **kwargs):
        return self.ets().jacobm(q, J=J, H=H, axes=axes, **kwargs)

    def jacob0_dot(self, q=None, qd=None, J0=None, representation=None, **kwargs):
        return self.ets().jacob0_dot(q, qd, J0=J0, representation=representation, **kwargs)

    def jacob0_analytical(self, q, representation="rpy/xyz", **kwargs):
        """reference DHRobot.jacob0_analytical (DHRobot.py:1200-1262) -> rotvelxform(R, inverse=True) @ jacob0"""
        return self.ets().jacob0_analytical(q, representation=representation, **kwargs)

    def ikine_LM(self, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, joint_limits=False, mask=None, seed=None,
                 **kwargs):
        """reference DHRobot.ikine_LM 2454-2474 (note joint_limits defaults to False here)."""
        return self.ets().ikine_LM(Tep=Tep, q0=q0, ilimit=ilimit, slimit=slimit, tol=tol,
                                   joint_limits=joint_limits, mask=mask, seed=seed, **kwargs)

    def ik_LM(self, Tep, **kwargs):
        return self.ets().ik_LM(Tep, **kwargs)

    def jtraj(self, T1, T2, t, device=None, **kwargs):
        """Joint-space trajectory between two end-effector poses (reference Robot.jtraj, Robot.py:917-961): both poses go
        through ``ikine_LM`` (``kwargs`` to the solver), the quintic ``jtraj`` joins the solutions; ``device=True`` leaves
        the (N,n) samples in HBM for ``rne`` / ``eval``."""
        from .trajectory import jtraj as _jtraj

        q1, q2 = self.ikine_LM(T1, **kwargs), self.ikine_LM(T2, **kwargs)
        return _jtraj(q1.q, q2.q, t, device=device)

    # ---- closed-form inverse kinematics (reference DHRobot.ikine_6s, which Puma560.ikine_a calls): csrc/b2k_ik6s.cu
    _IKINE_A_LETTERS = ("lr", "ud", "nf")

    @staticmethod
    def config_validate(config: str, allowables) -> str:
        """The reference's configuration-string rules: one letter of each pair in ``allowables`` (for example
        ("lr", "ud", "nf")), the first of a pair where the string has neither; both letters of a pair, or a letter of no
        pair, raise ValueError.  Returns the letters in the order of ``allowables``."""
        if not isinstance(config, str):
            raise TypeError("config must be a string")
        known = "".join(allowables)
        for ch in config:
            if ch not in known:
                raise ValueError(f"bad config specifier {ch!r}: the letters are {', '.join(allowables)}")
        out = ""
        for pair in allowables:
            given = set(pair) & set(config)
            if len(given) > 1:
                raise ValueError(f"config {config!r} gives more than one of {pair!r}")
            out += given.pop() if given else pair[0]
        return out

    def _ikine_a_table(self) -> np.ndarray:
        """(6,4) rows of (d, a, alpha, offset) for b2k_ikine_6s, after the checks its table cannot express"""
        if self.n != 6:
            raise ValueError(f"ikine_a: the closed form serves 6-joint arms; this robot has {self.n} joints")
        if self.mdh:
            raise ValueError("ikine_a: the closed form serves standard DH; this robot uses modified DH")
        for j, l in enumerate(self.links):
            if not l.isrevolute:
                raise ValueError(f"ikine_a: joint {j + 1} is prismatic; the closed form needs revolute joints")
            if l.flip:
                raise ValueError(f"ikine_a: joint {j + 1} is flipped; the closed form needs unflipped joints")
        return np.ascontiguousarray([[l.d, l.a, l.alpha, l.offset] for l in self.links], dtype=np.float64)

    def ikine_a(self, T, config="lun", dtype=None) -> IKSolution:
        """Analytic inverse kinematics of a Puma-type 6R arm (reference DHRobot.ikine_6s / Puma560.ikine_a): the exact
        joint solution for a shoulder (l / r), elbow (u / d) and wrist (n / f) configuration, with no iteration.

        The robot must be a standard-DH, all-revolute 6-joint arm with alpha = (pi/2, 0, -pi/2, +-pi/2, -+pi/2, any),
        a1 = a4 = a5 = 0, d5 = 0 and a2 != 0; any other robot raises ValueError naming what breaks the pattern.
        ``T`` is an SE3, a (4,4) or (N,4,4) array, or a CUDA tensor; ``config`` a string ("lun" default, missing letters
        filled by :meth:`config_validate`) or a sequence of up to 8 strings, all solved from one read of T in one launch.
        One pose gives ``IKSolution(q (6,), success, reason="Success" | "Out of reach")``; a batch q (N,6) with NaN
        rows where the pose is out of reach, success = every row reachable.  A sequence of configurations makes q
        (k,6) / (N,k,6).  numpy in gives numpy out, a CUDA tensor gives q on its device.  Joint limits are not applied."""
        configs = [config] if isinstance(config, str) else list(config)
        if not 1 <= len(configs) <= 8:
            raise ValueError(f"ikine_a: give 1 to 8 configurations, got {len(configs)}")
        codes = []
        for c in configs:
            v = self.config_validate(c, self._IKINE_A_LETTERS)
            codes.append(int(v[0] == "r") | int(v[1] == "d") << 1 | int(v[2] == "f") << 2)
        conf = np.array(codes, dtype=np.int32)
        dh = self._ikine_a_table()
        base = None if np.array_equal(self._base, np.eye(4)) else np.ascontiguousarray(self._base)
        tool = None if np.array_equal(self._tool, np.eye(4)) else np.ascontiguousarray(self._tool)
        L = _lib.lib()
        cp = conf.ctypes.data_as(_lib.ip)
        # the link pattern is checked by the C entry point; N = 0 validates without touching a device
        _lib.check(L.b2k_ikine_6s(_lib.F64, _lib.dptr(dh), _lib.dptr(base), _lib.dptr(tool), None, 0, len(conf), cp, None,
                                  None, None))
        T = getattr(T, "A", T)
        B.check_numeric(T, "T")
        if not B.is_tensor(T):
            T = np.asarray(T)
        if T.ndim not in (2, 3) or tuple(T.shape[-2:]) != (4, 4):
            raise ValueError(f"T must be (4,4) or (N,4,4); got {tuple(T.shape)}")
        single = T.ndim == 2
        dt = B.pick_dtype(T, dtype)
        Td = B.to_device(T, dt).reshape(-1, 4, 4).contiguous()
        N, k = Td.shape[0], len(conf)
        q = B.empty((N, k, 6), dt, like=Td)
        ok = B.empty_i32((N, k), like=Td)
        _lib.check(L.b2k_ikine_6s(B.code(dt), _lib.dptr(dh), _lib.dptr(base), _lib.dptr(tool), B.ptr(Td), N, k, cp, B.ptr(q),
                                  B.ptr(ok), B.stream_ptr(Td)))
        reached = B.to_host(ok).astype(bool)
        if not B.is_tensor(T):
            q = B.to_host(q)
        if isinstance(config, str):
            q, reached = q[:, 0], reached[:, 0]
        if single:
            q, reached = q[0], reached[0]
        missed = int(reached.size - reached.sum())
        if single and reached.ndim == 0:
            reason = "Success" if missed == 0 else "Out of reach"
        elif missed == 0:
            reason = "Success"
        else:
            what = "rows" if isinstance(config, str) else "solutions"
            reason = f"Out of reach: {missed} of {reached.size} {what}"
        return IKSolution(q=q, success=missed == 0, reason=reason)

    def ik_NR(self, Tep, **kwargs):
        return self.ets().ik_NR(Tep, **kwargs)

    def ik_GN(self, Tep, **kwargs):
        return self.ets().ik_GN(Tep, **kwargs)

    # reference DHRobot.py:1923-2452: positional wrappers over the C++ solvers.  (In the reference they
    # forward to ETS methods of the same lower-case names, which ETS does not define; here they work.)
    def ik_lm_chan(self, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, reject_jl=True, we=None, λ=1.0):
        return self.ets().ik_LM(Tep, q0, ilimit, slimit, tol, we, reject_jl, λ, "chan")

    def ik_lm_wampler(self, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, reject_jl=True, we=None, λ=1.0):
        return self.ets().ik_LM(Tep, q0, ilimit, slimit, tol, we, reject_jl, λ, "wampler")

    def ik_lm_sugihara(self, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, reject_jl=True, we=None, λ=1.0):
        return self.ets().ik_LM(Tep, q0, ilimit, slimit, tol, we, reject_jl, λ, "sugihara")

    def ik_nr(self, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, reject_jl=True, we=None, use_pinv=True,
              pinv_damping=0.0):
        return self.ets().ik_NR(Tep, q0, ilimit, slimit, tol, we, reject_jl, use_pinv, pinv_damping)

    def ik_gn(self, Tep, q0=None, ilimit=30, slimit=100, tol=1e-6, reject_jl=True, we=None, use_pinv=True,
              pinv_damping=0.0):
        return self.ets().ik_GN(Tep, q0, ilimit, slimit, tol, we, reject_jl, use_pinv, pinv_damping)

    # ---- inverse dynamics
    def _kinchanged(self):
        """A link's DH parameter changed: the cached ETS (and with it the compiled chain handle) and the
        packed RNE table are both stale (reference DHLink.py:448-563 @_listen_dyn on theta/d/a/alpha/sigma/mdh)."""
        self._ets_cache = None
        self._prefix_cache = None
        self._static_mass = None
        self._dynchanged = True

    def dynchanged(self, what=None):
        """Mark the packed dynamic parameters stale (reference BaseRobot.py:383-398)."""
        self._dynchanged = True
        self._static_mass = None

    def _pack_rne(self) -> np.ndarray:
        """24 doubles per link (reference DHRobot._init_rne 1340-1358)."""
        L = np.zeros(24 * self.n)
        for i, l in enumerate(self.links):
            j = 24 * i
            L[j:j + 6] = (l.alpha, l.a, l.theta, l.d, l.sigma, l.offset)
            L[j + 6] = l.m
            L[j + 7:j + 10] = l.r
            L[j + 10:j + 19] = l.I.flatten()
            L[j + 19:j + 22] = (l.Jm, l.G, l.B)
            L[j + 22:j + 24] = l.Tc
        return L

    def _init_rne(self):
        h = _lib.vp()
        L = self._pack_rne()
        _lib.check(_lib.lib().b2k_rne_create(self.n, self.mdh, _lib.dptr(L), C.byref(h)))
        self._rne_ob = h
        self._dynchanged = False

    def delete_rne(self):
        """reference DHRobot.delete_rne 1363-1371"""
        if self._rne_ob is not None:
            try:
                _lib.lib().b2k_rne_destroy(self._rne_ob)
            except Exception:
                pass
            self._dynchanged = False
            self._rne_ob = None

    def __del__(self):
        self.delete_rne()

    def rne(self, q, qd=None, qdd=None, gravity=None, fext=None, base_wrench=False, dtype=None):
        """Inverse dynamics tau = RNE(q, qd, qdd): (n,) for one state, (N,n) for a trajectory
        (reference DHRobot.rne 1373-1456 -> frne.frne per row).

        ``base_wrench=True`` returns ``(tau, wbase)``: tau as above and wbase (6,) / (N,6) = [fx, fy, fz, mx, my, mz],
        the wrench the base exerts on link 1, expressed in frame 0 (the chain's base frame, after ``robot.base``) with
        the moment about its origin.  Both come from the same recursion (one kernel launch)."""
        if self._rne_ob is None or self._dynchanged:  # @_check_rne, DHLink.py:24-51
            self.delete_rne()
            self._init_rne()
        n = self.n
        for x, nm in ((q, "q"), (qd, "qd"), (qdd, "qdd")):
            if x is None:
                raise ValueError(f"{nm} must be given")
            B.check_numeric(x, nm)
        dt = B.pick_dtype(q, dtype)
        host = not B.is_tensor(q)

        def norm(x):
            if B.is_tensor(x):
                return x.reshape(1, -1) if x.dim() == 1 else x
            a = np.asarray(x, dtype=dt if np.asarray(x).dtype in (np.float32, np.float64) else np.float64)
            return a.reshape(1, -1) if a.ndim == 1 else a

        single = (q.dim() if B.is_tensor(q) else np.ndim(q)) == 1
        q2, qd2, qdd2 = norm(q), norm(qd), norm(qdd)
        N = q2.shape[0]
        for x, nm in ((q2, "q"), (qd2, "qd"), (qdd2, "qdd")):
            if x.ndim != 2 or tuple(x.shape) != (N, n):
                raise ValueError(f"{nm} must have shape ({n},) or (N,{n}); got {tuple(x.shape)}")
        g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        # the recursion has no base: rotate gravity instead (reference 1431-1433), and hand it over negated (1449)
        g = self._base[:3, :3].T @ g
        ng = np.ascontiguousarray(-g)
        fx = None if fext is None else np.ascontiguousarray(np.asarray(fext, dtype=np.float64).reshape(6))
        L = _lib.lib()
        if host:
            t = B.require_cuda()
            qh, qdh, qddh = (np.ascontiguousarray(x, dtype=dt) for x in (q2, qd2, qdd2))
            tau = _lib.host_result((N, n), dt)
            if base_wrench:
                wb = _lib.host_result((N, 6), dt)
                _lib.check(L.b2k_rne_wrench_host(self._rne_ob, B.code(dt), qh.ctypes.data, qdh.ctypes.data, qddh.ctypes.data, N,
                                                 _lib.dptr(ng), _lib.dptr(fx), tau.ctypes.data, wb.ctypes.data,
                                                 t.cuda.current_device()))
            else:
                _lib.check(L.b2k_rne_host(self._rne_ob, B.code(dt), qh.ctypes.data, qdh.ctypes.data, qddh.ctypes.data, N,
                                          _lib.dptr(ng), _lib.dptr(fx), tau.ctypes.data, t.cuda.current_device()))
        else:
            qt, qdt, qddt = (B.to_device(x, dt) for x in (q2, qd2, qdd2))
            tau = B.empty((N, n), dt, like=qt)
            if base_wrench:
                wb = B.empty((N, 6), dt, like=qt)
                _lib.check(L.b2k_rne_wrench(self._rne_ob, B.code(dt), B.ptr(qt), B.ptr(qdt), B.ptr(qddt), N, _lib.dptr(ng),
                                            _lib.dptr(fx), B.ptr(tau), B.ptr(wb), B.stream_ptr(qt)))
            else:
                _lib.check(L.b2k_rne(self._rne_ob, B.code(dt), B.ptr(qt), B.ptr(qdt), B.ptr(qddt), N, _lib.dptr(ng),
                                     _lib.dptr(fx), B.ptr(tau), B.stream_ptr(qt)))
        if base_wrench:
            return (tau[0], wb[0]) if single else (tau, wb)
        return tau[0] if single else tau

    def nofriction(self, coulomb: bool = True, viscous: bool = False) -> "DHRobot":
        """A copy of the robot without Coulomb (default) and / or viscous joint friction (reference
        DynamicsMixin.nofriction, Dynamics.py:139-183; Link.nofriction, Link.py:1548-1590) -- the usual preparation for
        fdyn, whose adaptive integrators chatter on the Coulomb discontinuity at qd = 0."""
        import copy

        links = []
        for l in self.links:
            c = copy.copy(l)
            c._robot = None
            c.ets = l.ets
            if coulomb:
                c._Tc = np.zeros(2)
            if viscous:
                c._B = 0.0
            links.append(c)
        nf = DHRobot(links, name="NF/" + self.name, manufacturer=self.manufacturer, base=self._base, tool=self._tool, gravity=self._gravity)
        for k, v in self._configs.items():
            nf.addconfiguration(k, v)
        return nf

    def fdyn(self, T, q0, Q=None, Q_args=None, qd0=None, solver="RK45", solver_args=None, dt=None, progress=False, gravity=None,
             max_steps: int = 4096, dtype=None):
        """Integrate the forward dynamics over [0, T] (reference DynamicsMixin.fdyn, Dynamics.py:185-422).

        ``q0`` (n,) gives the reference's call: one trajectory, returned as the named tuple (t, q, qd) on the solver's
        own time steps, or on ``np.arange(0, T, dt)`` by linear interpolation when ``dt`` is given.  ``q0`` (B,n) (numpy
        or CUDA tensor) integrates an ENSEMBLE of B initial states at once, one lane per trajectory with its own adaptive
        step size: with ``dt`` q / qd are (B,M,n); without, t is (B,max_steps) and q / qd (B,max_steps,n), padded with NaN
        past ``count`` accepted steps per trajectory.

        ``Q`` selects the joint torque: ``None`` (zero torque, the reference's default); an (n,) or (B,n) array = constant
        torque; ``("pd", kp, kd, qstar)`` = the joint-space law kp (qstar - q) - kd qd; these run in the device-resident
        Dormand-Prince integrator (solver "RK45" with scipy's step control: ``solver_args`` rtol, atol, max_step,
        first_step).  A callable ``Q(robot, t, q, qd, **Q_args)`` -- the reference's signature -- cannot run inside a kernel:
        it is integrated by scipy on the host, as the reference does, with this robot's batched ``accel`` kernel as the
        right-hand side (any scipy solver; one trajectory)."""
        from ._fdyn import fdyn as _fdyn

        if not callable(Q) and (self._rne_ob is None or self._dynchanged):
            self.delete_rne()
            self._init_rne()

        def kernel_gravity(gravity):
            g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
            return -(self._base[:3, :3].T @ g)

        return _fdyn(self, _lib.lib().b2k_rne_fdyn if not callable(Q) else None, self._rne_ob, kernel_gravity, T, q0, Q=Q, Q_args=Q_args,
                     qd0=qd0, solver=solver, solver_args=solver_args, dt=dt, gravity=gravity, max_steps=max_steps, dtype=dtype)

    _RNE_MODES = {"rne": 0, "inertia": 1, "gravload": 2, "itorque": 3, "coriolis": 4, "accel": 5, "rne_wrench": 6}

    def rne_kernel_info(self, op="rne", dtype=np.float64, gravity=None, fext=None) -> str:
        """Which kernel serves `op` for this robot: the robot-specialised one (generated from the link table and
        compiled with NVRTC at first use; the line lists its multiply / FMA / add count per row, registers and
        shared memory) or the pre-compiled generic one, with the reason."""
        if self._rne_ob is None or self._dynchanged:
            self.delete_rne()
            self._init_rne()
        g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        g = np.ascontiguousarray(-(self._base[:3, :3].T @ g))
        buf = C.create_string_buffer(2048)
        _lib.check(_lib.lib().b2k_rne_spec_info(self._rne_ob, self._RNE_MODES[op], B.code(np.dtype(dtype)), _lib.dptr(g),
                                                int(fext is not None and np.any(np.asarray(fext) != 0)), buf, 2048))
        return buf.value.decode()

    # ---- dynamics built on the recursion (reference DynamicsMixin, Dynamics.py; SURVEY 8f-1)
    def _dyn(self, fn_name, ins, out_tail, gravity=None, use_gravity=False, dtype=None):
        """Shared front end of the fan-out kernels: every input (N,n) or (n,), one launch."""
        if self._rne_ob is None or self._dynchanged:
            self.delete_rne()
            self._init_rne()
        n = self.n
        for x in ins:
            B.check_numeric(x)
        dt = B.pick_dtype(ins[0], dtype)
        host = not B.is_tensor(ins[0])
        single = (ins[0].dim() if B.is_tensor(ins[0]) else np.ndim(ins[0])) == 1
        dev = []
        for x in ins:
            t = B.to_device(x, dt)
            t = t.reshape(1, -1) if t.dim() == 1 else t
            dev.append(t.contiguous())
        N = dev[0].shape[0]
        for t in dev:
            if t.dim() != 2 or tuple(t.shape) != (N, n):
                raise ValueError(f"inputs must have shape ({n},) or (N,{n}); got {tuple(t.shape)}")
        out = B.empty((N,) + out_tail, dt, like=dev[0])
        args = [self._rne_ob, B.code(dt)] + [B.ptr(t) for t in dev] + [N]
        if use_gravity:
            g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
            g = np.ascontiguousarray(-(self._base[:3, :3].T @ g))  # as DHRobot.rne: reference 1431-1433, 1449
            args.append(_lib.dptr(g))
        args += [B.ptr(out), B.stream_ptr(dev[0])]
        _lib.check(getattr(_lib.lib(), fn_name)(*args))
        if host:
            out = B.to_host(out)
        return out[0] if single else out

    def inertia(self, q, dtype=None):
        """Joint-space inertia matrix M(q): (n,n) or (N,n,n) (reference Dynamics.inertia, Dynamics.py:704-763)."""
        return self._dyn("b2k_rne_inertia", [q], (self.n, self.n), dtype=dtype)

    def gravload(self, q, gravity=None, dtype=None):
        """Gravity load tau_g(q) (reference Dynamics.gravload, Dynamics.py:863-921)."""
        return self._dyn("b2k_rne_gravload", [q], (self.n,), gravity=gravity, use_gravity=True, dtype=dtype)

    def itorque(self, q, qdd, dtype=None):
        """Inertia torque M(q) qdd (reference Dynamics.itorque, Dynamics.py:1407-1465)."""
        return self._dyn("b2k_rne_itorque", [q, qdd], (self.n,), dtype=dtype)

    def coriolis(self, q, qd, dtype=None):
        """Coriolis / centripetal matrix C(q, qd), friction ignored (reference Dynamics.coriolis, Dynamics.py:765-861)."""
        return self._dyn("b2k_rne_coriolis", [q, qd], (self.n, self.n), dtype=dtype)

    def accel(self, q, qd, torque, gravity=None, dtype=None):
        """Forward dynamics qdd = M(q)^-1 (torque - rne(q, qd, 0)), joint friction included
        (reference Dynamics.accel, Dynamics.py:424-510)."""
        return self._dyn("b2k_rne_accel", [q, qd, torque], (self.n,), gravity=gravity, use_gravity=True, dtype=dtype)

    # ---- static forces (reference DynamicsMixin, Dynamics.py): _static.py, csrc/b2k_static.cu
    def _static_mass_table(self) -> np.ndarray:
        """n x 4 doubles (m_j, c_j) for b2k_gravjac / b2k_paycap: c_j is link j's centre of mass in the frame right after
        its joint, tail_j r_j, with tail_j the link's elementary transforms behind the joint (DHLink._to_ets)."""
        if self._static_mass is None:
            M = np.zeros((self.n, 4))
            for j, l in enumerate(self.links):
                ets = list(l.ets)
                tail = np.eye(4)
                for et in ets[next(i for i, et in enumerate(ets) if et.isjoint) + 1:]:
                    tail = tail @ et.A()
                M[j, 0] = l.m
                M[j, 1:] = tail[:3, :3] @ l.r + tail[:3, 3]
            self._static_mass = np.ascontiguousarray(M)
        return self._static_mass

    def gravjac(self, q, gravity=None, dtype=None):
        """Gravity load and base-frame Jacobian from one walk (reference DynamicsMixin.gravjac): ``(tau, J0)``, tau (n,) /
        (N,n) = -sum_i J_ci^T m_i g from the link centre-of-mass Jacobians, g the world-frame gravity (default
        ``robot.gravity``); J0 (6,n) / (N,6,n) equals ``jacob0(q)`` (base and tool included).  tau equals ``gravload`` for
        robots without flipped joints; a flipped joint follows the chain here, as in ``jacob0``, while ``rne`` and
        ``gravload`` ignore ``flip`` (as the reference's frne does)."""
        return _static.gravjac(self, q, gravity=gravity, dtype=dtype)

    def pay(self, W, q=None, J=None, frame=1, dtype=None):
        """Joint torques of a payload wrench W = [fx fy fz mx my mz] applied to the end effector (reference
        DynamicsMixin.pay): tau = -J^T W, (n,) / (N,n).  W (6,) is one wrench for every row, (N,6) one per row; it is in
        the end-effector frame for ``frame=1`` (J = jacobe) and the world frame for ``frame=0`` (J = jacob0).  Give
        exactly one of q and J; a given J (6,n) / (N,6,n) is used as it is and ``frame`` does not enter."""
        return _static.pay(self.ets(), W, q=q, J=J, frame=frame, dtype=dtype)

    def paycap(self, w, tauR, frame=1, q=None, gravity=None, dtype=None):
        """Static payload capacity under joint torque limits (reference DynamicsMixin.paycap): ``(wmax, joint)``.
        With w^ = w / |w| per row, tau_B the gravity load and tau_P = pay(w^, q, frame), wmax_j = (tauR[j,0] - tau_B,j) /
        tau_P,j where tau_P,j > 0, (tauR[j,1] - tau_B,j) / tau_P,j where tau_P,j < 0, +inf where tau_P,j = 0; joint is
        the first argmin, so the capacity of a pose is wmax[joint].  tauR is (n,2): column 0 the largest torque, column 1
        the smallest.  wmax (n,) / (N,n); joint an int / (N,) int32 array.  A zero row of an (N,6) w gives NaN and -1."""
        return _static.paycap(self, w, tauR, frame=frame, q=q, gravity=gravity, dtype=dtype)

    def friction(self, qd, dtype=None):
        """Joint friction torque (reference DynamicsMixin.friction / Link.friction): tau_j = -(G_j^2 B_j qd_j +
        |G_j| Tc_j(qd_j)), Tc_j = Tc+ for qd_j > 0, Tc- for qd_j < 0, 0 at rest -- the terms ``rne`` adds, negated.
        (n,) / (N,n)."""
        return _static.friction(self, qd, dtype=dtype)

    def payload(self, m, p=(0.0, 0.0, 0.0)):
        """Put a point mass m at p (in the last link's frame; the tool does not enter) on the last link (reference
        DynamicsMixin.payload): its mass and centre of mass are replaced, its inertia tensor is kept.  ``payload(0)``
        removes the last link's mass.  Goes through the link setters, so the next rne / gravload / gravjac / paycap
        sees the new mass."""
        last = self.links[-1]
        last.m = m
        last.r = p

    # ---- operational-space dynamics (reference DynamicsMixin, Dynamics.py between gravload and itorque): _opspace.py
    def inertia_x(self, q, pinv=False, representation="rpy/xyz", Ji=None, dtype=None):
        """Operational-space inertia Mx = Ji^T M Ji, (6,6) or (N,6,6); Ji = inv / pinv of jacob0_analytical."""
        return _opspace.inertia_x(self, q, pinv=pinv, representation=representation, Ji=Ji, dtype=dtype)

    def coriolis_x(self, q, qd, pinv=False, representation="rpy/xyz", J=None, Ji=None, Jd=None, C=None, Mx=None, dtype=None):
        """Operational-space Coriolis matrix Cx = Ji^T C Ji - Mx Jad Ji, (6,6) or (N,6,6)."""
        return _opspace.coriolis_x(self, q, qd, pinv=pinv, representation=representation, J=J, Ji=Ji, Jd=Jd, C=C, Mx=Mx, dtype=dtype)

    def gravload_x(self, q, gravity=None, pinv=False, representation="rpy/xyz", Ji=None, dtype=None):
        """Operational-space gravity load Gx = Ji^T G, (6,) or (N,6)."""
        return _opspace.gravload_x(self, q, gravity=gravity, pinv=pinv, representation=representation, Ji=Ji, dtype=dtype)

    def accel_x(self, q, xd, wrench, gravity=None, pinv=False, representation="rpy/xyz", dtype=None):
        """Operational-space forward dynamics: task acceleration (6,) or (N,6) under the end-effector wrench."""
        return _opspace.accel_x(self, q, xd, wrench, gravity=gravity, pinv=pinv, representation=representation, dtype=dtype)
