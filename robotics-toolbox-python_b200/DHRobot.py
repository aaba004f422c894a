"""DH / MDH serial-link robots: kinematics through the compiled ETS chain, inverse dynamics
through the batched RNE kernel.

Mirrors the hot-path part of the reference's ``DHRobot`` (reference
src/roboticstoolbox/robot/DHRobot.py): ``ets()`` 878-918, ``fkine`` 920-979, ``jacobe`` 1066-1140,
``jacob0`` 1142-1198, ``rne`` 1373-1456 with its parameter packing ``_init_rne`` 1340-1361 and
dirty tracking (DHLink.py:24-51), ``ikine_LM`` 2454-2474, and the closed-form ``ikine_6s`` as ``ikine_a``; ``ikine_ur``
and ``ikine_panda`` are the closed forms of UR-type arms and of Panda-type arms at a given q7, which the reference lacks.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional

import numpy as np

from . import _buffers as B
from . import _identify
from . import _lib
from . import _opspace
from . import _static
from ._se3 import SE3
from .DHLink import DHLink
from .ET import ET
from .ETS import ETS, _mat44
from .IK import IKSolution
from ._identify import IdentifyResult  # noqa: F401  (the result type of identify)


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

    def partial_fkine0(self, q=None, n=3, **kwargs):
        return self.ets().partial_fkine0(q, n=n, **kwargs)

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

    # ---- closed-form inverse kinematics (reference DHRobot.ikine_6s, which Puma560.ikine_a calls; UR- and Panda-type arms):
    # csrc/b2k_ik6s.cu
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

    def _ikine_a_table(self, method="ikine_a", n=6, mdh=False) -> np.ndarray:
        """(n,4) rows of (d, a, alpha, offset) for b2k_ikine_6s / b2k_ikine_ur (n = 6, standard DH) or b2k_ikine_panda
        (n = 7, modified DH), after the checks their tables cannot express; ``method`` names the caller in the messages"""
        if self.n != n:
            raise ValueError(f"{method}: the closed form serves {n}-joint arms; this robot has {self.n} joints")
        if bool(self.mdh) != mdh:
            have, want = ("modified DH", "standard DH") if self.mdh else ("standard DH", "modified DH")
            raise ValueError(f"{method}: the closed form serves {want}; this robot uses {have}")
        for j, l in enumerate(self.links):
            if not l.isrevolute:
                raise ValueError(f"{method}: joint {j + 1} is prismatic; the closed form needs revolute joints")
            if l.flip:
                raise ValueError(f"{method}: joint {j + 1} is flipped; the closed form needs unflipped joints")
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
        return self._ikine_closed(T, config, dtype, "b2k_ikine_6s", "ikine_a")

    def ikine_ur(self, T, config="lun", dtype=None) -> IKSolution:
        """Analytic inverse kinematics of a UR-type 6R arm (Universal Robots UR3 / UR5 / UR10 and any arm of their link
        pattern): the exact joint solution for a shoulder (l / r), elbow (u / d) and wrist (n / f) configuration, up to
        eight per pose, with no iteration.

        The robot must be a standard-DH, all-revolute, unflipped 6-joint arm with alpha = (pi/2, 0, 0, pi/2, -pi/2, any),
        a1 = a4 = a5 = 0, a2 != 0 and a3 != 0; any other robot raises ValueError naming what breaks the pattern.  d1 ..
        d6, a6, alpha6, the offsets, the base and the tool are free.  The letters are predicates of the solution, in the
        frame of link 1 with X = a2 c2 + a3 c23 and Y = a2 s2 + a3 s23 the position of the wrist's first joint (O4):
        ``r`` iff O5 . x1 >= 0 (as for Puma arms), ``u`` iff the elbow lies above the shoulder-O4 line with the base z
        axis up, sign(X) (X a2 s2 - Y a2 c2) > 0, and ``n`` iff sin(theta5) >= 0.  Inputs, outputs, shapes, dtypes,
        placement and the reason strings are those of :meth:`ikine_a`.  Joint limits are not applied."""
        return self._ikine_closed(T, config, dtype, "b2k_ikine_ur", "ikine_ur")

    def ikine_panda(self, T, q7, config="lun", dtype=None) -> IKSolution:
        """Analytic inverse kinematics of a Panda-type 7R arm (Franka Emika Panda, :class:`models.PandaMDH`, and any arm of
        its link pattern) at a given last joint coordinate q7: the exact joint solution for a shoulder (l / r), elbow
        (u / d) and wrist (n / f) configuration, up to eight per pose, with no iteration.  Fixing q7 makes the 7R arm's
        one-parameter family of solutions finite; sweeping q7 over a batch explores its redundancy.

        The robot must be a modified-DH, all-revolute, unflipped 7-joint arm with alpha2 .. alpha6 = (-pi/2, pi/2, pi/2,
        -pi/2, pi/2), a2 = a3 = a6 = 0, d2 = d4 = d6 = 0, hypot(a4, d3) != 0 and hypot(a5, d5) != 0; any other robot
        raises ValueError naming what breaks the pattern.  a1, alpha1, d1, d3, a4, a5, d5, a7, alpha7, d7, the offsets,
        the base and the tool are free.  ``q7`` is a scalar or one value per pose, (N,) numpy or a CUDA tensor; it is
        q[6] of every returned solution as given, and a non-finite q7 gives a NaN row.  The letters are predicates of
        the solution, with O_k and x_k, z_k the origin and axes of link frame k: ``r`` iff sin(theta2) >= 0 (at
        sin(theta2) = 0 both shoulder codes return theta2 = atan2(R13, R33) within rounding of 0, so both read as ``r``),
        ``u`` iff ((O2 - O4) x (O6 - O4)) . z4 >= 0, ``n`` iff (O2 - O6) . x5 >= 0.  q has 7 columns: (7,), (N,7),
        (k,7) or (N,k,7); otherwise inputs, outputs, shapes, dtypes, placement and the reason strings are those of
        :meth:`ikine_a`.  Joint limits are not applied."""
        return self._ikine_closed(T, config, dtype, "b2k_ikine_panda", "ikine_panda", q7=q7)

    def _ikine_closed(self, T, config, dtype, entry, method, q7=None) -> IKSolution:
        """The body of ikine_a, ikine_ur and ikine_panda: ``entry`` is the C entry point, ``method`` names the caller in
        messages, ``q7`` is given for the 7R entry point only"""
        seven = entry == "b2k_ikine_panda"
        configs = [config] if isinstance(config, str) else list(config)
        if not 1 <= len(configs) <= 8:
            raise ValueError(f"{method}: give 1 to 8 configurations, got {len(configs)}")
        codes = []
        for c in configs:
            v = self.config_validate(c, self._IKINE_A_LETTERS)
            codes.append(int(v[0] == "r") | int(v[1] == "d") << 1 | int(v[2] == "f") << 2)
        conf = np.array(codes, dtype=np.int32)
        dh = self._ikine_a_table(method, 7, True) if seven else self._ikine_a_table(method)
        base = None if np.array_equal(self._base, np.eye(4)) else np.ascontiguousarray(self._base)
        tool = None if np.array_equal(self._tool, np.eye(4)) else np.ascontiguousarray(self._tool)
        solve = getattr(_lib.lib(), entry)
        cp = conf.ctypes.data_as(_lib.ip)
        no_q7 = (None,) if seven else ()
        # the link pattern is checked by the C entry point; N = 0 validates without touching a device
        _lib.check(solve(_lib.F64, _lib.dptr(dh), _lib.dptr(base), _lib.dptr(tool), None, *no_q7, 0, len(conf), cp, None, None,
                         None))
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
        q7d = (self._ikine_q7(q7, N, dt, Td, method),) if seven else ()
        q = B.empty((N, k, dh.shape[0]), dt, like=Td)
        ok = B.empty_i32((N, k), like=Td)
        _lib.check(solve(B.code(dt), _lib.dptr(dh), _lib.dptr(base), _lib.dptr(tool), B.ptr(Td), *map(B.ptr, q7d), N, k, cp,
                         B.ptr(q), B.ptr(ok), B.stream_ptr(Td)))
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

    @staticmethod
    def _ikine_q7(q7, N, dt, Td, method):
        """q7 as a contiguous (N,) tensor of dtype dt on the device of Td: a scalar is repeated, an array must be (N,)"""
        B.check_numeric(q7, "q7")
        if B.is_tensor(q7):
            if q7.is_cuda and q7.device != Td.device:
                raise ValueError(f"{method}: q7 is on {q7.device}, T on {Td.device}")
            if q7.ndim == 0:
                q7 = float(q7)
        else:
            q7 = np.asarray(q7)
            if q7.ndim == 0:
                q7 = float(q7)
        if isinstance(q7, float):
            return B.torch().full((N,), q7, dtype=B.tdtype(dt), device=Td.device)
        if tuple(q7.shape) != (N,):
            raise ValueError(f"{method}: q7 must be a scalar or have shape ({N},), one value per pose; got {tuple(q7.shape)}")
        return B.to_device(q7, dt, device=Td.device)

    def ik_NR(self, Tep, **kwargs):
        return self.ets().ik_NR(Tep, **kwargs)

    def ik_GN(self, Tep, **kwargs):
        return self.ets().ik_GN(Tep, **kwargs)

    def ikine_NR(self, Tep, **kwargs):
        return self.ets().ikine_NR(Tep, **kwargs)

    def ikine_GN(self, Tep, **kwargs):
        return self.ets().ikine_GN(Tep, **kwargs)

    def ikine_QP(self, Tep, **kwargs):
        return self.ets().ikine_QP(Tep, **kwargs)

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

    def _rne_handle(self):
        """The RNE handle of the current link parameters, rebuilt if they changed (reference @_check_rne, DHLink.py:24-51)."""
        if self._rne_ob is None or self._dynchanged:
            self.delete_rne()
            self._init_rne()
        return self._rne_ob

    def _kernel_gravity(self, gravity):
        """The gravity vector the kernels take: the recursion has no base, so gravity is rotated into the base frame
        instead (reference 1431-1433) and handed over negated (1449)."""
        g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        return np.ascontiguousarray(-(self._base[:3, :3].T @ g))

    def rne(self, q, qd=None, qdd=None, gravity=None, fext=None, base_wrench=False, dtype=None):
        """Inverse dynamics tau = RNE(q, qd, qdd): (n,) for one state, (N,n) for a trajectory
        (reference DHRobot.rne 1373-1456 -> frne.frne per row).

        ``base_wrench=True`` returns ``(tau, wbase)``: tau as above and wbase (6,) / (N,6) = [fx, fy, fz, mx, my, mz],
        the wrench the base exerts on link 1, expressed in frame 0 (the chain's base frame, after ``robot.base``) with
        the moment about its origin.  Both come from the same recursion (one kernel launch)."""
        h = self._rne_handle()
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
        ng = self._kernel_gravity(gravity)
        fx = None if fext is None else np.ascontiguousarray(np.asarray(fext, dtype=np.float64).reshape(6))
        L = _lib.lib()
        if host:
            t = B.require_cuda()
            qh, qdh, qddh = (np.ascontiguousarray(x, dtype=dt) for x in (q2, qd2, qdd2))
            tau = _lib.host_result((N, n), dt)
            if base_wrench:
                wb = _lib.host_result((N, 6), dt)
                _lib.check(L.b2k_rne_wrench_host(h, B.code(dt), qh.ctypes.data, qdh.ctypes.data, qddh.ctypes.data, N,
                                                 _lib.dptr(ng), _lib.dptr(fx), tau.ctypes.data, wb.ctypes.data,
                                                 t.cuda.current_device()))
            else:
                _lib.check(L.b2k_rne_host(h, B.code(dt), qh.ctypes.data, qdh.ctypes.data, qddh.ctypes.data, N,
                                          _lib.dptr(ng), _lib.dptr(fx), tau.ctypes.data, t.cuda.current_device()))
        else:
            qt, qdt, qddt = (B.to_device(x, dt) for x in (q2, qd2, qdd2))
            tau = B.empty((N, n), dt, like=qt)
            if base_wrench:
                wb = B.empty((N, 6), dt, like=qt)
                _lib.check(L.b2k_rne_wrench(h, B.code(dt), B.ptr(qt), B.ptr(qdt), B.ptr(qddt), N, _lib.dptr(ng),
                                            _lib.dptr(fx), B.ptr(tau), B.ptr(wb), B.stream_ptr(qt)))
            else:
                _lib.check(L.b2k_rne(h, B.code(dt), B.ptr(qt), B.ptr(qdt), B.ptr(qddt), N, _lib.dptr(ng),
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

        h = self._rne_ob if callable(Q) else self._rne_handle()
        return _fdyn(self, _lib.lib().b2k_rne_fdyn if not callable(Q) else None, h, self._kernel_gravity, T, q0, Q=Q, Q_args=Q_args,
                     qd0=qd0, solver=solver, solver_args=solver_args, dt=dt, gravity=gravity, max_steps=max_steps, dtype=dtype)

    def rollout(self, q0, tau, dt, qd0=None, sensitivities=False, gravity=None, dtype=None):
        """Fixed-step rollouts of the forward dynamics under a torque sequence, with their exact linearisation: the
        named tuple ``(t, q, qd, A, B)``.

        Each step holds its torque (zero-order hold) and takes one classical RK4 step of x = [q; qd] with
        f(x, tau) = [qd; accel(q, qd, tau)], ``accel`` exactly as this robot computes it (friction and armature kept):
        x_{k+1} = x_k + dt/6 (k1 + 2 k2 + 2 k3 + k4).  ``q0`` / ``qd0`` are (n,) or (N,n) (``qd0=None``: at rest), ``tau``
        is (K,n), shared by every trajectory, or (N,K,n); ``dt`` a positive, finite scalar.  t = k dt (k = 0..K, numpy),
        q / qd (N,K+1,n) with index 0 the initial state.  With ``sensitivities=True``, A (N,K,2n,2n) = d x_{k+1} / d x_k
        and B (N,K,2n,n) = d x_{k+1} / d tau_k, ``[i, j] = d out_i / d in_j``, chained through the four stages from
        ``accel_derivatives`` at each stage state (never differences; Coulomb friction contributes 0); else None.  One
        trajectory (``q0``, ``qd0`` 1-D, ``tau`` 2-D) drops the N axis; a 1-D input next to batched ones is broadcast.
        numpy in, numpy out; CUDA tensors in, tensors out on their device.  A singular M gives non-finite values from that
        step on.  One kernel launch: one lane per trajectory, generated for this robot (NVRTC); all-revolute arms only.

        Costs to plan for.  The first call per (robot, dtype, gravity pattern, sensitivities) compiles the kernel: a few
        seconds for the named arms, but the sensitivities program of an arm whose link table has no structure (general
        twist angles) takes up to about 20 s at n = 8 and 2 min at n = 10 on a CPU core.  The sensitivities kernel keeps
        each trajectory's working set, 15 n^2 reals, in local memory (about 5 KB per thread for a 6-joint arm in fp64),
        and the driver reserves that for every thread the device can hold: measured on an H100, 940 MB of device memory
        for the Puma560 in fp64, kept for the life of the process."""
        from ._rollout import rollout as _rollout

        if any(l.sigma != 0 for l in self.links):
            raise ValueError("rollout serves all-revolute arms; this robot has a prismatic joint")
        if self.n > _lib.MAX_JOINTS:
            raise ValueError(f"rollout serves up to {_lib.MAX_JOINTS} joints; this robot has {self.n}")
        return _rollout(self, _lib.lib().b2k_rne_rollout, self._rne_handle(), self._kernel_gravity, q0, tau, dt, qd0=qd0,
                        sensitivities=sensitivities, gravity=gravity, dtype=dtype)

    _RNE_MODES = {"rne": 0, "inertia": 1, "gravload": 2, "itorque": 3, "coriolis": 4, "accel": 5, "rne_wrench": 6}
    _ROLLOUT_MODES = (305, 308)  # b2k_rne_spec_info: the rollout kernel, states only / with sensitivities

    _DERIV_OPS = {"rne_derivatives": "inverse", "accel_derivatives": "forward"}

    def rne_kernel_info(self, op="rne", dtype=np.float64, gravity=None, fext=None) -> str:
        """Which kernel serves `op` for this robot: the robot-specialised one (generated from the link table and
        compiled with NVRTC at first use; the line lists its multiply / FMA / add count per row, registers and
        shared memory) or the pre-compiled generic one, with the reason.  ``op="rollout"`` gives two lines: the
        rollout kernel for states only and with sensitivities."""
        if op in self._DERIV_OPS or op == "rne_regressor":
            allrev = all(l.sigma == 0 for l in self.links)
            shape = (f"{'double' if np.dtype(dtype) == np.float64 else 'float'}, n={self.n}, {'MDH' if self.mdh else 'DH'}, "
                     f"{'all-revolute' if allrev else 'prismatic'}")
            if op == "rne_regressor":
                return f"generic k_rne_regressor<{shape}> (the robot-specialised path generates no regressor kernels)"
            return f"generic k_rne_deriv<{shape}, {self._DERIV_OPS[op]}> (the robot-specialised path generates no derivative kernels)"
        h = self._rne_handle()
        g = self._kernel_gravity(gravity)
        buf = C.create_string_buffer(2048)
        lines = []
        for mode in (self._ROLLOUT_MODES if op == "rollout" else (self._RNE_MODES[op],)):
            _lib.check(_lib.lib().b2k_rne_spec_info(h, mode, B.code(np.dtype(dtype)), _lib.dptr(g),
                                                    int(fext is not None and np.any(np.asarray(fext) != 0)), buf, 2048))
            lines.append(buf.value.decode())
        return "\n".join(lines)

    # ---- dynamics built on the recursion (reference DynamicsMixin, Dynamics.py; SURVEY 8f-1)
    def _dyn_inputs(self, ins, dtype):
        """The inputs of a batched dynamics call as contiguous (N, n) device tensors of one dtype: returns (dtype,
        whether the inputs were host arrays, whether they were single (n,) states, the tensors, N)."""
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
        return dt, host, single, dev, N

    def _dyn(self, fn_name, ins, out_tail, gravity=None, use_gravity=False, dtype=None, fext=None, use_fext=False, n_out=1):
        """Shared front end of the fan-out kernels: every input (N,n) or (n,), one launch.  With n_out > 1 the kernel
        writes that many outputs of the same shape, returned as a tuple."""
        h = self._rne_handle()
        n = self.n
        dt, host, single, dev, N = self._dyn_inputs(ins, dtype)
        outs = [B.empty((N,) + out_tail, dt, like=dev[0]) for _ in range(n_out)]
        args = [h, B.code(dt)] + [B.ptr(t) for t in dev] + [N]
        if use_gravity:
            g = self._kernel_gravity(gravity)
            args.append(_lib.dptr(g))
        if use_fext:
            fx = None if fext is None else np.ascontiguousarray(np.asarray(fext, dtype=np.float64).reshape(6))
            args.append(_lib.dptr(fx))
        args += [B.ptr(o) for o in outs] + [B.stream_ptr(dev[0])]
        _lib.check(getattr(_lib.lib(), fn_name)(*args))
        if host:
            outs = [B.to_host(o) for o in outs]
        outs = [o[0] if single else o for o in outs]
        return outs[0] if n_out == 1 else tuple(outs)

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

    def rne_derivatives(self, q, qd, qdd, gravity=None, fext=None, dtype=None):
        """Exact first derivatives of inverse dynamics: ``(dtau_dq, dtau_dqd)``, each (n,n) for one state or (N,n,n).

        Layout: ``[..., i, k] = d tau_i / d x_k`` -- rows are torques, columns the variable (numpy's Jacobian
        convention).  tau is exactly what ``rne(q, qd, qdd, gravity, fext)`` computes: gravity rotated by the base, the
        tip wrench, the armature term G^2 Jm qdd and joint friction.  Viscous friction adds G^2 B to the diagonal of
        ``dtau_dqd``; Coulomb friction is piecewise constant and adds 0 (also at qd = 0, where rne uses 0).  A
        prismatic joint is differentiated through d = q + offset.  Where rne keeps a reference quirk (the modified-DH
        prismatic first joint, ``flip`` ignored) this is the derivative of what the recursion computes.  d tau / d qdd
        is ``inertia(q)``.  The values are forward-mode tangents through the recursion (no finite differences), one
        kernel launch for the whole batch."""
        return self._dyn("b2k_rne_derivatives", [q, qd, qdd], (self.n, self.n), gravity=gravity, use_gravity=True, dtype=dtype,
                         fext=fext, use_fext=True, n_out=2)

    def accel_derivatives(self, q, qd, torque, gravity=None, dtype=None):
        """Exact first derivatives of forward dynamics: ``(dqdd_dq, dqdd_dqd, dqdd_dtau)``, each (n,n) or (N,n,n), in
        the layout of ``rne_derivatives`` (``[..., i, k] = d qdd_i / d x_k``).

        With qdd* = ``accel(q, qd, torque, gravity)`` (friction kept as accel keeps it) and M = ``inertia(q)``:
        ``dqdd_dq = -M^-1 dtau_dq`` and ``dqdd_dqd = -M^-1 dtau_dqd``, the inverse-dynamics derivatives taken at qdd*,
        and ``dqdd_dtau = M^-1``.  All three come from one kernel launch."""
        return self._dyn("b2k_rne_accel_derivatives", [q, qd, torque], (self.n, self.n), gravity=gravity, use_gravity=True,
                         dtype=dtype, n_out=3)

    # ---- parameter identification: the dynamics regressor (DESIGN f-16; no reference counterpart)
    def dynamic_parameters(self) -> np.ndarray:
        """The (14n,) float64 parameter vector pi of the current links, the one ``rne_regressor`` multiplies: 14 per link,
        link-major, ``[m, m rx, m ry, m rz, Ixx, Iyy, Izz, Ixy, Iyz, Ixz, Jm, B, Tc+, Tc-]``.  r is the link's centre of
        mass in its frame; the inertia entries are those of I_o = I + m (r.r E - r r^T), the link's inertia moved to the
        link-frame origin, in the order of the 6-vector form of ``I``.  The symmetric part of ``I`` is used: the link
        setter rejects an asymmetry above 1e-8, and ``rne_regressor(...) @ dynamic_parameters() == rne(...)`` holds up
        to that asymmetry.  The gear ratio G is not a parameter."""
        pi = np.zeros(14 * self.n)
        for j, l in enumerate(self.links):
            m, r = float(l.m), np.asarray(l.r, dtype=np.float64)
            Io = 0.5 * (l.I + l.I.T) + m * (r @ r * np.eye(3) - np.outer(r, r))
            pi[14 * j:14 * j + 14] = (m, *(m * r), Io[0, 0], Io[1, 1], Io[2, 2], Io[0, 1], Io[1, 2], Io[0, 2], l.Jm, l.B,
                                      l.Tc[0], l.Tc[1])
        return pi

    def rne_regressor(self, q, qd, qdd, gravity=None, dtype=None):
        """The dynamics regressor Y(q, qd, qdd): (n, 14n) for one state or (N, n, 14n), with
        ``Y @ dynamic_parameters() == rne(q, qd, qdd, gravity)`` (no tip wrench) for every link table rne serves:
        prismatic joints through d = q + offset, the modified-DH prismatic first joint as rne treats it, ``flip``
        ignored.  Y depends on the kinematics and the gear ratios only, not on the masses, inertias or friction.

        Column 14i + k of row j is the torque of joint j per unit of parameter k of link i: exact 0 for i < j.  The
        friction columns of link j (Jm, B, Tc+, Tc-) are G_j^2 qdd_j, G_j^2 qd_j, |G_j| [qd_j > 0] and |G_j| [qd_j < 0]
        in row j (0 at qd_j = 0, as rne) and 0 in every other row.  Input forms, dtype and device rules are those of
        ``rne_derivatives``; one kernel launch."""
        return self._dyn("b2k_rne_regressor", [q, qd, qdd], (self.n, 14 * self.n), gravity=gravity, use_gravity=True,
                         dtype=dtype)

    def regressor_gram(self, q, qd, qdd, tau, gravity=None, weights=None, dtype=None):
        """The normal equations of identification, accumulated on the device without Y existing in full: numpy
        ``(G, b, s)`` with G (14n, 14n) = sum Y^T W Y, b (14n,) = sum Y^T W tau and the float s = sum tau^T W tau over the
        rows, W = diag(weights) (n joint weights >= 0, default 1), always in float64.  q, qd, qdd, tau (N, n) or (n,),
        numpy or CUDA tensors; Y is computed in ``dtype`` (default: that of q) in chunks of 4096 rows.  G is exactly
        symmetric and two equal calls give equal bits."""
        import torch

        h = self._rne_handle()
        n, p = self.n, 14 * self.n
        dt, _, _, dev, N = self._dyn_inputs([q, qd, qdd, tau], dtype)
        w = None
        if weights is not None:
            w = np.ascontiguousarray(np.asarray(weights, dtype=np.float64))
            if w.shape != (n,):
                raise ValueError(f"weights must have shape ({n},); got {w.shape}")
        G = torch.empty((p, p), dtype=torch.float64, device=dev[0].device)
        b = torch.empty(p, dtype=torch.float64, device=dev[0].device)
        s = torch.empty(1, dtype=torch.float64, device=dev[0].device)
        _lib.check(_lib.lib().b2k_rne_regressor_gram(h, B.code(dt), *(B.ptr(t) for t in dev), N,
                                                     _lib.dptr(self._kernel_gravity(gravity)), _lib.dptr(w), B.ptr(G),
                                                     B.ptr(b), B.ptr(s), B.stream_ptr(dev[0])))
        return G.cpu().numpy(), b.cpu().numpy(), float(s.item())

    def identify(self, q, qd, qdd, tau, gravity=None, weights=None, friction=True, rcond=1e-10, dtype=None):
        """Least-squares identification of the link parameters from logged (q, qd, qdd, tau): the named tuple
        ``(pi, rank, rms)``.  pi (14n,) is the minimum-norm solution of tau = Y pi (the convention of
        ``dynamic_parameters``) from the normal equations of ``regressor_gram``: G is scaled to unit diagonal, and
        eigenvalues of the scaled G below ``rcond`` times the largest are dropped; rank is the number kept.  rcond must
        exceed the rounding of the scaled G in the compute type: the default 1e-10 suits float64; float32 rounds Y to
        about 1e-7, so an exact dependency between columns can leave an eigenvalue far above 1e-10 there (use about 1e-5).  Parameters
        whose column of Y is zero (below 16 eps of the compute type times the largest column norm) get 0.  ``friction=False`` drops the four friction parameters of every link (they come
        back as 0).  rms is the weighted residual sqrt((s - 2 pi.b + pi.G.pi) / (N n)); the three terms cancel, so an rms
        below about sqrt(eps) times the rms of tau is not resolved (an exact fit reads as 0 up to that level).

        Only combinations of parameters are identifiable in general, so pi is not a physical link table; base
        parameters and writing pi back into the links are left to the caller."""
        G, b, s = self.regressor_gram(q, qd, qdd, tau, gravity=gravity, weights=weights, dtype=dtype)
        n = self.n
        shape = tuple(q.shape) if hasattr(q, "shape") else np.shape(q)
        N = 1 if len(shape) == 1 else int(shape[0])
        keep = np.ones(14 * n, dtype=bool)
        if not friction:
            for j in range(n):
                keep[14 * j + 10:14 * j + 14] = False
        return _identify.solve(G, b, s, keep, np.finfo(B.pick_dtype(q, dtype)).eps, rcond, N, n)

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
