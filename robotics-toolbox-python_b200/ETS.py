"""Elementary transform sequences -- the operator API of the hot path.

Keeps the reference's ``ETS`` method names, argument meaning and error behaviour for the path
this package accelerates (reference src/roboticstoolbox/robot/ETS.py):

    eval / fkine   ETS.py:951-1141   -> b2k_fkine          (reference: fknm.ETS_fkine)
    jacob0         ETS.py:1143-1266  -> b2k_jacob0         (reference: fknm.ETS_jacob0, one q per call)
    jacobe         ETS.py:1268-1332  -> b2k_jacobe         (reference: fknm.ETS_jacobe, one q per call)
    ik_LM          ETS.py:2014-2170  -> b2k_ik_lm, C++ loop semantics   (reference: fknm.IK_LM_c)
    ikine_LM       ETS.py:2443-2637  -> b2k_ik_lm, Python solver semantics (reference: IK.IK_LM.solve)
    fkine_jacob0   (extension)       -> b2k_fkine_jacob0   one pass giving pose and Jacobian

All of them accept an (N, n) batch of joint coordinates (the reference only batches fkine) as a
numpy array / list (host: results come back as numpy) or a CUDA torch tensor (results stay on
the device).  There is no Python / sympy fallback: a non-numeric q raises TypeError exactly like
the reference's C layer does (fknm.cpp:1304-1318), and the reference's silent fall-through to
slow Python (ETS.py:1075-1078) is deliberately not reproduced.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Union

import numpy as np

from . import _buffers as B
from . import _lib
from ._se3 import SE3
from .ET import AXES, ET
from .IK import IKSolution


def _mat44(T, name):
    """None / SE3-like / array -> fp64 (4,4) or None."""
    if T is None:
        return None
    T = getattr(T, "A", T)
    T = np.ascontiguousarray(np.asarray(T, dtype=np.float64))
    if T.shape != (4, 4):
        raise ValueError(f"{name} must be a 4x4 matrix")
    return T


class ETS:
    """A sequence of :class:`ET` (reference ETS.py:57-69, 760-840)."""

    def __init__(self, arg: Union[None, ET, "ETS", List] = None):
        ets: List[ET] = []
        if arg is None:
            pass
        elif isinstance(arg, ET):
            ets = [arg.copy()]
        elif isinstance(arg, ETS):
            ets = [e.copy() for e in arg._ets]
        elif isinstance(arg, (list, tuple)):
            for a in arg:
                if isinstance(a, ET):
                    ets.append(a.copy())
                elif isinstance(a, ETS):
                    ets.extend(e.copy() for e in a._ets)
                else:
                    raise TypeError("bad arg")
        else:
            raise TypeError("Invalid arg")
        self._ets = ets
        self._assign_jindices()
        self._handle = None

    # jindex auto-numbering, reference ETS.py:803-840
    def _assign_jindices(self):
        joints = [e for e in self._ets if e.isjoint]
        n = len(joints)
        have = sum(1 for j in joints if j.jindex is not None)
        seq = sum(1 for k, j in enumerate(joints) if j.jindex is not None and j.jindex == k)
        self._auto_jindex = False
        if n and have == n - 1 and seq == n - 1 and joints[-1].jindex is None:
            joints[-1].jindex = n - 1
            self._auto_jindex = True
        elif have > 0 and have != n:
            raise ValueError("You can not have some jindices set for the ET's in arg. It must be all or none")
        elif have == 0 and n > 0:
            for k, j in enumerate(joints):
                j.jindex = k
            self._auto_jindex = True

    @staticmethod
    def from_links(link_ets: List["ETS"]) -> "ETS":
        """Concatenate per-link ETSs into a robot chain.  When every link's joint index was only
        auto-assigned (each link numbered its own joint 0), the joints are renumbered 0..n-1 in
        chain order -- what the reference's robot constructor does (BaseRobot.py:336-352)."""
        renumber = all(e._auto_jindex or e.n == 0 for e in link_ets)
        parts: List[ET] = []
        for e in link_ets:
            for et in e._ets:
                c = et.copy()
                if renumber and c.isjoint:
                    c._jindex = None
                parts.append(c)
        return ETS(parts)

    # ---- composition
    def __mul__(self, other):
        if isinstance(other, ET):
            return ETS([*self._ets, other])
        if isinstance(other, ETS):
            return ETS([*self._ets, *other._ets])
        return NotImplemented

    __add__ = __mul__

    def inv(self) -> "ETS":
        """Inverse of the ETS: the inverses of the individual ETs in reverse order (reference ETS.inv,
        ETS.py:545-576).  Joints keep their jindex, so explicit joint indices are essential."""
        return ETS([et.inv() for et in reversed(self._ets)])

    def __len__(self):
        return len(self._ets)

    def __iter__(self):
        return iter(self._ets)

    def __getitem__(self, i):
        r = self._ets[i]
        return ETS(r) if isinstance(i, slice) else r

    def __repr__(self):
        return " ⊕ ".join(repr(e) for e in self._ets)

    # ---- structure, reference ETS.py:400-760
    @property
    def n(self) -> int:
        return sum(1 for e in self._ets if e.isjoint)

    @property
    def m(self) -> int:
        return len(self._ets)

    def joints(self) -> List[ET]:
        return [e for e in self._ets if e.isjoint]

    def joint_idx(self) -> List[int]:
        return [i for i, e in enumerate(self._ets) if e.isjoint]

    @property
    def jindices(self) -> np.ndarray:
        return np.array([e.jindex for e in self.joints()], dtype=int)

    @property
    def qlim(self) -> np.ndarray:
        """(2, n) joint limits with the reference's defaults for unset limits (ET.py:109-115)."""
        ql = np.array([e._qlim_default() for e in self.joints()], dtype=np.float64).reshape(-1, 2)
        return ql.T.copy()

    @property
    def structure(self) -> str:
        return "".join("R" if e.isrotation else "P" for e in self.joints())

    def compile(self) -> "ETS":
        """Fold runs of constants into single SE(3) constants (reference ETS.py:857-906).  The
        native chain compiler applies the same rule internally; this is for inspection."""
        out: List[ET] = []
        acc = None
        for e in self._ets:
            if e.isjoint:
                if acc is not None:
                    out.append(ET.SE3(acc))
                    acc = None
                out.append(e.copy())
            else:
                acc = e.A() if acc is None else acc @ e.A()
        if acc is not None:
            out.append(ET.SE3(acc))
        return ETS(out)

    def describe(self) -> dict:
        """Neutral per-ET description: exactly what the reference marshals into fknm.ET_init
        (ET.py:100-125).  Consumed by b2k_chain_create and by the test oracle."""
        m = self.m
        d = {
            "isjoint": np.zeros(m, np.int32), "axis": np.zeros(m, np.int32), "flip": np.zeros(m, np.int32),
            "jindex": np.zeros(m, np.int32), "T": np.tile(np.eye(4), (m, 1, 1)), "qlim": np.zeros((m, 2)),
            "n": self.n,
        }
        for i, e in enumerate(self._ets):
            d["isjoint"][i] = int(e.isjoint)
            d["axis"][i] = AXES.get(e.axis, 0)
            d["flip"][i] = int(e.isflip)
            d["jindex"][i] = e.jindex if (e.isjoint and e.jindex is not None) else 0
            d["T"][i] = e.A() if not e.isjoint else np.eye(4)
            d["qlim"][i] = e._qlim_default()
        return d

    # ---- native handle
    def _update_internals(self):
        """Drop the compiled chain (call after mutating an ET's jindex / qlim); reference ETS.py:62-69."""
        self._release()
        ETS._frame_plans.clear()  # a cached fkine_all plan may have been derived from the old contents

    def _release(self):
        if getattr(self, "_handle", None):
            try:
                _lib.lib().b2k_chain_destroy(self._handle)
            except Exception:
                pass
        self._handle = None

    def __del__(self):
        self._release()

    @property
    def _chain(self):
        if self._handle is None:
            if self.n < 1:
                raise ValueError("the ETS has no joints; nothing to evaluate on the GPU")
            d = self.describe()
            h = _lib.vp()
            ip = _lib.ip
            T = np.ascontiguousarray(d["T"], dtype=np.float64)
            ql = np.ascontiguousarray(d["qlim"], dtype=np.float64)
            _lib.check(_lib.lib().b2k_chain_create(
                self.m, d["isjoint"].ctypes.data_as(ip), d["axis"].ctypes.data_as(ip),
                d["flip"].ctypes.data_as(ip), d["jindex"].ctypes.data_as(ip), _lib.dptr(T), _lib.dptr(ql),
                C.byref(h)))
            self._handle = h
            self._qwidth = int(max(self.jindices)) + 1
        return self._handle

    # ---- argument normalisation
    def _qbatch(self, q):
        """-> (q2d, single).  Shape rules of the reference's C layer (fknm.cpp:963-988): 1-D, (1,w)
        and (w,1) are ONE configuration, anything else is a trajectory of rows.  Deviation: for a
        1-joint chain an (N,1) array is N rows (the reference misreads it, SURVEY appendix C.1)."""
        B.check_numeric(q)
        nd = q.dim() if B.is_tensor(q) else np.ndim(q)
        if not B.is_tensor(q):
            q = np.asarray(q)
            if q.dtype not in (np.float32, np.float64):
                q = q.astype(np.float64)
        if nd == 0:
            q = q.reshape(1, 1)
            single = True
        elif nd == 1:
            q = q.reshape(1, -1)
            single = True
        elif nd == 2:
            r, c = q.shape
            if r == 1:
                single = True
            elif c == 1 and self.n > 1:
                q = q.reshape(1, -1)
                single = True
            else:
                single = False
        else:
            raise ValueError("q must be 1-D or 2-D")
        _ = self._chain
        if q.shape[1] < self._qwidth:
            raise ValueError(f"q has {q.shape[1]} columns but the ETS reads joint index {self._qwidth - 1}")
        if q.shape[1] > _lib.MAX_QWIDTH:
            raise ValueError(f"q rows wider than {_lib.MAX_QWIDTH} are not supported")
        return q, single

    # ------------------------------------------------------------------ forward kinematics
    def eval(self, q, base=None, tool=None, include_base: bool = True, dtype=None):
        """Forward kinematics as arrays: (4,4) for one q, (N,4,4) for an (N,n) batch
        (reference ETS.eval, ETS.py:1021-1078 -> fknm.ETS_fkine)."""
        q2, single = self._qbatch(q)
        dt = B.pick_dtype(q2, dtype)
        base = _mat44(base, "base") if include_base else None
        tool = _mat44(tool, "tool")
        L = _lib.lib()
        N = q2.shape[0]
        if not B.is_tensor(q2):
            t = B.require_cuda()
            qh = np.ascontiguousarray(q2, dtype=dt)
            T = _lib.host_result((N, 4, 4), dt)
            _lib.check(L.b2k_fkine_host(self._chain, B.code(dt), qh.ctypes.data, N, qh.shape[1], _lib.dptr(base),
                                        _lib.dptr(tool), T.ctypes.data, t.cuda.current_device()))
            return T[0] if single else T
        qd = B.to_device(q2, dt)
        T = B.empty((N, 4, 4), dt, like=qd)
        _lib.check(L.b2k_fkine(self._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(base), _lib.dptr(tool),
                               B.ptr(T), B.stream_ptr(qd)))
        return T[0] if single else T

    @staticmethod
    def eval_frames(chains, q, base=None, dtype=None):
        """Poses of several frames of one robot for the same q batch: ``chains[k]`` is the ETS from the robot's base to
        frame k + 1, frame 0 is the base itself.  Returns (K+1,4,4) for one configuration, (N,K+1,4,4) for a batch (a
        device tensor for device input, numpy for host input).  The chains are sorted into walks: a chain that is a
        prefix of a longer one is "the pose after its last joint times its constant tail" on the longer chain's walk,
        so a serial robot takes ONE launch for all of its frames and a branched one a launch per branch
        (``b2k_fkine_frames``); frames that depend on no joint are constants carried by the first launch.  The building
        block of ``fkine_all`` (reference Robot.fkine_all, Robot.py:638-700; DHRobot.fkine_all 1018-1064)."""
        if not chains:
            raise ValueError("no frames requested")
        jointed = [e for e in chains if e.n > 0]
        if not jointed:
            raise ValueError("none of the frames depends on a joint")
        widest = max(jointed, key=lambda e: int(max(e.jindices)))
        q2, single = widest._qbatch(q)
        dt = B.pick_dtype(q2, dtype)
        host = not B.is_tensor(q2)
        qd = B.to_device(q2, dt).contiguous()
        N = qd.shape[0]
        base = _mat44(base, "base")
        b0 = np.eye(4) if base is None else base
        if not ETS.frames_single_walk:
            # one pose launch per frame over the prefix chains into frame-major memory (each launch re-reads q and
            # re-walks its prefix); kept selectable for measurement
            frames = B.empty((len(chains) + 1, N, 4, 4), dt, like=qd)
            t = B.require_cuda()
            b0 = np.eye(4) if base is None else base
            frames[0] = t.as_tensor(b0, dtype=frames.dtype, device=frames.device)
            L = _lib.lib()
            for k, e in enumerate(chains):
                if e.n == 0:  # a static frame (a link before the first joint): base times the constant transforms
                    Tc = b0.copy()
                    for et in e:
                        Tc = Tc @ et.A()
                    frames[k + 1] = t.as_tensor(Tc, dtype=frames.dtype, device=frames.device)
                    continue
                _lib.check(L.b2k_fkine(e._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(base), None, B.ptr(frames[k + 1]),
                                       B.stream_ptr(qd)))
            out = frames.permute(1, 0, 2, 3)
            if host:
                out = np.ascontiguousarray(B.to_host(out.contiguous()))
            return out[0] if single else out
        K = len(chains)
        out = B.empty((N, K + 1, 4, 4), dt, like=qd)
        L = _lib.lib()
        for walk, after, slot, tails, nconst in ETS._frame_plan(chains):
            if nconst:  # the constants (base frame, links ahead of every joint) are expressed in the base frame
                tails = tails.copy()
                tails[:nconst] = b0 @ tails[:nconst]
            _lib.check(L.b2k_fkine_frames(walk._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(base), len(after),
                                          after.ctypes.data_as(_lib.ip), slot.ctypes.data_as(_lib.ip), _lib.dptr(tails),
                                          B.ptr(out), K + 1, B.stream_ptr(qd)))
        if host:
            out = B.to_host(out)
        return out[0] if single else out

    frames_single_walk = os.environ.get("B2K_FRAMES_SINGLE_WALK", "1") != "0"
    _frame_plans: dict = {}  # tuple(id(chain)) -> (the chains (kept alive: their ids stay theirs), launches)

    @staticmethod
    def _frame_plan(chains):
        """The launches of ``eval_frames`` for this list of chains, [(walk, after, slot, tails, nconst)], planned once
        per list of chain objects (a robot keeps its prefix chains; planning costs more host time than the launch)."""
        key = tuple(id(e) for e in chains)
        hit = ETS._frame_plans.get(key)
        if hit is not None:
            return hit[1]
        launches = []
        for walk, frames in ETS._frame_walks(chains):
            const = []
            if not launches:  # the constants ride on the first launch: the base frame and the links ahead of every joint
                const.append((0, -1, np.eye(4)))
                for k, e in enumerate(chains):
                    if e.n == 0:
                        Tc = np.eye(4)
                        for et in e:
                            Tc = Tc @ et.A()
                        const.append((k + 1, -1, Tc))
            frames = const + sorted(frames, key=lambda f: f[1])
            launches.append((walk, np.ascontiguousarray([f[1] for f in frames], dtype=np.int32),
                             np.ascontiguousarray([f[0] for f in frames], dtype=np.int32),
                             np.ascontiguousarray(np.stack([f[2] for f in frames]), dtype=np.float64), len(const)))
        if len(ETS._frame_plans) >= 32:
            ETS._frame_plans.pop(next(iter(ETS._frame_plans)))
        ETS._frame_plans[key] = (tuple(chains), launches)
        return launches

    @staticmethod
    def _frame_walks(chains):
        """Sort the jointed chains of ``eval_frames`` into walks: [(walk ETS, [(slot, after, tail 4x4), ...]), ...].  A
        chain belongs to the first longer chain it is a prefix of (same elementary transforms, joint indices and
        constants); ``after`` is the 0-based position of its last joint along the walk, ``tail`` the product of the
        constant transforms behind that joint."""
        descs = [e.describe() for e in chains]

        def is_prefix(k, w):
            m = chains[k].m
            if m > chains[w].m:
                return False
            dk, dw = descs[k], descs[w]
            return all(np.array_equal(dk[key][:m], dw[key][:m]) for key in ("isjoint", "axis", "flip", "jindex", "T"))

        walks = []  # [walk index, frames]
        for k in sorted((k for k, e in enumerate(chains) if e.n > 0), key=lambda k: -chains[k].m):
            owner = next((w for w in walks if is_prefix(k, w[0])), None)
            if owner is None:
                owner = [k, []]
                walks.append(owner)
            ets = list(chains[k])
            last = max(i for i, et in enumerate(ets) if et.isjoint)
            tail = np.eye(4)
            for et in ets[last + 1:]:
                tail = tail @ et.A()
            owner[1].append((k + 1, chains[k].n - 1, tail))
        return [(chains[w], fr) for w, fr in walks]

    def fkine(self, q, base=None, tool=None, include_base: bool = True, dtype=None) -> SE3:
        """Forward kinematics as an SE3 container (reference ETS.fkine, ETS.py:951-1019); one
        batched container instead of N Python objects."""
        T = self.eval(q, base, tool, include_base, dtype)
        return SE3(B.to_host(T) if B.is_tensor(T) else T)

    # ------------------------------------------------------------------ Jacobians
    def _jac(self, fn_name, q, tool, dtype):
        q2, single = self._qbatch(q)
        dt = B.pick_dtype(q2, dtype)
        tool = _mat44(tool, "tool")
        host = not B.is_tensor(q2)
        qd = B.to_device(q2, dt)
        N = qd.shape[0]
        J = B.empty((N, 6, self.n), dt, like=qd)
        fn = getattr(_lib.lib(), fn_name)
        _lib.check(fn(self._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(tool), B.ptr(J), B.stream_ptr(qd)))
        if host:
            J = B.to_host(J)
        return J[0] if single else J

    def jacob0(self, q, tool=None, dtype=None):
        """Geometric Jacobian in the start frame of the chain: (6,n) or (N,6,n)
        (reference ETS.jacob0, ETS.py:1143-1199 -> fknm.ETS_jacob0)."""
        return self._jac("b2k_jacob0", q, tool, dtype)

    def jacobe(self, q, tool=None, dtype=None):
        """Geometric Jacobian in the end-effector frame (reference ETS.jacobe, ETS.py:1268-1332)."""
        return self._jac("b2k_jacobe", q, tool, dtype)

    def fkine_jacob0(self, q, base=None, tool=None, include_base: bool = True, dtype=None):
        """Pose and base-frame Jacobian from ONE pass over q (extension; the reference needs
        ETS.eval + a Python loop of ETS.jacob0).  Returns (T, J)."""
        q2, single = self._qbatch(q)
        dt = B.pick_dtype(q2, dtype)
        base = _mat44(base, "base") if include_base else None
        tool = _mat44(tool, "tool")
        L = _lib.lib()
        N = q2.shape[0]
        n = self.n
        if not B.is_tensor(q2):
            t = B.require_cuda()
            qh = np.ascontiguousarray(q2, dtype=dt)
            T = _lib.host_result((N, 4, 4), dt)
            J = _lib.host_result((N, 6, n), dt)
            _lib.check(L.b2k_fkine_jacob0_host(self._chain, B.code(dt), qh.ctypes.data, N, qh.shape[1],
                                               _lib.dptr(base), _lib.dptr(tool), T.ctypes.data, J.ctypes.data,
                                               t.cuda.current_device()))
        else:
            qd = B.to_device(q2, dt)
            T = B.empty((N, 4, 4), dt, like=qd)
            J = B.empty((N, 6, n), dt, like=qd)
            _lib.check(L.b2k_fkine_jacob0(self._chain, B.code(dt), B.ptr(qd), N, qd.shape[1], _lib.dptr(base),
                                          _lib.dptr(tool), B.ptr(T), B.ptr(J), B.stream_ptr(qd)))
        return (T[0], J[0]) if single else (T, J)

    def fkine_jacob0_into(self, q, T, J, base=None, tool=None):
        """Zero-allocation host form of :meth:`fkine_jacob0`: q, T, J are caller-owned C-contiguous
        numpy arrays (ideally from ``pinned_empty``) of one dtype; results are written in place."""
        t = B.require_cuda()
        dt = q.dtype
        if T.dtype != dt or J.dtype != dt or dt not in (np.float32, np.float64):
            raise TypeError("q, T, J must share dtype float32 or float64")
        if not (q.flags.c_contiguous and T.flags.c_contiguous and J.flags.c_contiguous):
            raise ValueError("q, T, J must be C-contiguous")
        N = q.shape[0]
        if T.shape != (N, 4, 4) or J.shape != (N, 6, self.n):
            raise ValueError("T must be (N,4,4) and J (N,6,n)")
        _lib.check(_lib.lib().b2k_fkine_jacob0_host(
            self._chain, B.code(np.dtype(dt)), q.ctypes.data, N, q.shape[1], _lib.dptr(_mat44(base, "base")),
            _lib.dptr(_mat44(tool, "tool")), T.ctypes.data, J.ctypes.data, t.cuda.current_device()))

    # ------------------------------------------------------------------ functions of the Jacobian (SURVEY 8f-2)
    def _hess(self, q, J, tool, jac, dtype):
        if q is None and J is None:
            raise ValueError("one of q or the Jacobian must be supplied")
        if J is None:
            J = jac(q, tool=tool, dtype=dtype)
        host = not B.is_tensor(J)
        dt = B.pick_dtype(J, dtype)
        Jd = B.to_device(J, dt)
        single = Jd.dim() == 2
        Jd = (Jd.reshape(1, 6, -1) if single else Jd).contiguous()
        n = self.n
        if tuple(Jd.shape[1:]) != (6, n):
            raise ValueError(f"the Jacobian must be (6,{n}) or (N,6,{n})")
        N = Jd.shape[0]
        H = B.empty((N, n, 6, n), dt, like=Jd)
        _lib.check(_lib.lib().b2k_hessian(B.code(dt), n, B.ptr(Jd), N, B.ptr(H), B.stream_ptr(Jd)))
        if host:
            H = B.to_host(H)
        return H[0] if single else H

    def hessian0(self, q=None, J0=None, tool=None, dtype=None):
        """Manipulator Hessian in the base frame, (n,6,n) or (N,n,6,n), from q or from a given jacob0
        (reference ETS.hessian0, ETS.py:1334-1450 -> fknm.ETS_hessian0)."""
        return self._hess(q, J0, tool, self.jacob0, dtype)

    def hessiane(self, q=None, Je=None, tool=None, dtype=None):
        """Manipulator Hessian in the end-effector frame (reference ETS.hessiane, ETS.py:1452-1568)."""
        return self._hess(q, Je, tool, self.jacobe, dtype)

    def manipulability(self, q=None, J=None, method: str = "yoshikawa", axes="all", dtype=None):
        """Manipulability measure, scalar or (N,) (reference ETS.manipulability, ETS.py:1687-1820): "yoshikawa"
        sqrt|det(Ja Ja^T)|, "minsingular" the smallest singular value of Ja, "invcondition" 1 / cond(Ja); Ja = the
        rows of jacob0 selected by `axes`."""
        if method not in ("yoshikawa", "minsingular", "invcondition"):
            raise ValueError("Invalid method chosen")
        if isinstance(axes, str):
            mask = {"all": 63, "trans": 7, "rot": 56}.get(axes)
            if mask is None:
                raise ValueError("axes must be all, trans, rot or a 6-element bool list")
        else:
            ax = [bool(a) for a in axes]
            if len(ax) != 6:
                raise ValueError("axes must be all, trans, rot or a 6-element bool list")
            mask = sum(1 << k for k, a in enumerate(ax) if a)
        if q is None and J is None:
            raise ValueError("one of q or J must be supplied")
        if J is None:
            J = self.jacob0(q, dtype=dtype)
        Jd, dt, host, single = self._jprep(J, dtype)
        N = Jd.shape[0]
        m = B.empty((N,), dt, like=Jd)
        if method == "yoshikawa":
            _lib.check(_lib.lib().b2k_manipulability(B.code(dt), self.n, B.ptr(Jd), N, mask, B.ptr(m), B.stream_ptr(Jd)))
        else:
            _lib.check(_lib.lib().b2k_manipulability_svd(B.code(dt), self.n, B.ptr(Jd), N, mask, int(method == "invcondition"),
                                                         B.ptr(m), B.stream_ptr(Jd)))
        if host:
            m = B.to_host(m)
        return float(m[0]) if single else m

    @staticmethod
    def _axes_mask(axes):
        if isinstance(axes, str):
            mask = 63 if axes.startswith("all") else 7 if axes.startswith("trans") else 56 if axes.startswith("rot") else None
            if mask is None:
                raise ValueError("axes must be all, trans, rot or a 6-element bool list")
            return mask
        ax = [bool(a) for a in axes]
        if len(ax) != 6:
            raise ValueError("axes must be all, trans, rot or a 6-element bool list")
        return sum(1 << k for k, a in enumerate(ax) if a)

    def _jprep(self, J, dtype):
        host = not B.is_tensor(J)
        dt = B.pick_dtype(J, dtype)
        Jd = B.to_device(J, dt)
        single = Jd.dim() == 2
        Jd = (Jd.reshape(1, 6, -1) if single else Jd).contiguous()
        if tuple(Jd.shape[1:]) != (6, self.n):
            raise ValueError(f"the Jacobian must be (6,{self.n}) or (N,6,{self.n})")
        return Jd, dt, host, single

    def jacobm(self, q=None, J=None, H=None, axes="all", dtype=None):
        """Manipulability Jacobian dm/dq, (n,1) for one configuration like the reference, (N,n) for a batch
        (reference ETS.jacobm, ETS.py:1628-1685; Robot.jacobm with `axes`, Robot.py:1124-1232).  `H` is
        accepted for signature compatibility; the kernel forms the Hessian terms from J on the fly."""
        if q is None and J is None:
            raise ValueError("one of q or J must be supplied")
        if J is None:
            J = self.jacob0(q, dtype=dtype)
        elif not (B.is_tensor(J) or isinstance(J, np.ndarray)):
            raise TypeError("J must be an array")
        if H is not None and not (B.is_tensor(H) or isinstance(H, np.ndarray)):
            raise TypeError("Hessian must be numpy array of shape 6xnxn")
        mask = self._axes_mask(axes)
        Jd, dt, host, single = self._jprep(J, dtype)
        N = Jd.shape[0]
        Jm = B.empty((N, self.n), dt, like=Jd)
        _lib.check(_lib.lib().b2k_jacobm(B.code(dt), self.n, B.ptr(Jd), N, mask, B.ptr(Jm), B.stream_ptr(Jd)))
        if host:
            Jm = B.to_host(Jm)
        return Jm[0].reshape(self.n, 1) if single else Jm

    _REPRESENTATIONS = {"rpy/xyz": 0, "rpy/zyx": 1, "eul": 2, "exp": 3}

    def jacob0_analytical(self, q, representation: str = "rpy/xyz", tool=None, dtype=None):
        """Analytical Jacobian in the base frame, (6,n) or (N,6,n): blkdiag(I, A^-1(Gamma)) jacob0, which maps joint
        rates to the rates of the pose representation Gamma -- "rpy/xyz", "rpy/zyx", "eul" (ZYZ) or "exp"
        (reference ETS.jacob0_analytical, ETS.py:1570-1626 -> spatialmath rotvelxform(R, inverse=True, full=True)).
        Pose, Jacobian and the 3x3 rate transform are computed on the device in two launches."""
        if representation not in self._REPRESENTATIONS:
            raise ValueError(f"unknown representation {representation!r}; expecting one of {sorted(self._REPRESENTATIONS)}")
        q2, single = self._qbatch(q)
        dt = B.pick_dtype(q2, dtype)
        host = not B.is_tensor(q2)
        qd = B.to_device(q2, dt)
        T, J = self.fkine_jacob0(qd, tool=tool, include_base=False, dtype=dt)
        T, J = T.reshape(-1, 4, 4), J.reshape(-1, 6, self.n)
        N = J.shape[0]
        Ja = B.empty((N, 6, self.n), dt, like=J)
        _lib.check(_lib.lib().b2k_jacob0_analytical(B.code(dt), self.n, B.ptr(T), B.ptr(J), N, self._REPRESENTATIONS[representation],
                                                    B.ptr(Ja), B.stream_ptr(J)))
        if host:
            Ja = B.to_host(Ja)
        return Ja[0] if single else Ja

    def jacob0_dot(self, q=None, qd=None, J0=None, representation=None, dtype=None):
        """Time derivative of the base-frame Jacobian, (6,n) or (N,6,n): sum_i hessian0[i] qd[i]
        (reference Robot.jacob0_dot, Robot.py:964-1099).  With a ``representation`` the reference differentiates
        jacob0_analytical numerically (smb.numhess, Robot.py:1090-1092); here that is the central difference of
        the analytical Jacobian along the joint velocity, two device evaluations."""
        if representation is not None:
            if q is None or qd is None:
                raise ValueError("q and qd must be supplied")
            q2, single = self._qbatch(q)
            dt = B.pick_dtype(q2, dtype)
            host = not B.is_tensor(q2)
            qt = B.to_device(q2, dt)
            B.check_numeric(qd, "qd")
            vt = B.to_device(qd, dt).reshape(-1, self.n)
            if self._qwidth != self.n or qt.shape[1] != self.n:
                raise ValueError("analytical jacob0_dot needs q rows of exactly n joints")
            h = 1e-6 if dt == np.dtype(np.float64) else 1e-3
            out = (self.jacob0_analytical(qt + h * vt, representation, dtype=dt)
                   - self.jacob0_analytical(qt - h * vt, representation, dtype=dt)).reshape(-1, 6, self.n) / (2 * h)
            if host:
                out = B.to_host(out)
            return out[0] if single else out
        if qd is None or (q is None and J0 is None):
            raise ValueError("qd and one of q or J0 must be supplied")
        if J0 is None:
            J0 = self.jacob0(q, dtype=dtype)
        Jd, dt, host, single = self._jprep(J0, dtype)
        N = Jd.shape[0]
        B.check_numeric(qd, "qd")
        qdd = B.to_device(qd, dt).reshape(-1, self.n).contiguous()
        if qdd.shape[0] != N:
            raise ValueError(f"qd must have {N} rows of {self.n}")
        out = B.empty((N, 6, self.n), dt, like=Jd)
        _lib.check(_lib.lib().b2k_jacob_dot(B.code(dt), self.n, B.ptr(Jd), B.ptr(qdd), N, B.ptr(out), B.stream_ptr(Jd)))
        if host:
            out = B.to_host(out)
        return out[0] if single else out

    # ------------------------------------------------------------------ inverse kinematics
    def _ik(self, Tep, q0, ilimit, slimit, tol, mask, joint_limits, k, method, seed, semantics, rng_per_row, dtype,
            null=None):
        Tep = getattr(Tep, "A", Tep)
        B.check_numeric(Tep, "Tep")
        host = not B.is_tensor(Tep)
        dt = B.pick_dtype(Tep, dtype)
        Td = B.to_device(Tep, dt)
        if Td.dim() == 2:
            if tuple(Td.shape) != (4, 4):
                raise ValueError("Tep must be a 4x4 SE3 matrix")
            Td = Td.reshape(1, 4, 4)
            single = True
        elif Td.dim() == 3 and tuple(Td.shape[1:]) == (4, 4):
            single = False
        else:
            raise ValueError("Tep must be (4,4) or (N,4,4)")
        N = Td.shape[0]
        n = self.n
        q0d = None
        if q0 is not None:
            B.check_numeric(q0, "q0")
            q0d = B.to_device(q0, dt)
            if q0d.numel() == n:
                q0d = q0d.reshape(1, n).expand(N, n).contiguous()
            elif tuple(q0d.shape) != (N, n):
                raise ValueError(f"q0 must have {n} elements or shape ({N},{n})")
        we = None if mask is None else np.ascontiguousarray(np.asarray(mask, dtype=np.float64).reshape(6))
        if isinstance(method, int):
            meth = method  # _lib.IK_NR / _lib.IK_GN
        else:
            m = str(method).lower()
            meth = 2 if m.startswith("s") else (1 if m.startswith("w") else 0)  # fknm.cpp:481-495: 's', 'w', else chan
        q = B.empty((N, n), dt, like=Td)
        succ = B.empty_i32((N,), like=Td)
        its = B.empty_i32((N,), like=Td)
        srch = B.empty_i32((N,), like=Td)
        E = B.empty((N,), dt, like=Td)
        if seed is None:
            seed = int(np.random.default_rng().integers(0, 2**63 - 1))
        if null is None:
            _lib.check(_lib.lib().b2k_ik_lm(
                self._chain, B.code(dt), B.ptr(Td), N, B.ptr(q0d), int(ilimit), int(slimit), float(tol),
                int(bool(joint_limits)), _lib.dptr(we), float(k), meth, int(seed) & (2**64 - 1), semantics,
                int(bool(rng_per_row)), B.ptr(q), B.ptr(succ), B.ptr(its), B.ptr(srch), B.ptr(E), B.stream_ptr(Td)))
        else:  # the Python loop with the null-space terms (semantics is SEM_PYTHON)
            kq, km, ps, pi = null
            _lib.check(_lib.lib().b2k_ikine_null(
                self._chain, B.code(dt), B.ptr(Td), N, B.ptr(q0d), int(ilimit), int(slimit), float(tol),
                int(bool(joint_limits)), _lib.dptr(we), float(k), meth, int(seed) & (2**64 - 1),
                int(bool(rng_per_row)), float(kq), float(km), float(ps), _lib.dptr(pi), B.ptr(q), B.ptr(succ),
                B.ptr(its), B.ptr(srch), B.ptr(E), B.stream_ptr(Td)))
        if host:
            q, succ, its, srch, E = (B.to_host(x) for x in (q, succ, its, srch, E))
        return q, succ, its, srch, E, single

    def ik_LM(self, Tep, q0=None, ilimit: int = 30, slimit: int = 100, tol: float = 1e-6, mask=None,
              joint_limits: bool = True, k: float = 1.0, method: str = "chan", seed: Optional[int] = 0, dtype=None):
        """Levenberg-Marquardt IK with the semantics of the reference's C++ solver
        (ETS.ik_LM, ETS.py:2014-2170 -> fknm.IK_LM_c).  One target (4,4) returns the reference's tuple
        ``(q, success, iterations, searches, residual)``; an (N,4,4) batch returns the same tuple of
        arrays, row i being the reference called on target i."""
        q, s, it, sr, E, single = self._ik(Tep, q0, ilimit, slimit, tol, mask, joint_limits, k, method, seed,
                                           _lib.SEM_CPP, True, dtype)
        if single:
            return q[0], int(s[0]), int(it[0]), int(sr[0]), float(E[0])
        return q, s, it, sr, E

    def _ik_tuple(self, r):
        q, s, it, sr, E, single = r
        if single:
            return q[0], int(s[0]), int(it[0]), int(sr[0]), float(E[0])
        return q, s, it, sr, E

    def ik_NR(self, Tep, q0=None, ilimit: int = 30, slimit: int = 100, tol: float = 1e-6, mask=None,
              joint_limits: bool = True, pinv: int = True, pinv_damping: float = 0.0, seed: Optional[int] = 0,
              dtype=None):
        """Newton-Raphson IK with the semantics of the reference's C++ solver (ETS.ik_NR,
        ETS.py:2172-2298 -> fknm.IK_NR_c -> _IK_NR ik.cpp:121-155): dq = pinv_d(J) e.  Same return
        convention as :meth:`ik_LM`.  ``pinv=False`` (J.inverse() e, square chains only in the reference)
        yields the same step wherever J is invertible and is not a separate code path."""
        return self._ik_tuple(self._ik(Tep, q0, ilimit, slimit, tol, mask, joint_limits, pinv_damping, _lib.IK_NR,
                                       seed, _lib.SEM_CPP, True, dtype))

    def ik_GN(self, Tep, q0=None, ilimit: int = 30, slimit: int = 100, tol: float = 1e-6, mask=None,
              joint_limits: bool = True, pinv: int = True, pinv_damping: float = 0.0, seed: Optional[int] = 0,
              dtype=None):
        """Gauss-Newton IK with the semantics of the reference's C++ solver (ETS.ik_GN,
        ETS.py:2300-2430 -> fknm.IK_GN_c -> _IK_GN ik.cpp:79-119): the minimum-norm solution of
        (J^T We J) dq = J^T We e.  ``pinv_damping`` is accepted and ignored, as in the reference."""
        return self._ik_tuple(self._ik(Tep, q0, ilimit, slimit, tol, mask, joint_limits, 0.0, _lib.IK_GN,
                                       seed, _lib.SEM_CPP, True, dtype))

    def _null_args(self, kq, km, ps, pi):
        """(kq, km, ps, pi as an n-vector) for b2k_ikine_null, or None when neither null-space term is on.
        The terms of the reference's _calc_qnull run only for a gain > 0; on a chain of n <= 6 joints a full-rank J
        has no null space, and the terms are accepted (their arguments still checked) and ignored (DESIGN (f-7))."""
        kq, km = float(kq), float(km)
        if not (kq > 0 or km > 0):
            return None
        n = self.n
        pa = np.asarray(pi, dtype=np.float64)
        if pa.ndim == 0:
            pa = np.full(n, float(pa))
        elif pa.shape != (n,):
            raise ValueError(f"pi must be a scalar or have {n} elements, got shape {pa.shape}")
        pa = np.ascontiguousarray(pa)
        ps = float(ps)
        if not (np.isfinite(kq) and np.isfinite(km) and np.isfinite(ps) and np.isfinite(pa).all()):
            raise ValueError("kq, km, ps and pi must be finite")
        if kq > 0 and (pa == ps).any():
            raise ValueError(f"ps == pi at joint {int(np.argmax(pa == ps))}: the joint-limit term divides by ps - pi")
        if n < 7:
            return None
        return kq, km, ps, pa

    def _ikine(self, meth, Tep, q0, ilimit, slimit, tol, mask, joint_limits, seed, k, kq, km, dtype, ps=0.0,
               pi=0.3) -> IKSolution:
        q, s, it, sr, E, single = self._ik(Tep, q0, ilimit, slimit, tol, mask, joint_limits, k, meth, seed,
                                           _lib.SEM_PYTHON, False, dtype, null=self._null_args(kq, km, ps, pi))
        if B.is_tensor(q):
            q, s, it, sr, E = (B.to_host(x) for x in (q, s, it, sr, E))
        fail = "iteration and search limit reached"
        if single:
            ok = bool(s[0])
            return IKSolution(q=q[0], success=ok, iterations=int(it[0]), searches=int(sr[0]),
                              residual=float(E[0]), reason="Success" if ok else fail)
        ok = bool(s.all())
        return IKSolution(q=q, success=ok, iterations=int(it.sum()), searches=int(sr.sum()),
                          residual=float(E.min()), reason="" if ok else fail)

    def ikine_NR(self, Tep, q0=None, ilimit: int = 30, slimit: int = 100, tol: float = 1e-6, mask=None,
                 joint_limits: bool = True, seed: Optional[int] = None, pinv: bool = False, kq: float = 0.0,
                 km: float = 0.0, ps: float = 0.0, pi=0.3, dtype=None, **kwargs) -> IKSolution:
        """Newton-Raphson IK with the semantics of the reference's Python solver class (ETS.ikine_NR,
        ETS.py:2639-2776 -> IK_NR, IK.py:579-762: q += pinv(J) e or inv(J) e -- the same vector)."""
        return self._ikine(_lib.IK_NR, Tep, q0, ilimit, slimit, tol, mask, joint_limits, seed, 0.0, kq, km, dtype,
                           ps, pi)

    def ikine_GN(self, Tep, q0=None, ilimit: int = 30, slimit: int = 100, tol: float = 1e-6, mask=None,
                 joint_limits: bool = True, seed: Optional[int] = None, pinv: bool = False, kq: float = 0.0,
                 km: float = 0.0, ps: float = 0.0, pi=0.3, dtype=None, **kwargs) -> IKSolution:
        """Gauss-Newton IK with the semantics of the reference's Python solver class (ETS.ikine_GN,
        ETS.py:2778-2930 -> IK_GN, IK.py:1020-1219; its step is also q += pinv(J) e, IK.py:1214-1217)."""
        return self._ikine(_lib.IK_NR, Tep, q0, ilimit, slimit, tol, mask, joint_limits, seed, 0.0, kq, km, dtype,
                           ps, pi)

    def ikine_LM(self, Tep, q0=None, ilimit: int = 30, slimit: int = 100, tol: float = 1e-6, mask=None,
                 joint_limits: bool = True, seed: Optional[int] = None, k: float = 1.0, method: str = "chan",
                 kq: float = 0.0, km: float = 0.0, ps: float = 0.0, pi=0.3, dtype=None, **kwargs) -> IKSolution:
        """Levenberg-Marquardt IK with the semantics of the reference's Python solver class
        (ETS.ikine_LM, ETS.py:2443-2637 -> IK_LM.solve, IK.py:174-367, 912-1017): returns an
        :class:`IKSolution`; for an (N,4,4) trajectory q is (N,n), success is the conjunction,
        iterations / searches are summed and residual is the minimum (IK.py:263-290)."""
        return self._ikine(method, Tep, q0, ilimit, slimit, tol, mask, joint_limits, seed, k, kq, km, dtype, ps, pi)
