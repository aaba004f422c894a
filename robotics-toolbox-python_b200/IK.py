"""IK result container and solver class with the reference's names
(reference src/roboticstoolbox/robot/IK.py:24-101 IKSolution, 765-1017 IK_LM)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np


@dataclass
class IKSolution:
    """Same fields, order and iteration protocol as the reference dataclass (IK.py:24-68)."""

    q: np.ndarray
    success: bool
    iterations: int = 0
    searches: int = 0
    residual: float = 0.0
    reason: str = ""

    def __iter__(self):
        return iter((self.q, self.success, self.iterations, self.searches, self.residual, self.reason))

    def __str__(self):
        q = None if self.q is None else np.array2string(
            np.asarray(self.q), separator=", ",
            formatter={"float": lambda x: "{:.4g}".format(0 if abs(x) < 1e-6 else x)})
        if self.success:
            return (f"IKSolution: q={q}, success=True, iterations={self.iterations}, "
                    f"searches={self.searches}, residual={self.residual:.3g}")
        return (f"IKSolution: q={q}, success=False, reason={self.reason}, iterations={self.iterations}, "
                f"searches={self.searches}, residual={self.residual:.3g}")


class IK_LM:
    """Levenberg-Marquardt solver object (reference IK.py:765-1017).  ``solve(ets, Tep, q0)`` runs
    the fused GPU kernel with the Python solver's semantics (step, then test the pre-step error)."""

    def __init__(self, name: str = "IK Solver", ilimit: int = 30, slimit: int = 100, tol: float = 1e-6,
                 mask=None, joint_limits: bool = True, seed: Optional[int] = None, k: float = 1.0,
                 method: str = "chan", kq: float = 0.0, km: float = 0.0, ps: float = 0.0, pi=0.3, **kwargs):
        self.ilimit, self.slimit, self.tol = ilimit, slimit, tol
        self.mask = mask
        self.We = np.diag(np.ones(6) if mask is None else np.asarray(mask, dtype=float))
        self.joint_limits = joint_limits
        self.seed = seed
        self.k = k
        m = method.lower()
        self.method = "sugihara" if m.startswith("sugi") else ("wampler" if m.startswith("wamp") else "chan")
        self.kq, self.km, self.ps, self.pi = kq, km, ps, pi
        self.name = f"LM ({self.method.capitalize()} λ={k})"

    def solve(self, ets, Tep, q0=None) -> IKSolution:
        ets = ets.ets() if hasattr(ets, "ets") and callable(ets.ets) else ets
        return ets.ikine_LM(Tep, q0=q0, ilimit=self.ilimit, slimit=self.slimit, tol=self.tol, mask=self.mask,
                            joint_limits=self.joint_limits, seed=self.seed, k=self.k, method=self.method,
                            kq=self.kq, km=self.km, ps=self.ps, pi=self.pi)


class _IK_pinv:
    def __init__(self, name: str = "IK Solver", ilimit: int = 30, slimit: int = 100, tol: float = 1e-6,
                 mask=None, joint_limits: bool = True, seed: Optional[int] = None, pinv: bool = False,
                 kq: float = 0.0, km: float = 0.0, ps: float = 0.0, pi=0.3, **kwargs):
        self.ilimit, self.slimit, self.tol = ilimit, slimit, tol
        self.mask = mask
        self.We = np.diag(np.ones(6) if mask is None else np.asarray(mask, dtype=float))
        self.joint_limits = joint_limits
        self.seed = seed
        self.pinv = pinv
        self.kq, self.km, self.ps, self.pi = kq, km, ps, pi
        self.name = f"{self._tag} (pinv={pinv})"

    def _args(self):
        return dict(ilimit=self.ilimit, slimit=self.slimit, tol=self.tol, mask=self.mask,
                    joint_limits=self.joint_limits, seed=self.seed, pinv=self.pinv, kq=self.kq, km=self.km,
                    ps=self.ps, pi=self.pi)


class IK_NR(_IK_pinv):
    """Newton-Raphson solver object (reference IK.py:579-762); ``solve`` runs the fused GPU kernel."""
    _tag = "NR"

    def solve(self, ets, Tep, q0=None) -> IKSolution:
        ets = ets.ets() if hasattr(ets, "ets") and callable(ets.ets) else ets
        return ets.ikine_NR(Tep, q0=q0, **self._args())


class IK_GN(_IK_pinv):
    """Gauss-Newton solver object (reference IK.py:1020-1219); ``solve`` runs the fused GPU kernel."""
    _tag = "GN"

    def solve(self, ets, Tep, q0=None) -> IKSolution:
        ets = ets.ets() if hasattr(ets, "ets") and callable(ets.ets) else ets
        return ets.ikine_GN(Tep, q0=q0, **self._args())


class IK_QP:
    """Quadratic-programming solver object (reference IK_QP, IK.py); ``solve`` runs the fused GPU kernel, each step's
    QP solved exactly on the device (DESIGN (f-11))."""

    def __init__(self, name: str = "IK Solver", ilimit: int = 30, slimit: int = 100, tol: float = 1e-6,
                 mask=None, joint_limits: bool = True, seed: Optional[int] = None, kj: float = 1.0, ks: float = 1.0,
                 kq: float = 0.0, km: float = 0.0, ps: float = 0.0, pi=0.3, **kwargs):
        self.ilimit, self.slimit, self.tol = ilimit, slimit, tol
        self.mask = mask
        self.We = np.diag(np.ones(6) if mask is None else np.asarray(mask, dtype=float))
        self.joint_limits = joint_limits
        self.seed = seed
        self.kj, self.ks = kj, ks
        self.kq, self.km, self.ps, self.pi = kq, km, ps, pi
        self.name = f"QP (kj={kj}, ks={ks})"

    def solve(self, ets, Tep, q0=None) -> IKSolution:
        ets = ets.ets() if hasattr(ets, "ets") and callable(ets.ets) else ets
        return ets.ikine_QP(Tep, q0=q0, ilimit=self.ilimit, slimit=self.slimit, tol=self.tol, mask=self.mask,
                            joint_limits=self.joint_limits, seed=self.seed, kj=self.kj, ks=self.ks, kq=self.kq,
                            km=self.km, ps=self.ps, pi=self.pi)
