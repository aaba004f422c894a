"""Elementary transforms -- host-side description only.

Mirrors the constructor surface of the reference's ``ET`` (reference
src/roboticstoolbox/robot/ET.py:24-125 and the class methods at 610-900): ``ET.Rx/Ry/Rz/tx/ty/tz``
with ``eta=None`` meaning a variable joint, ``flip``, ``jindex``, ``qlim``, plus ``ET.SE3`` for a
constant 4x4.  An ET here owns no native object; an :class:`ETS` flattens its ETs into the
description that ``b2k_chain_create`` compiles (include/b2kin.h).  :class:`ET2` is the planar counterpart
(reference ET2: ``ET2.R/tx/ty/SE2``), described to the chain compiler through its 3-D embedding.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np

AXES = {"Rx": 0, "Ry": 1, "Rz": 2, "tx": 3, "ty": 4, "tz": 5}  # reference ET.py:244-266


def _rotx(t):
    c, s = math.cos(t), math.sin(t)
    return np.array([[1, 0, 0, 0], [0, c, -s, 0], [0, s, c, 0], [0, 0, 0, 1.0]])


def _roty(t):
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1.0]])


def _rotz(t):
    c, s = math.cos(t), math.sin(t)
    return np.array([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])


def _tr(x, y, z):
    T = np.eye(4)
    T[:3, 3] = (x, y, z)
    return T


_FUNCS = {
    "Rx": _rotx, "Ry": _roty, "Rz": _rotz,
    "tx": lambda e: _tr(e, 0, 0), "ty": lambda e: _tr(0, e, 0), "tz": lambda e: _tr(0, 0, e),
}


class ET:
    """One elementary transform: a constant SE(3) or a single-axis joint (reference ET.py:24-93)."""

    def __init__(self, axis: str, eta=None, T: Optional[np.ndarray] = None, jindex: Optional[int] = None,
                 unit: str = "rad", flip: bool = False, qlim=None):
        if axis not in AXES and axis != "SE3":
            raise ValueError(f"unknown ET axis {axis!r}")
        self._axis = axis
        if eta is not None and not isinstance(eta, (int, float, np.integer, np.floating)):
            # the reference falls back to sympy here (ETS.py:1077-1141); there is no symbolic GPU path
            raise TypeError("Symbolic value")
        if eta is not None and axis[0] == "R" and unit.lower().startswith("deg"):
            eta = math.radians(float(eta))
        self._eta = None if eta is None else float(eta)
        self._flip = bool(flip)
        self._jindex = jindex
        self._qlim = None if qlim is None else np.asarray(qlim, dtype=np.float64).reshape(2)
        if self._eta is None and T is None:
            if axis == "SE3":
                raise TypeError("ET.SE3 needs a constant matrix")
            self._joint = True
            self._T = np.eye(4)
        elif T is not None:
            self._joint = False
            self._T = np.array(T, dtype=np.float64).reshape(4, 4)
        else:
            self._joint = False
            self._T = _FUNCS[axis](self._eta)

    # ---- constructors, reference ET.py:610-900
    @classmethod
    def Rx(cls, eta=None, unit="rad", **kw):
        return cls("Rx", eta=eta, unit=unit, **kw)

    @classmethod
    def Ry(cls, eta=None, unit="rad", **kw):
        return cls("Ry", eta=eta, unit=unit, **kw)

    @classmethod
    def Rz(cls, eta=None, unit="rad", **kw):
        return cls("Rz", eta=eta, unit=unit, **kw)

    @classmethod
    def tx(cls, eta=None, **kw):
        return cls("tx", eta=eta, **kw)

    @classmethod
    def ty(cls, eta=None, **kw):
        return cls("ty", eta=eta, **kw)

    @classmethod
    def tz(cls, eta=None, **kw):
        return cls("tz", eta=eta, **kw)

    @classmethod
    def SE3(cls, T, **kw):
        T = getattr(T, "A", T)
        return cls("SE3", T=np.asarray(T, dtype=np.float64), **kw)

    # ---- properties, reference ET.py:240-520
    @property
    def axis(self) -> str:
        return self._axis

    @property
    def eta(self):
        return self._eta

    @property
    def isjoint(self) -> bool:
        return self._joint

    @property
    def isflip(self) -> bool:
        return self._flip

    @property
    def isrotation(self) -> bool:
        return self._axis[0] == "R"

    @property
    def istranslation(self) -> bool:
        return self._axis[0] == "t"

    @property
    def jindex(self):
        return self._jindex

    @jindex.setter
    def jindex(self, j):
        if not self.isjoint:
            raise ValueError("jindex is not valid for a static ET")
        self._jindex = j

    @property
    def qlim(self):
        return self._qlim

    @qlim.setter
    def qlim(self, v):
        self._qlim = None if v is None else np.asarray(v, dtype=np.float64).reshape(2)

    def _qlim_default(self):
        """The limits the reference hands its C struct (ET.py:109-115)."""
        if self._qlim is not None:
            return self._qlim
        return np.array([-math.pi, math.pi]) if self._axis[0] == "R" else np.array([0.0, 1.0])

    def A(self, q: float = 0.0) -> np.ndarray:
        """The 4x4 of this ET at joint coordinate q (reference ET.py:565-579).  Description-level
        helper for a SINGLE transform; batches go through ETS.eval on the GPU."""
        if not self._joint:
            return self._T.copy()
        q = -float(q) if self._flip else float(q)
        return _FUNCS[self._axis](q)

    A3 = A  # the 4x4 the chain compiler takes (ET2 embeds its 3x3 here)

    def _axis_code(self) -> int:
        """axis code of the chain description (B2K_RX..B2K_TZ; constants 0)"""
        return AXES.get(self._axis, 0)

    def copy(self) -> "ET":
        e = ET.__new__(ET)
        e.__dict__.update(self.__dict__)
        e._T = self._T.copy()
        e._qlim = None if self._qlim is None else self._qlim.copy()
        return e

    def inv(self) -> "ET":
        """Inverse of this ET (reference ET.inv, ET.py:506-539): a joint moves the other way (flip toggled), a
        constant gets the inverse matrix (and -eta)."""
        e = self.copy()
        if e._joint:
            e._flip = not e._flip
        else:
            e._T = np.linalg.inv(e._T)
            if e._eta is not None:
                e._eta = -e._eta
        return e

    def __mul__(self, other):
        from .ETS import ETS
        return ETS([self]) * other

    __add__ = __mul__

    def __repr__(self):
        if self._joint:
            j = "" if self._jindex is None else str(self._jindex)
            s = f"{self._axis}({'-' if self._flip else ''}q{j})"
        elif self._axis in ("SE3", "SE2"):
            s = f"{self._axis}(...)"
        elif self._axis[0] == "R":
            s = f"{self._axis}({math.degrees(self._eta):.4g}°)"
        else:
            s = f"{self._axis}({self._eta:.4g})"
        return s


# planar transforms: axis -> the 3-D axis code of the embedding (R acts as Rz)
AXES2 = {"R": AXES["Rz"], "tx": AXES["tx"], "ty": AXES["ty"]}


def _se2(c, s, x, y):
    return np.array([[c, -s, x], [s, c, y], [0, 0, 1.0]])


_FUNCS2 = {
    "R": lambda e: _se2(math.cos(e), math.sin(e), 0, 0),
    "tx": lambda e: _se2(1, 0, e, 0), "ty": lambda e: _se2(1, 0, 0, e),
}


def se2_to_se3(T):
    """The SE(3) matrix that acts in the xy plane as the 3x3 SE(2) matrix T does (z row and column of the identity)."""
    T = np.asarray(T, dtype=np.float64)
    A = np.eye(4)
    A[:2, :2] = T[:2, :2]
    A[:2, 3] = T[:2, 2]
    return A


class ET2(ET):
    """One planar elementary transform (reference ET2, ET.py): a constant SE(2) or a joint R (rotation about the
    normal of the plane), tx or ty.  It embeds into 3-D as Rz / tx / ty / an SE3 acting in the xy plane, which is
    how an :class:`ETS2` reaches the chain compiler."""

    def __init__(self, axis: str, eta=None, T: Optional[np.ndarray] = None, jindex: Optional[int] = None,
                 unit: str = "rad", flip: bool = False, qlim=None):
        if axis not in AXES2 and axis != "SE2":
            raise ValueError(f"unknown ET2 axis {axis!r}")
        self._axis = axis
        if eta is not None and not isinstance(eta, (int, float, np.integer, np.floating)):
            raise TypeError("Symbolic value")
        if eta is not None and axis == "R" and unit.lower().startswith("deg"):
            eta = math.radians(float(eta))
        self._eta = None if eta is None else float(eta)
        self._flip = bool(flip)
        self._jindex = jindex
        self._qlim = None if qlim is None else np.asarray(qlim, dtype=np.float64).reshape(2)
        if self._eta is None and T is None:
            if axis == "SE2":
                raise TypeError("ET2.SE2 needs a constant matrix")
            self._joint = True
            self._T = np.eye(3)
        elif T is not None:
            T = np.array(T, dtype=np.float64)
            if T.shape != (3, 3) or not np.array_equal(T[2], [0.0, 0.0, 1.0]):
                raise ValueError("ET2.SE2 needs a 3x3 SE(2) matrix (bottom row 0 0 1)")
            self._joint = False
            self._T = T
        else:
            self._joint = False
            self._T = _FUNCS2[axis](self._eta)

    @classmethod
    def R(cls, eta=None, unit="rad", **kw):
        return cls("R", eta=eta, unit=unit, **kw)

    @classmethod
    def tx(cls, eta=None, **kw):
        return cls("tx", eta=eta, **kw)

    @classmethod
    def ty(cls, eta=None, **kw):
        return cls("ty", eta=eta, **kw)

    @classmethod
    def SE2(cls, T, **kw):
        return cls("SE2", T=getattr(T, "A", T), **kw)

    def A(self, q: float = 0.0) -> np.ndarray:
        """The 3x3 of this ET2 at joint coordinate q."""
        if not self._joint:
            return self._T.copy()
        return _FUNCS2[self._axis](-float(q) if self._flip else float(q))

    def A3(self, q: float = 0.0) -> np.ndarray:
        """The 4x4 of the 3-D embedding at joint coordinate q."""
        return se2_to_se3(self.A(q))

    def _axis_code(self) -> int:
        return AXES2.get(self._axis, 0)

    def copy(self) -> "ET2":
        e = ET2.__new__(ET2)
        e.__dict__.update(self.__dict__)
        e._T = self._T.copy()
        e._qlim = None if self._qlim is None else self._qlim.copy()
        return e

    def __mul__(self, other):
        from .ETS import ETS2
        return ETS2([self]) * other

    __add__ = __mul__
