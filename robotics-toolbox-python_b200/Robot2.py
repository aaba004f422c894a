"""Planar serial robots: ``Robot2`` and ``Link2`` (reference Robot2 / Link2, robot/Robot.py and robot/Link.py), whose
kinematics delegate to :class:`ETS2` with the robot's base and tool.  Branched 2-D trees (the reference's
``models.ETS.Planar_Y``) are not supported."""
from __future__ import annotations

from typing import List, Optional, Union

import numpy as np

from ._se3 import SE2
from .ET import ET2
from .ETS import ETS2, _mat33
from .Robot import Link


class Link2(Link):
    """A planar link: an ETS2 ending in at most one joint, hanging off a parent link."""

    def __init__(self, ets=None, name: Optional[str] = None, parent: Union["Link2", str, None] = None,
                 jindex: Optional[int] = None, qlim=None, **kwargs):
        if ets is None:
            ets = ETS2()
        elif isinstance(ets, ET2):
            ets = ETS2(ets)
        elif not isinstance(ets, ETS2):
            raise TypeError("The ets argument must be of type ETS2 or ET2")
        super().__init__(ets, name=name, parent=parent, jindex=jindex, qlim=qlim)

    def A(self, q: float = 0.0) -> np.ndarray:
        """link transform (3x3) at joint coordinate q"""
        T = np.eye(3)
        for et in self.ets:
            T = T @ (et.A(q) if et.isjoint else et.A())
        return T


class Robot2:
    """A planar serial robot, from an ETS2 or from a list of Link2 forming one chain."""

    def __init__(self, arg, name: str = "", base=None, tool=None, **kwargs):
        if isinstance(arg, ETS2):
            ets = ETS2(arg)
        elif isinstance(arg, (list, tuple)) and arg and all(isinstance(l, Link2) for l in arg):
            ets = self._chain_of(list(arg))
        else:
            raise TypeError("arg must be an ETS2 or a list of Link2")
        if ets.n < 1:
            raise ValueError("a Robot2 needs at least one joint")
        self._ets = ets
        self.name = name
        self.base = base
        self.tool = tool
        self._configs = {}
        self.addconfiguration("qz", np.zeros(self.n))
        self.addconfiguration("qr", np.zeros(self.n))

    @staticmethod
    def _chain_of(links: List[Link2]) -> ETS2:
        """The links in chain order (parents by reference or name; none given = list order) -> one ETS2."""
        byname = {l.name: l for l in links if l.name}
        for l in links:
            if l.parent is None and l.parent_name is not None:
                if l.parent_name not in byname:
                    raise ValueError(f"link {l.name}: unknown parent {l.parent_name}")
                l.parent = byname[l.parent_name]
        if all(l.parent is None for l in links):
            parent = {id(b): a for a, b in zip(links, links[1:])}
        else:
            parent = {id(l): l.parent for l in links if l.parent is not None}
        children = {}
        for l in links:
            p = parent.get(id(l))
            if p is not None:
                if not any(p is m for m in links):
                    raise ValueError(f"the parent of link {l.name} is not a link of this robot")
                children.setdefault(id(p), []).append(l)
        for l in links:
            if len(children.get(id(l), [])) > 1:
                raise ValueError(f"link {l.name!r} has {len(children[id(l)])} children: Robot2 is a serial chain, "
                                 "branched 2-D trees are not supported")
        roots = [l for l in links if id(l) not in parent]
        if len(roots) != 1:
            raise ValueError("Multiple base links" if roots else "Invalid link configuration provided, must have a base link")
        order, cur = [], roots[0]
        while cur is not None:
            order.append(cur)
            nxt = children.get(id(cur), [])
            cur = nxt[0] if nxt else None
        parts = []
        for l in order:
            e = l.ets
            if l.isjoint and l.jindex is not None and e[-1].jindex != l.jindex:
                ets = [et.copy() for et in e]
                ets[-1].jindex = l.jindex
                e = ETS2(ets)
            parts.append(e)
        return ETS2.from_links(parts)

    # ---- structure
    @property
    def n(self) -> int:
        return self._ets.n

    @property
    def qlim(self) -> np.ndarray:
        return self._ets.qlim

    @property
    def base(self) -> SE2:
        return SE2(self._base)

    @base.setter
    def base(self, T):
        self._base = np.eye(3) if T is None else _mat33(T, "base")

    @property
    def tool(self) -> SE2:
        return SE2(self._tool)

    @tool.setter
    def tool(self, T):
        self._tool = np.eye(3) if T is None else _mat33(T, "tool")

    def ets(self) -> ETS2:
        return self._ets

    def addconfiguration(self, name, q):
        self._configs[name] = np.asarray(q, dtype=np.float64)
        setattr(self, name, self._configs[name])

    # ---- kinematics: base and tool default to the robot's
    def _bt(self, base, tool):
        return (self._base if base is None else base), (self._tool if tool is None else tool)

    def eval(self, q, base=None, tool=None, include_base: bool = True, dtype=None):
        b, t = self._bt(base, tool)
        return self._ets.eval(q, b, t, include_base, dtype)

    def fkine(self, q, base=None, tool=None, include_base: bool = True, dtype=None) -> SE2:
        b, t = self._bt(base, tool)
        return self._ets.fkine(q, b, t, include_base, dtype)

    def jacob0(self, q, tool=None, dtype=None):
        return self._ets.jacob0(q, self._bt(None, tool)[1], dtype)

    def jacobe(self, q, tool=None, dtype=None):
        return self._ets.jacobe(q, self._bt(None, tool)[1], dtype)

    def fkine_jacob0(self, q, base=None, tool=None, include_base: bool = True, dtype=None):
        b, t = self._bt(base, tool)
        return self._ets.fkine_jacob0(q, b, t, include_base, dtype)

    def __repr__(self):
        return f"Robot2({self.name!r}, n={self.n}): {self._ets}"
