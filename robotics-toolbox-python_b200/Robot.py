"""ETS-based robots as rigid-body trees: the delegations of the reference's RobotKinematicsMixin
(reference src/roboticstoolbox/robot/RobotKinematics.py:28-97 fkine, 158 jacob0, 219 jacobe, 736-746 ik_LM,
1209-1226 ikine_LM) over the chain ``BaseRobot.ets(start, end)`` extracts from a link tree
(BaseRobot.py:162-345 _sort_links, 1426-1467 _find_ets, 1554-1652 ets), the batched inverse dynamics of
``Robot.rne`` (Robot.py:1704-1903) and ``Robot.URDF`` ingestion (Robot.py URDF / tools/urdf/urdf.py:1694-1758)."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Union

import numpy as np

from . import _buffers as B
from . import _lib
from . import _opspace
from . import _static
from ._se3 import SE3
from .DHLink import _inertia
from .ET import ET
from .ETS import ETS, _mat44


class Link:
    """A rigid link = an ETS ending in at most one joint (reference Link.py:120-215), hanging off a parent link,
    with the dynamic parameters Robot.rne reads (m, r; I, Jm, B, Tc, G are carried for URDF round trips)."""

    def __init__(self, ets=None, name: Optional[str] = None, parent: Union["Link", str, None] = None, jindex: Optional[int] = None,
                 m: float = 0.0, r=None, I=None, Jm: float = 0.0, B: float = 0.0, Tc=None, G: float = 0.0, qlim=None, **kwargs):  # noqa: E741
        if ets is None:
            ets = ETS()
        elif isinstance(ets, ET):
            ets = ETS(ets)
        elif not isinstance(ets, ETS):
            raise TypeError("The ets argument must be of type ETS or ET")
        if ets.n > 1 or (ets.n == 1 and not ets[-1].isjoint):
            raise ValueError("a Link's ETS may contain one joint, as its last transform")
        self.ets = ets
        self.name = name
        self.parent = parent if isinstance(parent, Link) else None
        self.parent_name = parent if isinstance(parent, str) else None
        self.children: List["Link"] = []
        self._jindex = jindex
        self.m = float(m)
        self.r = np.zeros(3) if r is None else np.asarray(r, dtype=np.float64).reshape(3)
        self.I = np.zeros((3, 3)) if I is None else _inertia(I)  # noqa: E741
        self.Jm, self.B, self.G = float(Jm), float(B), float(G)
        self.Tc = np.zeros(2) if Tc is None else np.asarray(Tc, dtype=np.float64).ravel()
        if qlim is not None and self.isjoint:
            self.ets[-1].qlim = np.asarray(qlim, dtype=np.float64).reshape(2)

    @property
    def isjoint(self) -> bool:
        return self.ets.n == 1

    @property
    def v(self) -> Optional[ET]:
        """the variable (joint) transform of the link, reference Link.v"""
        return self.ets[-1] if self.isjoint else None

    @property
    def jindex(self) -> Optional[int]:
        return self._jindex

    @jindex.setter
    def jindex(self, j):
        self._jindex = j

    @property
    def qlim(self):
        return None if not self.isjoint else self.ets[-1].qlim

    def A(self, q: float = 0.0) -> np.ndarray:
        """link transform at joint coordinate q (reference Link.A, Link.py:1381-1420)"""
        T = np.eye(4)
        for et in self.ets:
            T = T @ (et.A(q) if et.isjoint else et.A())
        return T

    def __repr__(self):
        p = self.parent.name if self.parent is not None else None
        return f"Link({self.name!r}, {self.ets}, parent={p!r}, jindex={self._jindex})"


_AXES = {"Rx": 0, "Ry": 1, "Rz": 2, "tx": 3, "ty": 4, "tz": 5}


class Robot:
    """An ETS robot: a tree of links (reference Robot / ERobot)."""

    def __init__(self, arg, name: str = "", manufacturer: str = "", base=None, tool=None, gravity=None, **kwargs):
        if isinstance(arg, ETS):
            links = self._split(arg)
        elif isinstance(arg, (list, tuple)) and all(isinstance(l, Link) for l in arg):
            links = list(arg)
        else:
            raise TypeError("arg must be an ETS or a list of Link")
        self.name, self.manufacturer = name, manufacturer
        self._sort_links(links)
        self._sub_ets = {}
        self._T = np.eye(4) if base is None else _mat44(base, "base")
        self._tool = None if tool is None else _mat44(tool, "tool")
        self._gravity = np.array([0.0, 0.0, -9.81]) if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        self._configs = {}
        self._tree = None

    @staticmethod
    def _split(ets: ETS) -> List[Link]:
        links, cur, parent = [], [], None
        for e in ets:
            cur.append(e)
            if e.isjoint:
                parent = Link(ETS(cur), name=f"link{len(links)}", parent=parent, jindex=e.jindex)
                links.append(parent)
                cur = []
        if cur:
            links.append(Link(ETS(cur), name="ee", parent=parent))
        return links

    def _sort_links(self, links: List[Link]):
        """Names, parents, children, base link, end-effector links, joint numbering and link order
        (reference BaseRobot._sort_links, BaseRobot.py:162-372)."""
        self._linkdict = {}
        for k, link in enumerate(links):
            if link.name is None or link.name == "":
                link.name = f"link-{k}"
            if link.name in self._linkdict:
                raise ValueError(f"link name {link.name} is not unique")
            self._linkdict[link.name] = link
            link.children = []
        for link in links:
            if link.parent is None and link.parent_name is not None:
                if link.parent_name not in self._linkdict:
                    raise ValueError(f"link {link.name}: unknown parent {link.parent_name}")
                link.parent = self._linkdict[link.parent_name]
        if all(link.parent is None for link in links):  # no structure given: a serial chain in list order
            for i in range(len(links) - 1):
                links[i + 1].parent = links[i]
        base = None
        for link in links:
            if link.parent is not None:
                if link.parent.name not in self._linkdict or self._linkdict[link.parent.name] is not link.parent:
                    raise ValueError(f"the parent of link {link.name} is not a link of this robot")
                link.parent.children.append(link)
            else:
                if base is not None:
                    raise ValueError("Multiple base links")
                base = link
        if base is None:
            raise ValueError("Invalid link configuration provided, must have a base link")
        self._base_link = base
        self._ee_links = [l for l in links if not l.children]
        joints = [l for l in links if l.isjoint]
        auto = all(l._jindex is None for l in joints) or all(getattr(l.ets, "_auto_jindex", False) for l in joints)
        if auto:  # number the joints and order the links depth first from the base (BaseRobot.py:333-346)
            order, k = [], 0
            for link in self.dfs_links(base):
                if link.isjoint:
                    link._jindex = k
                    k += 1
                order.append(link)
            links = order
        elif all(l._jindex is not None for l in joints):
            want = set(range(len(joints)))
            for l in joints:
                if l._jindex not in want:
                    raise ValueError(f"joint index {l._jindex} was repeated or out of range")
                want.discard(l._jindex)
        else:
            raise ValueError("all links must have a jindex, or none have a jindex")
        for l in joints:  # the joint ET reads the robot-wide q at the link's jindex
            if l.ets[-1].jindex != l._jindex:
                ets = [et.copy() for et in l.ets]
                ets[-1].jindex = l._jindex
                l.ets = ETS(ets)
        self.links = links

    def dfs_links(self, start: Link, func=None) -> List[Link]:
        """depth-first, parents before children, children in the order they were attached (BaseRobot.py:1846-1880)"""
        visited = []

        def vis(link):
            visited.append(link)
            if func is not None:
                func(link)
            for c in link.children:
                if c not in visited:
                    vis(c)

        vis(start)
        return visited

    # ---- structure
    @property
    def base_link(self) -> Link:
        return self._base_link

    @property
    def ee_links(self) -> List[Link]:
        return self._ee_links

    @property
    def base(self) -> SE3:
        return SE3(self._T)

    @base.setter
    def base(self, T):
        self._T = np.eye(4) if T is None else _mat44(T, "base")

    @property
    def gravity(self) -> np.ndarray:
        return self._gravity

    @gravity.setter
    def gravity(self, g):
        self._gravity = np.asarray(g, dtype=np.float64).reshape(3)

    @property
    def n(self) -> int:
        return sum(1 for l in self.links if l.isjoint)

    @property
    def qlim(self):
        out = np.zeros((2, self.n))
        for l in self.links:
            if l.isjoint:
                out[:, l.jindex] = l.ets[-1].qlim
        return out

    def __getitem__(self, i):
        return self._linkdict[i] if isinstance(i, str) else self.links[i]

    def __len__(self):
        return len(self.links)

    def addconfiguration(self, name, q):
        self._configs[name] = np.asarray(q, dtype=np.float64)
        setattr(self, name, self._configs[name])

    def _getlink(self, link, default: Link) -> Link:
        """Link reference or name -> Link (reference BaseRobot._getlink 1377-1424)."""
        if link is None:
            return default
        if isinstance(link, str):
            if link in self._linkdict:
                return self._linkdict[link]
            raise ValueError(f"no link named {link}")
        if isinstance(link, Link):
            if link.name in self._linkdict and self._linkdict[link.name] is link:
                return link
            raise ValueError("link not in robot links")
        raise TypeError("unknown argument")

    def _find_ets(self, link: Link, end: Link, explored: set, path: Optional[ETS]) -> Optional[ETS]:
        """Depth-first search whose neighbours are a node's children AND its parent; moving to a child multiplies the
        child's transform on, moving to the parent multiplies the inverse of the link being left
        (reference BaseRobot._find_ets, BaseRobot.py:1426-1467)."""
        toplevel = path is None
        explored.add(id(link))
        if link is end:
            return path
        if toplevel:
            path = link.ets
        for child in link.children:
            if id(child) not in explored:
                p = self._find_ets(child, end, explored, path * child.ets)
                if p is not None:
                    return p
        if toplevel:
            path = None
        if link.parent is not None and id(link.parent) not in explored:
            up = link.ets.inv() if path is None else path * link.ets.inv()
            p = self._find_ets(link.parent, end, explored, up)
            if p is not None:
                return p
        return None

    def ets(self, start=None, end=None) -> ETS:
        """``robot.ets()``: the chain from the base link to the (first) end-effector; ``robot.ets(start=l1, end=l2)``:
        the kinematics from link ``l1`` to link ``l2`` (Link reference or name) wherever the two sit in the tree --
        down a branch, up towards the base (inverted link transforms), or up one branch and down another
        (reference BaseRobot.ets 1554-1652).  Joints keep the jindex they have in the whole robot, so q stays the
        robot's full joint vector."""
        a = self._getlink(start, self._base_link)
        if end is None and len(self._ee_links) > 1:
            print("multiple end-effectors present, ambiguous, using self.ee_links[0]")
        b = self._getlink(end, self._ee_links[0])
        key = (a.name, b.name)
        if key not in self._sub_ets:
            ets = a.ets if a is b else self._find_ets(a, b, set(), None)
            if ets is None:
                raise ValueError("Could not find the requested ETS in this robot")
            self._sub_ets[key] = ETS([et.copy() for et in ets])
        return self._sub_ets[key]

    def _base_arg(self):
        return None if np.array_equal(self._T, np.eye(4)) else self._T

    def _tool_arg(self, tool):
        if tool is not None:
            return tool
        return self._tool

    # RobotKinematics.py:92-97: fkine applies the robot's base
    def fkine(self, q, end=None, start=None, tool=None, include_base: bool = True, **kw) -> SE3:
        return self.ets(start, end).fkine(q, base=self._base_arg(), tool=self._tool_arg(tool), include_base=include_base, **kw)

    def eval(self, q, end=None, start=None, tool=None, include_base: bool = True, **kw):
        return self.ets(start, end).eval(q, base=self._base_arg(), tool=self._tool_arg(tool), include_base=include_base, **kw)

    def fkine_all(self, q, dtype=None):
        """Pose of every link frame (reference Robot.fkine_all, Robot.py:638-700): frame 0 is the base transform, frame i
        the pose of the link whose number is i (its position in ``robot.links`` + 1).  (L+1,4,4) for one q,
        (N,L+1,4,4) for a batch; tool transforms do not enter, as in the reference."""
        chains = [self.ets(end=l) for l in self.links]
        return ETS.eval_frames(chains, q, base=self._base_arg(), dtype=dtype)

    # RobotKinematics.py:158 / 219: the Jacobians do NOT see the base
    def jacob0(self, q, end=None, start=None, tool=None, **kw):
        return self.ets(start, end).jacob0(q, tool=self._tool_arg(tool), **kw)

    def pay(self, W, q=None, J=None, frame=1, end=None, start=None, tool=None, dtype=None):
        """Joint torques -J^T W of a payload wrench on the end effector of ``ets(start, end)`` (reference
        DynamicsMixin.pay); see DHRobot.pay.  J = jacobe (frame 1) or jacob0 (frame 0) of that chain with the tool, as
        ``jacobe`` / ``jacob0`` give them; tau has one entry per joint of the chain, in chain order (the columns of J)."""
        e = self.ets(start, end)
        T = self._tool_arg(tool)
        if T is not None and q is not None:
            T = _mat44(T, "tool")
            if not np.array_equal(T, np.eye(4)):
                e = ETS([*e, ET.SE3(T)])
        return _static.pay(e, W, q=q, J=J, frame=frame, dtype=dtype)

    def jacobe(self, q, end=None, start=None, tool=None, **kw):
        return self.ets(start, end).jacobe(q, tool=self._tool_arg(tool), **kw)

    def jacob0_analytical(self, q, representation="rpy/xyz", end=None, start=None, tool=None, **kw):
        return self.ets(start, end).jacob0_analytical(q, representation=representation, tool=self._tool_arg(tool), **kw)

    def fkine_jacob0(self, q, tool=None, **kw):
        return self.ets().fkine_jacob0(q, base=self._base_arg(), tool=self._tool_arg(tool), **kw)

    def hessian0(self, q=None, J0=None, end=None, start=None, tool=None, **kw):
        return self.ets(start, end).hessian0(q, J0=J0, tool=self._tool_arg(tool), **kw)

    def hessiane(self, q=None, Je=None, end=None, start=None, tool=None, **kw):
        return self.ets(start, end).hessiane(q, Je=Je, tool=self._tool_arg(tool), **kw)

    def manipulability(self, q=None, J=None, method="yoshikawa", axes="all", end=None, start=None, **kw):
        return self.ets(start, end).manipulability(q, J=J, method=method, axes=axes, **kw)

    def jacobm(self, q=None, J=None, H=None, end=None, start=None, axes="all", **kw):
        """reference Robot.jacobm, Robot.py:1101-1232"""
        return self.ets(start, end).jacobm(q, J=J, H=H, axes=axes, **kw)

    def jacob0_dot(self, q, qd, J0=None, representation=None, **kw):
        """reference Robot.jacob0_dot, Robot.py:964-1099"""
        return self.ets().jacob0_dot(q, qd, J0=J0, representation=representation, **kw)

    def ik_LM(self, Tep, end=None, start=None, **kw):
        return self.ets(start, end).ik_LM(Tep, **kw)

    def ikine_LM(self, Tep, end=None, start=None, **kw):
        return self.ets(start, end).ikine_LM(Tep, **kw)

    def jtraj(self, T1, T2, t, device=None, **kwargs):
        """Joint-space trajectory between two end-effector poses (reference Robot.jtraj, Robot.py:917-961): both poses go
        through ``ikine_LM`` (``kwargs`` to the solver), the quintic ``jtraj`` joins the solutions; ``device=True`` leaves
        the (N,n) samples in HBM for ``rne`` / ``eval``."""
        from .trajectory import jtraj as _jtraj

        q1, q2 = self.ikine_LM(T1, **kwargs), self.ikine_LM(T2, **kwargs)
        return _jtraj(q1.q, q2.q, t, device=device)

    # reference RobotKinematics.py:748-1027 (ik_NR, ik_GN), 1228-1525 (ikine_NR, ikine_GN)
    def ik_NR(self, Tep, end=None, start=None, **kw):
        return self.ets(start, end).ik_NR(Tep, **kw)

    def ik_GN(self, Tep, end=None, start=None, **kw):
        return self.ets(start, end).ik_GN(Tep, **kw)

    def ikine_NR(self, Tep, end=None, start=None, **kw):
        return self.ets(start, end).ikine_NR(Tep, **kw)

    def ikine_GN(self, Tep, end=None, start=None, **kw):
        return self.ets(start, end).ikine_GN(Tep, **kw)

    # ---- inverse dynamics of the tree (reference Robot.rne, Robot.py:1704-1903)
    def tree_description(self) -> dict:
        """The tree as Robot.rne walks it: links grouped so that static links travel with the next joint link in
        link order (Robot.py:1763-1772); per group the parent group, the folded constant transform, the joint
        (axis, flip, jindex) and the 6x6 spatial inertia = sum of SpatialInertia(m, r) of the group's links
        (Robot.py:1775-1783: mass and centre of mass only -- the links' rotational inertia is not used there)."""
        joints = [l for l in self.links if l.isjoint]
        group_of = {id(l): g for g, l in enumerate(joints)}
        desc = dict(parent=[], axis=[], flip=[], jindex=[], C=[], I6=[])
        for g, joint in enumerate(joints):
            # the group: the joint link and the static links between it and the next joint towards the base.  For a
            # serial robot (and for any tree listed depth first) this is the reference's "static links travel with the
            # first joint that follows them in link order"; a static LEAF is in no group -- the reference drops trailing
            # ones and would glue one that sits mid-list onto the next branch's joint, which has no physical meaning.
            members, up = [joint], joint.parent
            while up is not None and not up.isjoint:
                members.insert(0, up)
                up = up.parent
            if up is None:
                desc["parent"].append(-1)
            else:
                if group_of[id(up)] >= g:
                    raise ValueError("links must be ordered so that a parent's joint precedes its children (Robot.rne walks them in order)")
                desc["parent"].append(group_of[id(up)])
            Cm = np.eye(4)
            I6 = np.zeros((6, 6))
            for l in members:
                for et in l.ets:
                    if not et.isjoint:
                        Cm = Cm @ et.A()
                sk = np.array([[0, -l.r[2], l.r[1]], [l.r[2], 0, -l.r[0]], [-l.r[1], l.r[0], 0]])
                I6 += np.block([[l.m * np.eye(3), l.m * sk.T], [l.m * sk, l.m * sk @ sk.T]])
            jet = joint.ets[-1]
            desc["axis"].append(_AXES[jet.axis])
            desc["flip"].append(int(jet.isflip))
            desc["jindex"].append(int(joint.jindex))
            desc["C"].append(Cm)
            desc["I6"].append(I6)
        n = len(joints)
        assert n == self.n
        return desc

    def _tree_handle(self):
        # the kernels are generated from the links' masses and centres of mass: a changed parameter (link.m = ..., or an
        # in-place edit of link.r) must not keep serving the old program
        sig = np.concatenate([np.r_[l.m, np.asarray(l.r, dtype=np.float64).reshape(3)] for l in self.links]).tobytes()
        if self._tree is not None and sig != getattr(self, "_tree_sig", None):
            _lib.lib().b2k_tree_destroy(self._tree)
            self._tree = None
        self._tree_sig = sig
        if self._tree is None:
            d = self.tree_description()
            n = len(d["parent"])
            if n > 16:
                raise ValueError("Robot.rne supports up to 16 joints")
            i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731
            keep = [i32(d[k]) for k in ("parent", "axis", "flip", "jindex")]
            Cm = np.ascontiguousarray(np.asarray(d["C"], dtype=np.float64)[:, :3, :].reshape(n, 12))
            I6 = np.ascontiguousarray(np.asarray(d["I6"], dtype=np.float64).reshape(n, 36))
            h = _lib.vp()
            _lib.check(_lib.lib().b2k_tree_create(n, *(k.ctypes.data_as(_lib.ip) for k in keep), _lib.dptr(Cm), _lib.dptr(I6), C.byref(h)))
            self._tree = h
        return self._tree

    def __del__(self):
        h = getattr(self, "_tree", None)
        if h is not None:
            try:
                _lib.lib().b2k_tree_destroy(h)
            except Exception:
                pass

    def rne(self, q, qd, qdd, symbolic: bool = False, gravity=None, dtype=None):
        """Inverse dynamics of the link tree, tau = rne(q, qd, qdd): (n,) for one state, (N,n) for a trajectory
        (reference Robot.rne, Robot.py:1704-1903 -- a Python loop over rows and spatial-vector objects there; one
        kernel generated for this robot here).  Kept from the reference: only mass and centre of mass of the links
        enter (no rotational inertia, no motor / friction terms), a flipped joint's motion subspace is the unflipped
        axis, torques are ordered by joint group."""
        if symbolic:
            raise TypeError("Symbolic value")
        for x, nm in ((q, "q"), (qd, "qd"), (qdd, "qdd")):
            B.check_numeric(x, nm)
        n = self.n
        dt = B.pick_dtype(q, dtype)
        host = not B.is_tensor(q)
        single = (q.dim() if B.is_tensor(q) else np.ndim(q)) == 1
        dev = []
        for x, nm in ((q, "q"), (qd, "qd"), (qdd, "qdd")):
            t = B.to_device(x, dt)
            t = t.reshape(1, -1) if t.dim() == 1 else t
            if t.dim() != 2 or t.shape[1] != n:
                raise ValueError(f"{nm} must have shape ({n},) or (N,{n}); got {tuple(t.shape)}")
            dev.append(t.contiguous())
        N = dev[0].shape[0]
        if any(t.shape[0] != N for t in dev):
            raise ValueError("q, qd, qdd must have the same number of rows")
        g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        ag = np.ascontiguousarray(-g)  # a_grav = -gravity (Robot.py:1785-1788)
        tau = B.empty((N, n), dt, like=dev[0])
        _lib.check(_lib.lib().b2k_tree_rne(self._tree_handle(), B.code(dt), B.ptr(dev[0]), B.ptr(dev[1]), B.ptr(dev[2]), N,
                                           _lib.dptr(ag), B.ptr(tau), B.stream_ptr(dev[0])))
        if host:
            tau = B.to_host(tau)
        return tau[0] if single else tau

    _DYN_OPS = {"rne": 0, "inertia": 1, "gravload": 2, "itorque": 3, "coriolis": 4, "accel": 5}

    def rne_kernel_info(self, dtype=np.float64, gravity=None, op="rne") -> str:
        g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        ag = np.ascontiguousarray(-g)
        buf = C.create_string_buffer(2048)
        _lib.check(_lib.lib().b2k_tree_info(self._tree_handle(), self._DYN_OPS[op], B.code(np.dtype(dtype)), _lib.dptr(ag), buf, 2048))
        return buf.value.decode()

    # ---- dynamics built on the recursion (reference DynamicsMixin, Dynamics.py, which BaseRobot inherits: each method
    #      there is a Python loop of self.rne calls; here one generated kernel per operation, b2k_tree_dyn)
    def _tree_dyn(self, op, ins, names, out_tail, gravity=None, dtype=None):
        for x, nm in zip(ins, names):
            B.check_numeric(x, nm)
        n = self.n
        dt = B.pick_dtype(ins[0], dtype)
        host = not B.is_tensor(ins[0])
        single = (ins[0].dim() if B.is_tensor(ins[0]) else np.ndim(ins[0])) == 1
        dev = []
        for x, nm in zip(ins, names):
            t = B.to_device(x, dt)
            t = t.reshape(1, -1) if t.dim() == 1 else t
            if t.dim() != 2 or t.shape[1] != n:
                raise ValueError(f"{nm} must have shape ({n},) or (N,{n}); got {tuple(t.shape)}")
            dev.append(t.contiguous())
        N = dev[0].shape[0]
        if any(t.shape[0] != N for t in dev):
            raise ValueError(", ".join(names) + " must have the same number of rows")
        g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
        ag = np.ascontiguousarray(-g)
        out = B.empty((N,) + tuple(out_tail), dt, like=dev[0])
        ptrs = [B.ptr(t) for t in dev] + [None] * (3 - len(dev))
        _lib.check(_lib.lib().b2k_tree_dyn(self._tree_handle(), self._DYN_OPS[op], B.code(dt), ptrs[0], ptrs[1], ptrs[2], N,
                                           _lib.dptr(ag), B.ptr(out), B.stream_ptr(dev[0])))
        if host:
            out = B.to_host(out)
        return out[0] if single else out

    def inertia(self, q, dtype=None):
        """Joint-space inertia matrix M(q), (n,n) or (N,n,n) (Dynamics.py:700-758: n rne calls per row there)."""
        return self._tree_dyn("inertia", (q,), ("q",), (self.n, self.n), dtype=dtype)

    def gravload(self, q, gravity=None, dtype=None):
        """Gravity torque rne(q, 0, 0) (Dynamics.py:861-915)."""
        return self._tree_dyn("gravload", (q,), ("q",), (self.n,), gravity=gravity, dtype=dtype)

    def itorque(self, q, qdd, dtype=None):
        """Inertia torque M(q) qdd = rne(q, 0, qdd) without gravity (Dynamics.py:1418-1459)."""
        return self._tree_dyn("itorque", (q, qdd), ("q", "qdd"), (self.n,), dtype=dtype)

    def coriolis(self, q, qd, dtype=None):
        """Coriolis / centripetal matrix C(q, qd), (n,n) or (N,n,n) (Dynamics.py:760-857: n(n+1)/2 rne calls per row)."""
        return self._tree_dyn("coriolis", (q, qd), ("q", "qd"), (self.n, self.n), dtype=dtype)

    def accel(self, q, qd, torque, gravity=None, dtype=None):
        """Forward dynamics qdd = M(q)^-1 (torque - rne(q, qd, 0)) (Dynamics.py:424-503: n + 1 rne calls and a numpy
        solve per row there)."""
        return self._tree_dyn("accel", (q, qd, torque), ("q", "qd", "torque"), (self.n,), gravity=gravity, dtype=dtype)

    # ---- operational-space dynamics (reference DynamicsMixin, Dynamics.py between gravload and itorque): _opspace.py
    def _opspace_robot(self):
        """The tree kernels list torque columns in joint-group order, the Jacobian lists joints in chain order: the two
        only meet when both are q order and the chain to the end-effector moves every joint."""
        if list(self.tree_description()["jindex"]) != list(range(self.n)):
            raise ValueError("operational-space dynamics needs the joint groups in q order (jindex 0..n-1)")
        if list(self.ets().jindices) != list(range(self.n)):
            raise ValueError("operational-space dynamics needs the Jacobian to the end-effector to cover all n joints in q order")
        return self

    def inertia_x(self, q, pinv=False, representation="rpy/xyz", Ji=None, dtype=None):
        """Operational-space inertia Mx = Ji^T M Ji, (6,6) or (N,6,6); Ji = inv / pinv of jacob0_analytical."""
        return _opspace.inertia_x(self._opspace_robot(), q, pinv=pinv, representation=representation, Ji=Ji, dtype=dtype)

    def coriolis_x(self, q, qd, pinv=False, representation="rpy/xyz", J=None, Ji=None, Jd=None, C=None, Mx=None, dtype=None):
        """Operational-space Coriolis matrix Cx = Ji^T C Ji - Mx Jad Ji, (6,6) or (N,6,6)."""
        return _opspace.coriolis_x(self._opspace_robot(), q, qd, pinv=pinv, representation=representation, J=J, Ji=Ji, Jd=Jd, C=C,
                                   Mx=Mx, dtype=dtype)

    def gravload_x(self, q, gravity=None, pinv=False, representation="rpy/xyz", Ji=None, dtype=None):
        """Operational-space gravity load Gx = Ji^T G, (6,) or (N,6)."""
        return _opspace.gravload_x(self._opspace_robot(), q, gravity=gravity, pinv=pinv, representation=representation, Ji=Ji,
                                   dtype=dtype)

    def accel_x(self, q, xd, wrench, gravity=None, pinv=False, representation="rpy/xyz", dtype=None):
        """Operational-space forward dynamics: task acceleration (6,) or (N,6) under the end-effector wrench."""
        return _opspace.accel_x(self._opspace_robot(), q, xd, wrench, gravity=gravity, pinv=pinv, representation=representation,
                                dtype=dtype)

    def fdyn(self, T, q0, Q=None, Q_args=None, qd0=None, solver="RK45", solver_args=None, dt=None, progress=False, gravity=None,
             max_steps: int = 4096, dtype=None):
        """Integrate the forward dynamics of the tree robot over [0, T] (DynamicsMixin.fdyn, Dynamics.py:185-422, inherited
        by the reference's Robot through BaseRobot).  Arguments, torque laws, ensemble form ((B,n) initial states, one lane
        per trajectory) and return values as ``DHRobot.fdyn``; the right-hand side is this robot's generated ``accel``
        recursion (b2k_tree_fdyn)."""
        from ._fdyn import fdyn as _fdyn

        def kernel_gravity(gravity):
            g = self._gravity if gravity is None else np.asarray(gravity, dtype=np.float64).reshape(3)
            return -g  # a_grav = -gravity (Robot.py:1785-1788)

        callable_q = callable(Q)
        return _fdyn(self, None if callable_q else _lib.lib().b2k_tree_fdyn, None if callable_q else self._tree_handle(), kernel_gravity,
                     T, q0, Q=Q, Q_args=Q_args, qd0=qd0, solver=solver, solver_args=solver_args, dt=dt, gravity=gravity,
                     max_steps=max_steps, dtype=dtype)

    # ---- model ingestion
    @classmethod
    def URDF(cls, file_path, **kwargs) -> "Robot":
        """Build a robot from a URDF / xacro file (reference Robot.URDF / URDF_read -> tools/urdf/urdf.py)."""
        from .urdf import urdf_to_links

        links, name = urdf_to_links(file_path, **kwargs)
        return cls(links, name=name)


ERobot = Robot
