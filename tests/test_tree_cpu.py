"""Host logic of the rigid-body tree robots (no GPU): link sorting and joint numbering, the tree path search behind
Robot.ets(start, end) (reference BaseRobot.py:162-372, 1426-1467, 1554-1652), URDF / xacro ingestion (reference
tools/urdf/urdf.py:1694-1780), and the tree description Robot.rne hands to the kernel generator.  Kinematics of the
extracted chains are checked with the CPU oracle on the chain descriptions (the oracle is the checker, nothing is
computed by the product here)."""
import os

import numpy as np
import pytest

import b2kin as rtb
from oracle import chains as ch
from oracle import oracle as orc

HERE = os.path.dirname(__file__)
URDF_DIR = os.path.join(HERE, "golden", "urdf")
ET, ETS, Link, Robot = rtb.ET, rtb.ETS, rtb.Link, rtb.Robot


def fk(ets, q):
    return orc.Chain(ets.describe()).fkine(np.atleast_2d(q))


def make_tree():
    """base -> l1(Rz) -> l2(Ry) -> l3(Rx) -> ee_a ; l2 -> b1(tz) -> b2(Rz) -> ee_b"""
    l1 = Link(ETS(ET.tz(0.3)) * ET.Rz(), name="l1")
    l2 = Link(ETS(ET.tx(0.2)) * ET.Ry(), name="l2", parent=l1)
    l3 = Link(ETS(ET.tx(0.25)) * ET.Rx(), name="l3", parent=l2)
    ea = Link(ETS(ET.tz(0.1)), name="ee_a", parent=l3)
    b1 = Link(ETS(ET.Rx(0.4)) * ET.ty(0.1) * ET.tz(), name="b1", parent="l2")
    b2 = Link(ETS(ET.tx(0.15)) * ET.Rz(flip=True), name="b2", parent=b1)
    eb = Link(ETS(ET.Ry(-0.3)) * ET.tx(0.05), name="ee_b", parent=b2)
    return Robot([l1, l2, b1, l3, b2, ea, eb], name="tree")


def test_link_sorting_and_joint_numbering():
    r = make_tree()
    assert r.n == 5 and r.base_link.name == "l1"
    assert [l.name for l in r.ee_links] == ["ee_a", "ee_b"]
    # depth-first from the base, children in the order they were attached (BaseRobot.py:333-346, 1846-1880)
    assert [l.name for l in r.links] == ["l1", "l2", "b1", "b2", "ee_b", "l3", "ee_a"]
    assert {l.name: l.jindex for l in r.links if l.isjoint} == {"l1": 0, "l2": 1, "b1": 2, "b2": 3, "l3": 4}
    assert [l.name for l in r["l2"].children] == ["b1", "l3"]
    assert r["b1"].parent is r["l2"]
    with pytest.raises(ValueError, match="not unique"):
        Robot([Link(ETS(ET.Rz()), name="a"), Link(ETS(ET.Rz()), name="a")])
    with pytest.raises(ValueError, match="Multiple base"):
        a, b = Link(ETS(ET.Rz()), name="a"), Link(ETS(ET.Rz()), name="b")
        c = Link(ETS(ET.Rz()), name="c", parent=a)
        Robot([a, b, c])
    # explicit numbering is kept, and must be a permutation
    r2 = Robot([Link(ETS(ET.Rz(jindex=1)), name="a", jindex=1), Link(ETS(ET.Rz(jindex=0)), name="b", jindex=0, parent="a")])
    assert [l.jindex for l in r2.links] == [1, 0]
    with pytest.raises(ValueError, match="repeated or out of range"):
        Robot([Link(ETS(ET.Rz(jindex=1)), name="a", jindex=1), Link(ETS(ET.Rz(jindex=1)), name="b", jindex=1, parent="a")])
    # no structure given: a serial chain in list order (BaseRobot.py:218-220)
    r3 = Robot([Link(ETS(ET.Rz()), name="a"), Link(ETS(ET.tx(1)) * ET.Ry(), name="b")])
    assert r3["b"].parent is r3["a"] and r3.n == 2


def test_tree_path_search_matches_explicit_chains():
    r = make_tree()
    rng = np.random.default_rng(0)
    q = rng.uniform(-1, 1, (8, 5))
    L = {l.name: l for l in r.links}

    def chain(*parts):  # explicit product of link transforms (inverse where noted), keeping the robot-wide jindices
        e = None
        for name, inv in parts:
            x = L[name].ets.inv() if inv else L[name].ets
            e = x if e is None else e * x
        return e

    # default: base link to the first end-effector (ee_links keeps the order the links were given in)
    np.testing.assert_allclose(fk(r.ets(), q), fk(chain(("l1", 0), ("l2", 0), ("l3", 0), ("ee_a", 0)), q), atol=1e-14)
    # down the other branch
    np.testing.assert_allclose(fk(r.ets(end="ee_b"), q), fk(chain(("l1", 0), ("l2", 0), ("b1", 0), ("b2", 0), ("ee_b", 0)), q), atol=1e-14)
    # a sub-chain: start link's own transform included (_find_ets: path = link.ets at the top level)
    np.testing.assert_allclose(fk(r.ets(start="l2", end="b2"), q), fk(chain(("l2", 0), ("b1", 0), ("b2", 0)), q), atol=1e-14)
    # towards the base: inverses of the links being left, from the start link up to (not including) the end link
    np.testing.assert_allclose(fk(r.ets(start="l3", end="l1"), q), fk(chain(("l3", 1), ("l2", 1)), q), atol=1e-14)
    # up one branch, down the other: b2 -> b1 -> l2 -> l3 -> ee_a
    e = r.ets(start="b2", end="ee_a")
    np.testing.assert_allclose(fk(e, q), fk(chain(("b2", 1), ("b1", 1), ("l3", 0), ("ee_a", 0)), q), atol=1e-14)
    # consistency: T(l1->ee_a) == T(l1->b2) . T(b2->ee_a) with b2's own transform counted once on each side of the pivot
    Tab = fk(r.ets(end="b2"), q)
    Tba = fk(e, q)
    np.testing.assert_allclose(Tab @ Tba, fk(chain(("l1", 0), ("l2", 0), ("l3", 0), ("ee_a", 0)), q), atol=1e-13)
    # start == end: that link's own ETS (BaseRobot.py:1631-1632)
    assert len(r.ets(start="l2", end="l2")) == len(L["l2"].ets)
    assert r.ets(start="b2", end="ee_a") is e  # cached
    with pytest.raises(ValueError):
        r.ets(end="nope")
    # joints keep their robot-wide jindex
    assert list(r.ets(end="ee_a").jindices) == [0, 1, 4]


def test_tree_description_for_rne():
    r = make_tree()
    for name, m, rr in (("l1", 1.0, [0.1, 0, 0]), ("l2", 2.0, [0, 0.1, 0]), ("b1", 0.5, [0, 0, 0.05]), ("b2", 0.3, [0.02, 0, 0]), ("l3", 0.7, [0.1, 0, 0.02])):
        r[name].m, r[name].r = m, np.array(rr, dtype=float)
    d = r.tree_description()
    assert d["parent"] == [-1, 0, 1, 2, 1] and d["jindex"] == [0, 1, 2, 3, 4]
    assert d["axis"] == [2, 1, 5, 2, 0] and d["flip"] == [0, 0, 0, 1, 0]
    np.testing.assert_allclose(d["C"][2], ch.trotx(0.4) @ ch.transl(0, 0.1, 0))
    np.testing.assert_allclose(d["I6"][1], orc.spatial_inertia(2.0, [0, 0.1, 0]))
    # a static link between two joints travels with the NEXT joint (Robot.py:1763-1772): Spong's arm with a static middle link
    l1 = Link(ETS(ET.Ry()), m=1, r=[0.5, 0, 0], name="l1")
    l2 = Link(ETS(ET.tx(0.4)), m=0.2, r=[0.1, 0, 0], parent=l1, name="l2")
    l3 = Link(ETS(ET.tx(0.6)) * ET.Ry(), m=1, r=[0.5, 0, 0], parent=l2, name="l3")
    d3 = Robot([l1, l2, l3]).tree_description()
    assert d3["parent"] == [-1, 0]
    np.testing.assert_allclose(d3["C"][1], ch.transl(1.0, 0, 0))
    np.testing.assert_allclose(d3["I6"][1], orc.spatial_inertia(0.2, [0.1, 0, 0]) + orc.spatial_inertia(1, [0.5, 0, 0]))


def test_urdf_ingestion_of_a_branched_robot():
    r = Robot.URDF(os.path.join(URDF_DIR, "two_arm.urdf"))
    assert r.name == "two_arm" and r.n == 5 and r.base_link.name == "torso"
    assert [l.name for l in r.ee_links] == ["l_flange", "r_skew"]
    jn = {l.name: l.jindex for l in r.links if l.isjoint}
    assert jn == {"l_upper": 0, "l_fore": 1, "r_upper": 2, "r_slide": 3, "r_skew": 4}
    assert r["l_fore"].ets[-1].axis == "Ry" and r["l_fore"].ets[-1].isflip  # axis 0 -1 0
    assert r["r_slide"].ets[-1].axis == "tz" and not r["r_slide"].ets[-1].isflip
    np.testing.assert_allclose(r.qlim[:, 0], [-2.0, 2.5])
    np.testing.assert_allclose(r.qlim[:, 3], [0.0, 0.2])
    assert r["l_upper"].m == 1.5 and np.allclose(r["l_upper"].r, [0.15, 0, 0])
    # kinematics of the left arm: T = transl(0,0.2,0.5) Rz(pi/2) Rz(q0) transl(0.3,0,0) Rx(pi/2) Ry(-q1) transl(0.25,0,0) Ry(0.3)
    q = np.array([0.3, -0.7, 0.1, 0.05, 0.2])
    want = (ch.transl(0, 0.2, 0.5) @ ch.trotz(np.pi / 2) @ ch.trotz(q[0]) @ ch.transl(0.3, 0, 0) @ ch.trotx(np.pi / 2)
            @ ch.troty(-q[1]) @ ch.transl(0.25, 0, 0) @ ch.troty(0.3))
    np.testing.assert_allclose(fk(r.ets(end="l_flange"), q)[0], want, atol=1e-12)
    # the skew axis (1 1 0) is rotated onto z by a constant: the joint turns about that axis in the parent frame
    e = r.ets(start="r_skew", end="r_skew")
    R0, R1 = fk(e, np.zeros(5))[0, :3, :3], fk(e, np.array([0, 0, 0, 0, 0.9]))[0, :3, :3]
    Rrel = R1 @ R0.T
    np.testing.assert_allclose(orc.trlog(Rrel), 0.9 * np.array([1, 1, 0]) / np.sqrt(2), atol=1e-12)
    # across the branches: hand to hand
    Tl, Tr = fk(r.ets(end="l_flange"), q)[0], fk(r.ets(end="r_skew"), q)[0]
    # (up: the inverses of l_flange, l_fore, l_upper; down: r_upper, r_slide, r_skew; the torso's own ETS is the identity)
    np.testing.assert_allclose(fk(r.ets(start="l_flange", end="r_skew"), q)[0], np.linalg.inv(Tl) @ Tr, atol=1e-12)
    with pytest.raises(FileNotFoundError):
        Robot.URDF("/nonexistent.urdf")


def test_xacro_expansion():
    r = Robot.URDF(os.path.join(URDF_DIR, "macro_arm.urdf.xacro"))
    assert r.name == "macro_arm" and r.n == 3 and [l.name for l in r.links] == ["base", "s1", "s2", "s3"]
    assert [r[k].m for k in ("s1", "s2", "s3")] == [2.0, 1.0, 0.5]
    np.testing.assert_allclose(r["s1"].r, [0.1, 0, 0])
    np.testing.assert_allclose(r.qlim, np.tile([[-np.pi / 2], [np.pi / 2]], (1, 3)))
    assert [r[k].ets[-1].axis for k in ("s1", "s2", "s3")] == ["Rz", "Ry", "Rz"] and r["s3"].ets[-1].isflip
    q = np.array([0.2, -0.4, 0.9])
    want = (ch.transl(0, 0, 0.1) @ ch.trotz(q[0]) @ ch.transl(0.4, 0, 0) @ ch.trotx(np.pi / 2) @ ch.troty(q[1])
            @ ch.transl(0.2, 0, 0) @ ch.trotz(-np.pi / 4) @ ch.trotz(-q[2]))
    np.testing.assert_allclose(fk(r.ets(), q)[0], want, atol=1e-12)
    r2 = Robot.URDF(os.path.join(URDF_DIR, "macro_arm.urdf.xacro"), args={"reach": "1.0"})
    np.testing.assert_allclose(r2["s1"].r, [0.25, 0, 0])


def test_changed_link_parameters_rebuild_the_tree_program():
    """Robot.rne's kernels are generated from the link masses / centres of mass; editing them after the first call must
    rebuild the handle (the DH classes track this with dirty flags, reference DHRobot.py:1326-1361)."""
    import ctypes as C

    l1 = rtb.Link(rtb.ETS(rtb.ET.Ry()), m=1, r=[0.5, 0, 0], name="l1")
    l2 = rtb.Link(rtb.ETS(rtb.ET.tx(1)) * rtb.ET.Ry(), m=1, r=[0.5, 0, 0], parent=l1, name="l2")
    rob = rtb.Robot([l1, l2])
    info0 = rob.rne_kernel_info()
    h0 = rob._tree_handle()
    assert rob._tree_handle() is h0
    l2.m = 3.0
    h1 = rob._tree_handle()
    assert h1 is not h0
    l2.r[1] = 0.25  # in-place edit of the centre of mass
    h2 = rob._tree_handle()
    assert h2 is not h1
    assert rob.rne_kernel_info() != info0  # an off-axis centre of mass adds terms to the generated recursion
    assert isinstance(h2, C.c_void_p)


def test_frame_walks_of_fkine_all():
    """ETS._frame_walks (the plan behind fkine_all / b2k_fkine_frames): every link frame is 'the pose after joint
    `after` of its walk, times a constant tail'.  Checked with the oracle: FK of the walk cut behind that joint, times
    the tail, equals FK of the link's own chain -- for a serial DH robot (one walk), a DH robot with joint offsets and
    a prismatic joint, and a branched tree (a walk per branch, static links on constants)."""
    rng = np.random.default_rng(5)

    def check(chains, qwidth, nwalks):
        walks = ETS._frame_walks(chains)
        assert len(walks) == nwalks
        Q = rng.uniform(-2, 2, (7, qwidth))
        seen = set()
        for walk, frames in walks:
            ets = list(walk)
            joints = [i for i, et in enumerate(ets) if et.isjoint]
            for slot, after, tail in frames:
                assert 0 <= after < walk.n and slot not in seen
                seen.add(slot)
                cut = ETS(ets[:joints[after] + 1])
                want = fk(chains[slot - 1], Q)
                np.testing.assert_allclose(fk(cut, Q) @ tail, want, rtol=1e-12, atol=1e-13)
        assert seen == {k + 1 for k, e in enumerate(chains) if e.n > 0}

    puma = rtb.models.Puma560()
    check([ETS.from_links([l.ets for l in puma.links[:k + 1]]) for k in range(puma.n)], 6, 1)
    mixed = rtb.DHRobot([rtb.RevoluteDH(d=0.3, a=0.1, alpha=0.5, offset=0.2), rtb.PrismaticDH(theta=0.4, a=0.2, alpha=-0.3),
                         rtb.RevoluteDH(d=0.1, a=0.3, alpha=0.7, flip=True)])
    check([ETS.from_links([l.ets for l in mixed.links[:k + 1]]) for k in range(mixed.n)], 3, 1)
    r = make_tree()
    chains = [r.ets(end=l) for l in r.links]
    check(chains, r.n, 2)  # two branches; their common trunk rides on the longer branch's walk
