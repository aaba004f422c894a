"""Planar kinematics without a GPU: the float64 restatement in planar_ref.py -- the specification test_gpu_planar.py
checks the kernel against -- is pinned to the oracle's 3-D chain on the embedded description and to central differences
of its own eval; the host logic of ET2 / ETS2 / Robot2 / SE2; and b2k_fkine_planar's rejections before any CUDA call."""
import math
import os
import sys

import numpy as np
import pytest

import b2kin as rtb
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import planar_ref as ref  # noqa: E402

E = rtb.ET2


def emb(T):
    """SE(2) -> the SE(3) acting in the xy plane"""
    A = np.eye(4)
    A[:2, :2] = T[:2, :2]
    A[:2, 3] = T[:2, 2]
    return A


@pytest.mark.parametrize("n", range(1, 11))
def test_restatement_matches_the_oracle_3d_chain(n):
    rng = np.random.default_rng(300 + n)
    ets = ref.random_chain(rng, n, wide=3)
    base, tool = ref.random_pose(rng), ref.random_pose(rng)
    q = rng.uniform(-3, 3, (40, n + 3))
    C = orc.Chain(ets.describe())
    T3 = C.fkine(q, emb(base), emb(tool))
    T2 = ref.eval_(ets, q, base, tool)
    np.testing.assert_allclose(T2, T3[:, [0, 1, 3]][:, :, [0, 1, 3]], rtol=0, atol=1e-14)
    J3 = C.jacob0(q, emb(tool))
    J2 = ref.jacob0(ets, q, tool)
    np.testing.assert_allclose(J2, J3[:, [0, 1, 5]], rtol=0, atol=1e-14)
    np.testing.assert_array_equal(J3[:, [2, 3, 4]], 0)  # the embedding never leaves the plane
    Je3 = C.jacobe(q, emb(tool))
    np.testing.assert_allclose(ref.jacobe(ets, q, tool), Je3[:, [0, 1, 5]], rtol=0, atol=1e-14)


@pytest.mark.parametrize("n", [1, 2, 5, 10])
def test_restatement_jacobian_is_the_derivative_of_eval(n):
    rng = np.random.default_rng(400 + n)
    ets = ref.random_chain(rng, n, wide=2)
    tool = ref.random_pose(rng)
    q = rng.uniform(-3, 3, (16, n + 2))
    J = ref.jacob0(ets, q, tool)
    T = ref.eval_(ets, q, tool=tool)
    h = 1e-6
    for k, col in enumerate(ets.jindices):
        dq = np.zeros_like(q)
        dq[:, col] = h
        dT = (ref.eval_(ets, q + dq, tool=tool) - ref.eval_(ets, q - dq, tool=tool)) / (2 * h)
        np.testing.assert_allclose(J[:, 0, k], dT[:, 0, 2], atol=1e-8)
        np.testing.assert_allclose(J[:, 1, k], dT[:, 1, 2], atol=1e-8)
        # dtheta/dq from dR = [[-s, -c], [c, -s]] dtheta
        np.testing.assert_allclose(J[:, 2, k], (dT[:, :2, :2] @ np.transpose(T[:, :2, :2], (0, 2, 1)))[:, 1, 0], atol=1e-8)


def test_et2_constructors_and_defaults():
    r, x, y = E.R(), E.tx(), E.ty()
    assert r.isjoint and r.isrotation and not x.isrotation and x.istranslation
    np.testing.assert_array_equal(r._qlim_default(), [-math.pi, math.pi])
    np.testing.assert_array_equal(y._qlim_default(), [0.0, 1.0])
    np.testing.assert_allclose(E.R(90, unit="deg").A(), [[0, -1, 0], [1, 0, 0], [0, 0, 1]], atol=1e-16)
    np.testing.assert_array_equal(E.tx(2.0).A(), [[1, 0, 2], [0, 1, 0], [0, 0, 1]])
    np.testing.assert_array_equal(E.ty(flip=True).A(0.5), [[1, 0, 0], [0, 1, -0.5], [0, 0, 1]])
    np.testing.assert_allclose(E.R(flip=True).A(0.3), E.R().A(-0.3))
    T = ref.random_pose(np.random.default_rng(0))
    np.testing.assert_array_equal(E.SE2(T).A(), T)
    np.testing.assert_array_equal(E.SE2(rtb.SE2(T)).A(), T)
    np.testing.assert_allclose(E.SE2(T).inv().A() @ T, np.eye(3), atol=1e-15)
    assert E.R().inv().isflip and not E.R(flip=True).inv().isflip
    assert E.tx(0.5).inv().eta == -0.5
    with pytest.raises(TypeError):
        E.R("theta")
    with pytest.raises(ValueError):
        E.SE2(np.eye(4))
    with pytest.raises(ValueError):
        E.SE2([[1, 0, 0], [0, 1, 0], [1, 0, 1]])
    with pytest.raises(ValueError):
        E("Rx")


def test_ets2_jindex_numbering_and_structure():
    e = E.R() * E.tx(1.0) * E.ty() * E.R(flip=True)
    assert isinstance(e, rtb.ETS2) and e.n == 3 and e.m == 4
    np.testing.assert_array_equal(e.jindices, [0, 1, 2])
    assert e.structure == "RPR"
    np.testing.assert_array_equal(e.qlim, [[-math.pi, 0, -math.pi], [math.pi, 1, math.pi]])
    p = rtb.ETS2([E.R(jindex=2), E.tx(0.5), E.ty(jindex=0), E.R(jindex=1)])
    np.testing.assert_array_equal(p.jindices, [2, 0, 1])
    with pytest.raises(ValueError, match="all or none"):
        rtb.ETS2([E.R(jindex=2), E.ty(), E.R()])
    with pytest.raises(TypeError):
        rtb.ETS2([E.R(), rtb.ET.Rz()])
    with pytest.raises(TypeError):
        E.R() * rtb.ET.tx(1.0)
    assert isinstance(e[1:3], rtb.ETS2) and e[1:3].m == 2


def test_ets2_compile_inv_and_embedding():
    rng = np.random.default_rng(5)
    e = rtb.ETS2([E.tx(0.3), E.R(0.4), E.R(), E.ty(0.2), E.SE2(ref.random_pose(rng)), E.tx(), E.ty(-1.0)])
    c = e.compile()
    assert [et.axis for et in c] == ["SE2", "R", "SE2", "tx", "SE2"]
    q = rng.uniform(-2, 2, (8, 2))
    np.testing.assert_allclose(ref.eval_(c, q), ref.eval_(e, q), atol=1e-15)
    ei = e.inv()
    np.testing.assert_allclose(ref.eval_(ei, q) @ ref.eval_(e, q), np.broadcast_to(np.eye(3), (8, 3, 3)), atol=1e-14)
    d = e.describe()
    np.testing.assert_array_equal(d["axis"][d["isjoint"] == 1], [2, 3])  # R -> Rz, tx -> tx
    np.testing.assert_array_equal(d["T"][4][2], [0, 0, 1, 0])
    np.testing.assert_array_equal(d["T"][4][:, 2], [0, 0, 1, 0])
    np.testing.assert_array_equal(d["T"][1][[0, 1]][:, [0, 1, 3]], e[1].A()[:2])


def test_se2_container():
    A = np.tile(np.eye(3), (4, 1, 1))
    A[:, 0, 2] = np.arange(4)
    s = rtb.SE2(A)
    assert len(s) == 4 and s.t.shape == (4, 2) and s.R.shape == (4, 2, 2)
    assert isinstance(s[2], rtb.SE2) and s[2].t[0] == 2
    assert [float(p.t[0]) for p in s] == [0, 1, 2, 3]
    assert rtb.SE2(np.eye(3)).A.shape == (3, 3)
    with pytest.raises(ValueError):
        rtb.SE2(np.eye(4))


def test_robot2_from_ets_and_links():
    r = rtb.models.ETS.Planar2()
    assert r.n == 2 and np.array_equal(r.qz, [0, 0])
    np.testing.assert_array_equal(r.qlim, [[-math.pi, -math.pi], [math.pi, math.pi]])
    L = rtb.Link2
    l0 = L(E.R(), name="l0")
    l1 = L(E.tx(1.0) * E.R(), name="l1", parent=l0)
    l2 = L(E.tx(1.0), name="ee", parent="l1")
    rl = rtb.Robot2([l2, l0, l1])  # any list order: the parents fix the chain
    assert rl.n == 2
    q = np.array([[0.3, -0.7]])
    np.testing.assert_allclose(ref.eval_(rl.ets(), q), ref.eval_(r.ets(), q), atol=1e-15)
    rs = rtb.Robot2([L(E.R()), L(E.tx(1.0) * E.R()), L(E.tx(1.0))])  # no parents: list order
    np.testing.assert_array_equal(rs.ets().jindices, [0, 1])
    rj = rtb.Robot2([L(E.R(), jindex=1), L(E.tx(1.0) * E.R(), jindex=0)])
    np.testing.assert_array_equal(rj.ets().jindices, [1, 0])
    r.addconfiguration("qx", [0.1, 0.2])
    assert np.array_equal(r.qx, [0.1, 0.2])
    np.testing.assert_array_equal(r.base.A, np.eye(3))
    np.testing.assert_array_equal(l0.A(0.0), np.eye(3))


def test_robot2_rejects_a_branched_tree():
    L = rtb.Link2
    b = L(E.R(), name="base")
    a1 = L(E.tx(1.0) * E.R(), name="arm1", parent=b)
    a2 = L(E.ty(1.0) * E.R(), name="arm2", parent=b)
    with pytest.raises(ValueError, match="'base' has 2 children"):
        rtb.Robot2([b, a1, a2])
    with pytest.raises(TypeError):
        rtb.Robot2([rtb.Link(rtb.ET.Rz())])
    with pytest.raises(TypeError):
        L(rtb.ET.Rz())


def test_q_shapes_are_checked_before_the_device():
    e = rtb.models.ETS.Planar2().ets()
    with pytest.raises(ValueError):
        e._qbatch(np.zeros((2, 2, 2)))
    with pytest.raises(ValueError, match="columns"):
        e._qbatch(np.zeros(1))
    with pytest.raises(TypeError):
        e._qbatch(["a", "b"])
    q, single = e._qbatch([0.1, 0.2])
    assert single and q.shape == (1, 2)
    q, single = e._qbatch(np.zeros((2, 1)))
    assert single and q.shape == (1, 2)
    q, single = rtb.ETS2(E.R())._qbatch(np.zeros((7, 1)))
    assert not single and q.shape == (7, 1)


# ---------------------------------------------------------------- the C ABI rejects bad arguments before any CUDA call
def _call(ets, dtype=1, N=4, ldq=None, base=None, tool=None, frame=0, T=True, J=True):
    lib = rtb._lib.lib()
    buf = np.zeros(4096)
    p = buf.ctypes.data
    b = None if base is None else np.ascontiguousarray(base, dtype=np.float64)
    t = None if tool is None else np.ascontiguousarray(tool, dtype=np.float64)
    n0 = lib.b2k_launch_count()
    rc = lib.b2k_fkine_planar(ets._chain, dtype, p, N, ets.n if ldq is None else ldq, rtb._lib.dptr(b), rtb._lib.dptr(t),
                              frame, p if T else None, p if J else None, None)
    assert lib.b2k_launch_count() == n0
    return rc, lib.b2k_last_error().decode()


@pytest.mark.parametrize("case, match", [
    (dict(dtype=2), "dtype"),
    (dict(N=-1), "negative"),
    (dict(ldq=0), "row width"),
    (dict(ldq=17), "row width"),
    (dict(frame=2), "frame"),
    (dict(frame=-1), "frame"),
    (dict(T=False, J=False), "both NULL"),
    (dict(base=np.eye(3) * 2), "not a scaled rotation|bottom row"),
    (dict(tool=[[1, 0, 0], [0, 1, 0], [0, 1, 1]]), "bottom row"),
    (dict(tool=[[1, 0.5, 0], [0, 1, 0], [0, 0, 1]]), "not a scaled rotation"),
])
def test_cabi_rejects_bad_arguments(case, match):
    rc, msg = _call(rtb.models.ETS.Planar2().ets(), **case)
    assert rc == -1 and __import__("re").search(match, msg), msg


def test_cabi_rejects_a_null_chain():
    lib = rtb._lib.lib()
    buf = np.zeros(64)
    assert lib.b2k_fkine_planar(None, 1, buf.ctypes.data, 1, 2, None, None, 0, buf.ctypes.data, None, None) == -1
    assert b"NULL" in lib.b2k_last_error()


@pytest.mark.parametrize("ets, match", [
    (rtb.ETS([rtb.ET.Rz(), rtb.ET.tx(1.0), rtb.ET.Rx()]), "joint 1 is Rx"),
    (rtb.ETS([rtb.ET.Rz(), rtb.ET.tz()]), "joint 1 is tz"),
    (rtb.ETS([rtb.ET.Rz(), rtb.ET.Ry(0.1), rtb.ET.Rz()]), "constant before joint 1 has an out-of-plane rotation"),
    (rtb.ETS([rtb.ET.tz(0.2), rtb.ET.Rz()]), "constant before joint 0 has a non-zero z translation"),
    (rtb.ETS([rtb.ET.Rz(), rtb.ET.Rx(0.3)]), "constant after the last joint has an out-of-plane rotation"),
])
def test_cabi_rejects_a_non_planar_chain_naming_the_transform(ets, match):
    rc, msg = _call(ets)
    assert rc == -1 and match in msg, msg


def test_cabi_n0_touches_no_device():
    rc, msg = _call(rtb.models.ETS.Planar2().ets(), N=0)
    assert rc == 0, msg
