"""Operational-space dynamics without a GPU: the C ABI rejects bad arguments before any CUDA call, and the oracle's
restatement of DynamicsMixin.inertia_x / coriolis_x / gravload_x / accel_x is pinned by identities that do not depend on
how it was written -- the operational-space equation of motion and the Penrose conditions of its pseudo-inverse."""
import os
import sys

import numpy as np
import pytest

import b2kin as rtb
from oracle import chains as ch
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import opspace_ref as ops  # noqa: E402

lib = rtb._lib.lib()


def _ops(dtype=1, n=6, inverse=0, Ja=8, Ji_in=None, M=8, Cm=8, Jd=8, G=8, Mx_in=None, xd=8, w=8, N=4, Ji=None, Mx=8, Cx=None,
         Gx=None, qd=None, tau=None):
    rc = lib.b2k_opspace(dtype, n, inverse, Ja, Ji_in, M, Cm, Jd, G, Mx_in, xd, w, N, Ji, Mx, Cx, Gx, qd, tau, None)
    return rc, lib.b2k_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(n=0), "n must be 1..10"),
    (dict(n=11, inverse=1), "n must be 1..10"),
    (dict(n=7, inverse=0), "inv needs a square"),
    (dict(n=3, inverse=0), "inv needs a square"),
    (dict(inverse=2), "inverse must be"),
    (dict(dtype=2), "bad dtype"),
    (dict(N=-1), "bad N"),
    (dict(Mx=None), "no output requested"),
    (dict(Ja=None), "need Ja or a given Ji"),
    (dict(M=None), "Mx needs M"),
    (dict(Mx=None, Cx=8, Cm=None), "Cx needs C, Jd"),
    (dict(Mx=None, Cx=8, Jd=None), "Cx needs C, Jd"),
    (dict(Mx=None, Cx=8, M=None), "Cx needs C, Jd"),
    (dict(Mx=None, Gx=8, G=None), "Gx needs G"),
    (dict(Mx=None, qd=8, xd=None), "qd needs xd"),
    (dict(Mx=None, tau=8, w=None), "tau needs Ja and w"),
    (dict(Mx=None, tau=8, Ja=None, Ji_in=8), "tau needs Ja and w"),
])
def test_opspace_entry_rejects_bad_arguments_before_launching(kw, msg):
    rc, err = _ops(**kw)
    assert rc == -1
    assert msg in err, err


def test_opspace_entry_accepts_what_it_documents_without_work():
    # N = 0 returns before touching the device: the argument combinations below are the valid ones
    assert _ops(N=0)[0] == 0
    assert _ops(N=0, Mx=None, Cx=8, M=None, Mx_in=8)[0] == 0
    assert _ops(N=0, n=7, inverse=1, Ja=None, Ji_in=8, Mx=None, Gx=8)[0] == 0
    assert _ops(N=0, Mx=None, qd=8, tau=8)[0] == 0


@pytest.mark.parametrize("args,msg", [
    ((1, 0, 8, 8, 8, 8, 4, 8, None), "n must be 1..10"),
    ((1, 11, 8, 8, 8, 8, 4, 8, None), "n must be 1..10"),
    ((3, 6, 8, 8, 8, 8, 4, 8, None), "bad dtype"),
    ((1, 6, 8, 8, None, 8, 4, 8, None), "must not be NULL"),
    ((1, 6, 8, 8, 8, 8, 4, None, None), "must not be NULL"),
    ((1, 6, 8, 8, 8, 8, -2, 8, None), "bad N"),
])
def test_xdd_entry_rejects_bad_arguments_before_launching(args, msg):
    assert lib.b2k_opspace_xdd(*args) == -1
    assert msg in lib.b2k_last_error().decode()


def _dh_robot(name):
    links = {"puma": ch.puma560_links, "ur10": ch.ur10_links}[name]()
    chain = orc.Chain(ch.dh_to_ets(links))
    L = orc.nofriction_L(ch.pack_rne(links))  # nofriction(coulomb=True, viscous=True)
    rne = lambda q, qd, qdd, grav: orc.rne(6, 0, L, -np.asarray(grav, dtype=float), q, qd, qdd)  # noqa: E731
    return chain, rne


@pytest.mark.parametrize("name", ["puma", "ur10"])
@pytest.mark.parametrize("pinv", [False, True])
def test_oracle_satisfies_the_operational_space_equation_of_motion(name, pinv):
    """Mx accel_x(q, xd, w) + Cx(q, Ji xd) xd + Gx = w on a friction-free arm, away from representation singularities.
    The Jad terms cancel exactly, so the identity holds to rounding whatever the difference step."""
    chain, rne = _dh_robot(name)
    rng = np.random.default_rng({"puma": 1, "ur10": 2}[name])
    q = rng.uniform(-2.5, 2.5, (120, 6))
    q = q[np.linalg.cond(ops.ja(chain, q)) < 1e3][:30]
    assert len(q) >= 20
    xd, w = rng.normal(size=(len(q), 6)), rng.normal(size=(len(q), 6)) * 10
    g = np.array([0.0, 0.0, -9.81])
    Ji = ops.ji(ops.ja(chain, q), pinv)
    qd = np.einsum("kij,kj->ki", Ji, xd)
    Mx = ops.inertia_x(rne, chain, 6, q, pinv)
    Cx = ops.coriolis_x(rne, rne, chain, 6, q, qd, pinv)
    Gx = ops.gravload_x(rne, chain, 6, q, g, pinv)
    xdd = ops.accel_x(rne, chain, 6, q, xd, w, g, pinv)
    lhs = np.einsum("kab,kb->ka", Mx, xdd) + np.einsum("kab,kb->ka", Cx, xd) + Gx
    scale = np.maximum.reduce([np.abs(w).max(1), np.abs(Gx).max(1), np.abs(np.einsum("kab,kb->ka", Mx, xdd)).max(1)])
    assert (np.abs(lhs - w).max(1) / scale).max() < 1e-6
    # Mx is the symmetric positive definite task-space inertia
    np.testing.assert_allclose(Mx, Mx.transpose(0, 2, 1), rtol=1e-9, atol=1e-9 * np.abs(Mx).max())
    assert (np.linalg.eigvalsh((Mx + Mx.transpose(0, 2, 1)) / 2) > 0).all()


@pytest.mark.parametrize("case", ["panda_mdh", "three_joint", "singular"])
def test_oracle_pinv_rows_satisfy_the_penrose_conditions(case):
    rng = np.random.default_rng(7)
    if case == "panda_mdh":
        chain = orc.Chain(ch.dh_to_ets(ch.panda_mdh_links(), mdh=True, tool=ch.panda_mdh_tool()))
        Ja = ops.ja(chain, rng.uniform(-2, 2, (50, 7)))
    elif case == "three_joint":
        chain = orc.Chain(ch.dh_to_ets(ch.ur10_links()[:3]))
        Ja = ops.ja(chain, rng.uniform(-2, 2, (50, 3)))
    else:  # exactly rank deficient: a zero column
        chain, _ = _dh_robot("puma")
        Ja = ops.ja(chain, rng.uniform(-2, 2, (50, 6)))
        Ja[:, :, 2] = 0
    X = ops.ji(Ja, pinv=True)
    AX, XA = Ja @ X, X @ Ja
    tol = 1e-9
    for got, want in ((AX @ Ja, Ja), (XA @ X, X), (AX.transpose(0, 2, 1), AX), (XA.transpose(0, 2, 1), XA)):
        assert np.abs(got - want).max() <= tol * max(1.0, np.abs(want).max())


def test_robot_methods_refuse_what_the_kernels_cannot_serve_before_launching():
    panda = rtb.models.PandaMDH()
    with pytest.raises(np.linalg.LinAlgError):  # numpy's inv of a 6x7 Jacobian
        panda.inertia_x(panda.qr)
    with pytest.raises(np.linalg.LinAlgError):
        panda.accel_x(panda.qr, np.zeros(6), np.zeros(6))
    # a tree robot whose joint groups are not in q order: the torque columns and the Jacobian columns would not match
    ET, ETS, Link = rtb.ET, rtb.ETS, rtb.Link
    links, parent = [], None
    for k, (ji, kind) in enumerate(((2, "Rz"), (0, "Ry"), (1, "Ry"))):
        parent = Link(ETS(ET.tx(0.3)) * getattr(ET, kind)(jindex=ji), name=f"l{k}", parent=parent, jindex=ji, m=1.0, r=[0.1, 0, 0])
        links.append(parent)
    rob = rtb.Robot(links)
    assert list(rob.tree_description()["jindex"]) == [2, 0, 1]
    for call in (lambda: rob.inertia_x(np.zeros(3), pinv=True), lambda: rob.gravload_x(np.zeros(3), pinv=True),
                 lambda: rob.coriolis_x(np.zeros(3), np.zeros(3), pinv=True),
                 lambda: rob.accel_x(np.zeros(3), np.zeros(6), np.zeros(6), pinv=True)):
        with pytest.raises(ValueError, match="q order"):
            call()
