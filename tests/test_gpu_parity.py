"""GPU parity tests: the CUDA path (through the C ABI) against
  (1) the committed golden fixtures produced by the compiled reference (tests/golden/*.npz),
  (2) the literal KATs of the reference's own tests (tests/golden/reference_kats.json),
  (3) the CPU oracle on fresh seeded inputs, including ragged / edge sizes,
  (4) size-independent properties at BASELINE.json's full sizes (1M rows).
Tolerances (BASELINE.json north_star): fp64 rtol 1e-10 (+ atol 1e-12: analytically-zero entries
come out as +-1e-17, see the golden 1.29e-16 at reference tests/test_ETS.py:330); fp32 rtol 1e-4,
atol 1e-5.
"""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import chains as ch  # noqa: E402
from oracle import oracle as orc  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")
KAT = json.load(open(os.path.join(G, "reference_kats.json")))
TOL = {np.float64: dict(rtol=1e-10, atol=1e-12), np.float32: dict(rtol=1e-4, atol=1e-5)}
AX = ["Rx", "Ry", "Rz", "tx", "ty", "tz"]


# Fraction of rows whose (success, iterations, searches) must equal the reference's / the oracle's sequential loop.
# Not 1.0: the kernel solves the LM normal equations by Cholesky where the reference forms A.inverse() (ik.cpp:171), and
# contracts a*b+c into FMAs; a row whose residual lands within rounding of `tol`, or which passes close to a singular
# configuration, can take one iteration more or less (scripts/ik_diff.py lists the rows; DESIGN 3.5).
IK_COUNTER_PARITY = 0.97


def ets_from_desc(z, p=""):
    """Rebuild a product ETS from a fixture's neutral chain description."""
    ets = []
    m = len(z[p + "isjoint"])
    for i in range(m):
        if z[p + "isjoint"][i]:
            ets.append(rtb.ET(AX[int(z[p + "axis"][i])], flip=bool(z[p + "flip"][i]), jindex=int(z[p + "jindex"][i]),
                              qlim=z[p + "qlim"][i]))
        else:
            ets.append(rtb.ET.SE3(z[p + "T"][i]))
    return rtb.ETS(ets)


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def host(t):
    return t.cpu().numpy()


def opt(a):
    return None if a.size == 0 else a


def ref_inputs(Q, dt):
    """fp32 runs are compared on the fp32-rounded inputs (the rounding of q is not the kernel's error)."""
    return Q.astype(dt).astype(np.float64)


# ------------------------------------------------------------------ KATs of the reference's own tests
def test_kat_panda_pose_and_jacobian():
    panda = rtb.models.Panda()
    q = np.array(KAT["panda_fkine"]["q"])
    np.testing.assert_array_almost_equal(panda.fkine(q).A, np.array(KAT["panda_fkine"]["T"]), decimal=6)
    ans = np.array(KAT["panda_jacob0"]["J"])
    # the reference accepts q as list, 1-D, (1,n) and (n,1) (tests/test_ETS.py:295-359)
    for qq in (q, list(q), q[None, :], q[:, None]):
        J = panda.jacob0(qq)
        assert J.shape == (6, 7)
        np.testing.assert_array_almost_equal(J, ans, decimal=6)
    with pytest.raises(TypeError):
        panda.ets().jacob0("Wfgsrth")
    # jacobe == tr2jac(T^T) @ jacob0 (tests/test_ETS.py:365-398)
    T = panda.ets().eval(q)
    blk = np.zeros((6, 6)); blk[:3, :3] = T[:3, :3].T; blk[3:, 3:] = T[:3, :3].T
    np.testing.assert_array_almost_equal(panda.jacobe(q), blk @ panda.jacob0(q))


def test_kat_puma_rne():
    puma = rtb.models.Puma560()
    for c in KAT["puma560_rne"]["cases"]:
        tau = puma.rne(puma.qn, np.full(6, float(c["qd"])), np.full(6, float(c["qdd"])), gravity=c.get("gravity"),
                       fext=c.get("fext"))
        assert tau.shape == (6,)
        np.testing.assert_array_almost_equal(tau, np.array(c["tau"], dtype=float), decimal=4)
    # trajectory form (tests/test_DHRobot.py:1065-1076) and delete / re-init (1078-1090)
    z, o = np.zeros(6), np.ones(6)
    t = puma.rne(np.c_[puma.qn, puma.qn].T, np.c_[z, o].T, np.c_[z, o].T)
    np.testing.assert_array_almost_equal(t[0], KAT["puma560_rne"]["cases"][0]["tau"], decimal=4)
    np.testing.assert_array_almost_equal(t[1], KAT["puma560_rne"]["cases"][2]["tau"], decimal=4)
    puma.delete_rne()
    np.testing.assert_array_almost_equal(puma.rne(puma.qn, z, z), KAT["puma560_rne"]["cases"][0]["tau"], decimal=4)


def test_kat_ik_converges():
    """tests/test_IK.py:186-251, 451-492, 632-708: success + small residual for all three methods."""
    panda = rtb.models.Panda()
    Tep = panda.fkine(panda.qr).A
    for method, k in (("chan", 1.0), ("sugihara", 0.1), ("wampler", 0.01)):
        q, ok, it, sr, E = panda.ik_LM(Tep, method=method, k=k)
        assert ok == 1 and E < 1e-5 and q.shape == (7,)
        assert np.abs(panda.fkine(q).A - Tep).max() < 5e-3
        sol = panda.ikine_LM(Tep, method=method, k=k, seed=0)
        assert sol.success and sol.residual < 1e-5
        assert np.abs(panda.fkine(sol.q).A - Tep).max() < 5e-3
    puma = rtb.models.Puma560()
    T = puma.fkine(puma.qn).A
    sol = puma.ikine_LM(T, seed=0)  # tests/test_DHRobot.py:965-972
    assert sol.success
    np.testing.assert_array_almost_equal(puma.fkine(sol.q).A, T, decimal=4)


# ------------------------------------------------------------------ fixtures from the compiled reference
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["panda_fkj.npz", "ur10_fkj.npz"])
def test_fixture_fkj(name, dt):
    z = np.load(os.path.join(G, name))
    e = ets_from_desc(z)
    Q = z["Q"]
    if dt == np.float32:
        keep = np.abs(Q).max(axis=1) < 100  # fp32 cannot even represent the 1e6-rad row's angles
        Q = Q[keep]
        C = orc.Chain({k: z[k] for k in ("isjoint", "axis", "flip", "jindex", "T", "qlim")})
        Qr = ref_inputs(Q, dt)
        Tr, J0r, Jer = C.fkine(Qr), C.jacob0(Qr), C.jacobe(Qr)
    else:
        Tr, J0r, Jer = z["Tfk"], z["J0"], z["Je"]
    q = dev(Q, dt)
    np.testing.assert_allclose(host(e.eval(q)), Tr, **TOL[dt])
    np.testing.assert_allclose(host(e.jacob0(q)), J0r, **TOL[dt])
    np.testing.assert_allclose(host(e.jacobe(q)), Jer, **TOL[dt])
    T, J = e.fkine_jacob0(q)
    np.testing.assert_allclose(host(T), Tr, **TOL[dt])
    np.testing.assert_allclose(host(J), J0r, **TOL[dt])


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_fixture_random_chains(dt):
    """All six ET kinds, flips, SE3 constants, n = 1..10, base and tool."""
    z = np.load(os.path.join(G, "random_fkj.npz"))
    for c in range(int(z["nchains"])):
        p = f"c{c}_"
        e = ets_from_desc(z, p)
        base, tool = opt(z[p + "base"]), opt(z[p + "tool"])
        Q = z[p + "Q"]
        if dt == np.float32:
            C = orc.Chain({k: z[p + k] for k in ("isjoint", "axis", "flip", "jindex", "T", "qlim")})
            Qr = ref_inputs(Q, dt)
            Tr, J0r, Jer = C.fkine(Qr, base, tool), C.jacob0(Qr, tool), C.jacobe(Qr, tool)
        else:
            Tr, J0r, Jer = z[p + "Tfk"], z[p + "J0"], z[p + "Je"]
        q = dev(Q, dt)
        tol = dict(TOL[dt])
        if dt == np.float64:
            tol["atol"] = 1e-11  # chains with |t| up to ~5: scale the absolute floor with the reach
        np.testing.assert_allclose(host(e.eval(q, base=base, tool=tool)), Tr, err_msg=f"chain {c}", **tol)
        np.testing.assert_allclose(host(e.jacob0(q, tool=tool)), J0r, err_msg=f"chain {c}", **tol)
        np.testing.assert_allclose(host(e.jacobe(q, tool=tool)), Jer, err_msg=f"chain {c}", **tol)
        T, J = e.fkine_jacob0(q, base=base, tool=tool)
        np.testing.assert_allclose(host(T), Tr, err_msg=f"chain {c}", **tol)
        np.testing.assert_allclose(host(J), J0r, err_msg=f"chain {c}", **tol)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_fixture_rne(dt):
    tol = dict(rtol=1e-10, atol=1e-10) if dt == np.float64 else dict(rtol=2e-4, atol=2e-3)
    z = np.load(os.path.join(G, "puma_rne.npz"))
    puma = rtb.models.Puma560()
    a = [dev(z[k], dt) for k in ("q", "qd", "qdd")]
    if dt == np.float32:  # compare on the rounded inputs
        L = puma._pack_rne()
        qq = [ref_inputs(z[k], dt) for k in ("q", "qd", "qdd")]
        want = [orc.rne(6, 0, L, -z["gravity"], *qq), orc.rne(6, 0, L, -z["gravity"], *qq, z["fext"]),
                orc.rne(6, 0, L, np.zeros(3), *qq), orc.rne(6, 0, L, -z["g2"], *qq, z["fext"])]
    else:
        want = [z["tau"], z["tau_fext"], z["tau_zerog"], z["tau_g2"]]
    np.testing.assert_allclose(host(puma.rne(*a)), want[0], **tol)
    np.testing.assert_allclose(host(puma.rne(*a, fext=z["fext"])), want[1], **tol)
    np.testing.assert_allclose(host(puma.rne(*a, gravity=[0, 0, 0])), want[2], **tol)
    np.testing.assert_allclose(host(puma.rne(*a, gravity=z["g2"], fext=z["fext"])), want[3], **tol)
    if dt == np.float64:
        z = np.load(os.path.join(G, "panda_mdh_rne.npz"))
        pm = rtb.models.PandaMDH()
        a = [dev(z[k]) for k in ("q", "qd", "qdd")]
        np.testing.assert_allclose(host(pm.rne(*a)), z["tau"], **tol)
        np.testing.assert_allclose(host(pm.rne(*a, fext=z["fext"])), z["tau_fext"], **tol)


def test_fixture_rne_random_links():
    """Random DH / MDH robots with prismatic joints, offsets, friction -- reference frne outputs."""
    z = np.load(os.path.join(G, "random_rne.npz"))
    for c in range(int(z["ncases"])):
        p = f"c{c}_"
        L = z[p + "L"].reshape(-1, 24)
        mdh = bool(int(z[p + "mdh"]))
        links = []
        for l in L:
            links.append(rtb.DHLink(alpha=l[0], a=l[1], theta=l[2], d=l[3], sigma=int(l[4]), offset=l[5], mdh=mdh,
                                    m=l[6], r=l[7:10], I=l[10:19].reshape(3, 3), Jm=l[19], G=l[20], B=l[21], Tc=l[22:24]))
        rob = rtb.DHRobot(links, gravity=z[p + "gravity"])
        tau = rob.rne(dev(z[p + "q"]), dev(z[p + "qd"]), dev(z[p + "qdd"]), fext=z[p + "fext"])
        np.testing.assert_allclose(host(tau), z[p + "tau"], rtol=1e-9, atol=1e-9, err_msg=f"case {c}")


def test_dynamics_fanouts():
    """inertia / gravload / itorque / coriolis / accel (SURVEY 8f-1): reference KATs
    (tests/test_DHRobot.py:1092-1200), the fixture produced through the compiled frne, and the oracle on
    a larger random batch incl. an MDH robot and a robot with prismatic joints."""
    k = KAT["puma560_dynamics"]
    puma = rtb.models.Puma560()
    qn = puma.qn
    dec = k["decimal"]
    M = puma.inertia(qn)
    assert M.shape == (6, 6)
    np.testing.assert_array_almost_equal(M, np.array(k["inertia"]), decimal=dec)
    np.testing.assert_array_almost_equal(puma.gravload(qn), np.array(k["gravload"], dtype=float), decimal=dec)
    np.testing.assert_array_almost_equal(puma.itorque(qn, k["itorque"]["qdd"]), k["itorque"]["taui"], decimal=dec)
    np.testing.assert_array_almost_equal(puma.coriolis(qn, k["coriolis"]["qd"]), np.array(k["coriolis"]["C"], dtype=float), decimal=dec)
    np.testing.assert_array_almost_equal(puma.accel(qn, k["accel"]["qd"], k["accel"]["torque"]), k["accel"]["qdd"], decimal=dec)
    q2 = np.c_[qn, qn].T  # trajectory forms of the same tests
    a2 = puma.accel(q2, np.tile(k["accel"]["qd"], (2, 1)), np.tile(k["accel"]["torque"], (2, 1)))
    assert a2.shape == (2, 6)
    np.testing.assert_array_almost_equal(a2[1], k["accel"]["qdd"], decimal=dec)
    assert puma.coriolis(q2, np.tile(k["coriolis"]["qd"], (2, 1))).shape == (2, 6, 6)
    z = np.load(os.path.join(G, "puma_dynamics.npz"))
    tol = dict(rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(host(puma.inertia(dev(z["q"]))), z["inertia"], **tol)
    np.testing.assert_allclose(host(puma.gravload(dev(z["q"]))), z["gravload"], **tol)
    np.testing.assert_allclose(host(puma.itorque(dev(z["q"]), dev(z["qdd"]))), z["itorque"], **tol)
    np.testing.assert_allclose(host(puma.coriolis(dev(z["q"]), dev(z["qd"]))), z["coriolis"], **tol)
    np.testing.assert_allclose(host(puma.accel(dev(z["q"]), dev(z["qd"]), dev(z["torque"]))), z["accel"], rtol=1e-9, atol=1e-9)
    # larger batches against the oracle: MDH Panda (n=7), and a DH robot with prismatic joints
    rng = np.random.default_rng(31)
    robots = [rtb.models.PandaMDH(),
              rtb.DHRobot([rtb.RevoluteDH(d=0.3, a=0.1, alpha=1.2, m=2, r=[0.1, 0, 0.05], I=[0.1, 0.2, 0.15], Jm=1e-4, G=50, B=1e-3, Tc=[0.1, -0.2]),
                           rtb.PrismaticDH(theta=0.4, a=0.2, alpha=-0.7, m=1.5, r=[0, 0.1, 0], I=[0.05, 0.04, 0.03], Jm=2e-4, G=30, B=2e-3, Tc=[0.05, -0.05]),
                           rtb.RevoluteDH(d=0.1, a=0.25, alpha=0.0, m=1, r=[0.05, 0.02, 0], I=[0.02, 0.03, 0.01], Jm=1e-4, G=-40, B=1e-3, Tc=[0.02, -0.03])])]
    for rob in robots:
        n = rob.n
        L = rob._pack_rne()
        mdh = rob.mdh
        g = rob.gravity
        f = lambda q, qd, qdd, grav: orc.rne(n, mdh, L, -np.asarray(grav, dtype=float), q, qd, qdd)  # noqa: E731
        Lnf = orc.nofriction_L(L)
        fnf = lambda q, qd, qdd, grav: orc.rne(n, mdh, Lnf, -np.asarray(grav, dtype=float), q, qd, qdd)  # noqa: E731
        N = 333
        q = rng.uniform(-2, 2, (N, n)); qd = rng.normal(size=(N, n)); qdd = rng.normal(size=(N, n)); tq = rng.normal(size=(N, n))
        np.testing.assert_allclose(host(rob.inertia(dev(q))), orc.dyn_inertia(f, n, q), **tol)
        np.testing.assert_allclose(host(rob.gravload(dev(q))), orc.dyn_gravload(f, n, q, g), **tol)
        np.testing.assert_allclose(host(rob.itorque(dev(q), dev(qdd))), orc.dyn_itorque(f, n, q, qdd), **tol)
        np.testing.assert_allclose(host(rob.coriolis(dev(q), dev(qd))), orc.dyn_coriolis(fnf, n, q, qd), **tol)
        np.testing.assert_allclose(host(rob.accel(dev(q), dev(qd), dev(tq))), orc.dyn_accel(f, n, q, qd, tq, g), rtol=1e-8, atol=1e-8)
        # structural properties: M symmetric positive definite; itorque == M qdd; rne == M qdd + C qd + g + friction
        Mq = host(rob.inertia(dev(q)))
        np.testing.assert_allclose(Mq, Mq.transpose(0, 2, 1), atol=1e-10)
        assert (np.linalg.eigvalsh(Mq) > 0).all()
        np.testing.assert_allclose(host(rob.itorque(dev(q), dev(qdd))), np.einsum("kij,kj->ki", Mq, qdd), atol=1e-9)
    # fp32 runs
    M32 = host(puma.inertia(dev(z["q"], np.float32)))
    np.testing.assert_allclose(M32, z["inertia"], rtol=2e-4, atol=2e-4)


def test_hessian_and_manipulability():
    """hessian0 / hessiane / manipulability (SURVEY 8f-2): fknm.ETS_hessian0/e fixture, the reference test's
    literal golden (tests/test_ETS.py:718-1128: q as array, list, (1,n), (n,1) and J0=J), and the oracle."""
    z = np.load(os.path.join(G, "panda_hessian.npz"))
    e = ets_from_desc(z)
    tol = dict(rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(e.hessian0(dev(z["Q"]))), z["H0"], **tol)
    np.testing.assert_allclose(host(e.hessiane(dev(z["Q"]))), z["He"], **tol)
    np.testing.assert_allclose(host(e.hessian0(dev(z["Q"]), tool=z["tool"])), z["H0_tool"], **tol)
    np.testing.assert_allclose(host(e.hessian0(J0=dev(z["J0"]))), z["H0"], **tol)
    q1 = z["Q"][0]
    ans = z["kat_hessian0_q1"]
    for qq in (q1, list(q1), q1[None, :], q1[:, None]):
        H = e.hessian0(qq)
        assert H.shape == (7, 6, 7)
        np.testing.assert_array_almost_equal(H, ans, decimal=6)
    np.testing.assert_array_almost_equal(e.hessian0(J0=e.jacob0(q1)), ans, decimal=6)
    with pytest.raises(ValueError):
        e.hessian0()
    H32 = host(e.hessian0(dev(z["Q"], np.float32)))
    np.testing.assert_allclose(H32, z["H0"], rtol=1e-4, atol=1e-5)
    # manipulability (yoshikawa) for all / trans / rot / explicit axes, and the square case on a 6-joint arm
    J = z["J0"]
    for axes, mask in (("all", [1] * 6), ("trans", [1, 1, 1, 0, 0, 0]), ("rot", [0, 0, 0, 1, 1, 1]), ([1, 0, 1, 0, 1, 1], [1, 0, 1, 0, 1, 1])):
        want = np.array([orc.yoshikawa(Jk, mask) for Jk in J])
        np.testing.assert_allclose(host(e.manipulability(dev(z["Q"]), axes=axes)), want, rtol=1e-9, atol=1e-12)
    assert isinstance(e.manipulability(q1), float)
    ur = rtb.models.UR10().ets()
    Q6 = np.random.default_rng(6).uniform(-3, 3, (50, 6))
    J6 = host(ur.jacob0(dev(Q6)))
    np.testing.assert_allclose(host(ur.manipulability(dev(Q6))), [orc.yoshikawa(Jk) for Jk in J6], rtol=1e-9, atol=1e-12)
    with pytest.raises(ValueError):
        e.manipulability(q1, method="asada")
    # manipulability Jacobian: reference test literal (tests/test_ERobot.py:28-52: q as array, list, (1,n), (n,1), J=)
    kat = KAT["panda_jacobm"]
    pe = rtb.models.Panda().ets()
    qk = np.array(kat["q"])
    for qq in (qk, list(qk), qk[None, :], qk[:, None]):
        Jm = pe.jacobm(qq)
        assert Jm.shape == (7, 1)
        np.testing.assert_array_almost_equal(Jm.ravel(), kat["Jm"], decimal=kat["decimal"])
    np.testing.assert_array_almost_equal(pe.jacobm(J=pe.jacob0(qk)).ravel(), kat["Jm"], decimal=kat["decimal"])
    with pytest.raises(TypeError):
        pe.jacobm([1, 3], "qwe")
    with pytest.raises(TypeError):
        pe.jacobm("Wfgsrth")
    with pytest.raises(ValueError):
        pe.jacobm(qk, axes="abcdef")
    sel = np.abs(np.linalg.det(z["J0"] @ z["J0"].transpose(0, 2, 1))) > 1e-8  # away from singular configurations
    for axes, mask in (("all", [1] * 6), ("trans", [1, 1, 1, 0, 0, 0]), ("rot", [0, 0, 0, 1, 1, 1])):
        want = np.stack([orc.jacobm(Jk, Hk, mask).ravel() for Jk, Hk in zip(z["J0"], z["H0"])])
        got = host(e.jacobm(dev(z["Q"]), axes=axes))
        np.testing.assert_allclose(got[sel], want[sel], rtol=1e-7, atol=1e-10)
    np.testing.assert_allclose(host(rtb.models.Panda().jacobm(dev(z["Q"]), axes="trans")),
                               host(e.jacobm(J=dev(z["J0"]), axes="trans")), rtol=1e-9, atol=1e-12)
    # Jacobian time derivative = tensordot(hessian0, qd) (Robot.py:1099)
    QD = np.random.default_rng(8).normal(size=z["Q"].shape)
    want = np.stack([orc.jacob_dot(Hk, v) for Hk, v in zip(z["H0"], QD)])
    np.testing.assert_allclose(host(e.jacob0_dot(dev(z["Q"]), dev(QD))), want, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(e.jacob0_dot(z["Q"][2], QD[2]), want[2], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(e.jacob0_dot(dev(z["Q"], np.float32), dev(QD, np.float32))), want, rtol=2e-4, atol=2e-4)
    puma = rtb.models.Puma560()
    assert puma.jacob0_dot(puma.qn, [0.1, -0.2, 0.3, -0.4, 0.5, -0.6]).shape == (6, 6)
    assert abs(puma.manipulability(puma.qn) - 0.0786) < 1e-4  # tests/test_DHRobot.py:1262-1279
    assert abs(puma.manipulability(puma.qn, axes="trans") - 0.111181) < 1e-4
    assert abs(puma.manipulability(puma.qn, axes="rot") - 2.44949) < 1e-4


def test_fixture_ik_fp64_explicit_q0():
    """Row i of the batch == the reference called on target i: explicit q0, slimit=1, fp64."""
    z = np.load(os.path.join(G, "panda_ik.npz"))
    e = rtb.models.Panda().ets()
    Tep, q0 = dev(z["Tep"]), dev(z["q0"])
    for tag, method, k in (("chan1", "chan", 1.0), ("chan01", "chan", 0.1), ("sugi", "sugihara", 1e-4)):
        q, s, it, sr, E = (host(x) for x in e.ik_LM(Tep, q0=q0, slimit=1, joint_limits=False, k=k, method=method))
        same = (s == z[tag + "_success"]) & (it == z[tag + "_it"]) & (sr == z[tag + "_search"])
        assert same.all(), f"{tag}: rows {np.nonzero(~same)[0]} do not reproduce the reference's counters"
        ok = same & (s == 1)
        np.testing.assert_allclose(q[ok], z[tag + "_q"][ok], atol=1e-7)
        np.testing.assert_allclose(E[ok], z[tag + "_E"][ok], atol=1e-11)
    # fmod wrap + joint-limit rejection (ik.cpp:50-52)
    q, s, it, sr, E = (host(x) for x in e.ik_LM(Tep, q0=q0, slimit=1, joint_limits=True, k=1.0))
    assert ((s == z["jl_success"]) & (it == z["jl_it"])).all()
    # masked (position-only) solve
    q, s, it, sr, E = (host(x) for x in e.ik_LM(Tep, q0=q0, slimit=1, joint_limits=False, mask=z["mask"], k=1.0))
    assert (s == z["mask_success"]).mean() >= 0.95
    pos_err = np.abs(orc.Chain(e.describe()).fkine(q)[:, :3, 3] - z["Tep"][:, :3, 3]).max(axis=1)
    assert (pos_err[s == 1] < 5e-3).all()


IKNR_CASES = [("nr_d", "nr", 0.1, False), ("nr_d_mask", "nr", 0.1, True), ("nr", "nr", 0.0, False),
              ("gn", "gn", 0.0, False), ("gn_mask", "gn", 0.0, True), ("nr_inv", "nr", 0.0, False)]


def test_fixture_ik_nr_gn():
    """fknm.IK_NR_c / IK_GN_c (explicit q0, slimit=1, fp64) on Panda (n=7), UR10 (n=6) and a 3-joint chain:
    damped Newton-Raphson reproduces the reference row for row; undamped runs (chaotic near singular
    configurations, and the kernel uses a 6x6 Cholesky where the reference uses an SVD) are held to outcome
    statistics, to the well-started half of the batch, and to the oracle."""
    z = np.load(os.path.join(G, "ik_nr_gn.npz"))
    for name in ("panda", "ur10", "ur3"):
        e = ets_from_desc(z, name + "_")
        C = orc.Chain(e.describe())
        Tep, q0 = z[name + "_Tep"], z[name + "_q0"]
        half = len(Tep) // 2
        for tag, meth, damp, masked in IKNR_CASES:
            if f"{name}_{tag}_q" not in z:
                continue
            mask = z["mask"] if masked else None
            fn = e.ik_GN if meth == "gn" else e.ik_NR
            q, s, it, sr, E = (host(x) for x in fn(dev(Tep), q0=dev(q0), slimit=1, joint_limits=False, mask=mask,
                                                    pinv_damping=damp))
            rs, rit, rq = z[f"{name}_{tag}_success"], z[f"{name}_{tag}_it"], z[f"{name}_{tag}_q"]
            want = C.ik_lm(Tep, q0, 30, 1, 1e-6, False, mask, damp, meth)
            if damp > 0:
                same = (s == rs) & (it == rit)
                assert same.mean() >= 0.99, (name, tag, same.mean())
                ok = same & (s == 1)
                np.testing.assert_allclose(q[ok], rq[ok], atol=1e-7)
                np.testing.assert_allclose(E[ok], z[f"{name}_{tag}_E"][ok], atol=1e-11)
                assert ((s == want[1]) & (it == want[2])).mean() >= 0.99
            else:
                assert abs(s.mean() - rs.mean()) < 0.06, (name, tag, s.mean(), rs.mean())
                assert abs(s.mean() - want[1].mean()) < 0.06, (name, tag, s.mean(), want[1].mean())
                near = ((s == rs) & (it == rit))[:half]
                assert near.mean() >= 0.9, (name, tag, near.mean())
            okr = s == 1  # whatever path it took, a reported success is a solution
            Tq = C.fkine(q[okr])
            if not masked:
                assert np.abs(Tq - Tep[okr]).max() < 5e-3
            else:
                assert np.abs(Tq[:, :3, 3] - Tep[okr][:, :3, 3]).max() < 5e-3


def test_ik_nr_gn_restarts_and_python_semantics():
    """Multi-start Newton-Raphson / Gauss-Newton (both loops, both precisions) against the oracle run with
    the same counter-based restart stream, plus the solver-class entry points."""
    e = rtb.models.Panda().ets()
    C = orc.Chain(e.describe())
    rng = np.random.default_rng(4)
    qs = rng.uniform(-2.8, 2.8, (1500, 7))
    Tep = C.fkine(qs)
    for sem in (0, 1):
        for meth, code in (("nr", rtb._lib.IK_NR), ("gn", rtb._lib.IK_GN)):
            damp = 0.1 if meth == "nr" else 0.0
            want = C.ik_lm(Tep, None, 30, 20, 1e-6, True, None, damp, meth, seed=9, semantics=sem, rng_per_row=True)
            got = e._ik(dev(Tep), None, 30, 20, 1e-6, None, True, damp, code, 9, sem, True, None)[:5]
            q, s, it, sr, E = (host(x) for x in got)
            assert abs(s.mean() - want[1].mean()) < 0.02, (sem, meth, s.mean(), want[1].mean())
            if damp > 0:
                same = (s == want[1]) & (it == want[2]) & (sr == want[3])
                assert same.mean() >= 0.97, (sem, meth, same.mean())
                ok = same & (s == 1)
                np.testing.assert_allclose(q[ok], want[0][ok], atol=1e-6)
            ok = s == 1
            # the C++ loop returns the q it tested (E < tol <=> |e| < 1.4e-3); the Python loop returns q AFTER one more
            # step (IK.py:314-348), which for a pseudo-inverse step near a singularity can move the pose by ~1e-2
            assert np.abs(C.fkine(q[ok]) - Tep[ok]).max() < (5e-3 if sem == 0 else 5e-2)
            assert (np.abs(q[ok]) <= np.pi + 1e-9).all()
    q32, s32, *_ = (host(x) for x in e.ik_NR(dev(Tep, np.float32), pinv_damping=0.1, seed=2))
    assert s32.mean() > 0.99
    sol = rtb.IK_NR(seed=3).solve(e, Tep[:200])
    assert sol.q.shape == (200, 7) and sol.searches >= 200
    sol = rtb.IK_GN(seed=3, slimit=50).solve(rtb.models.Panda(), Tep[0])
    assert sol.q.shape == (7,)
    if sol.success:
        assert np.abs(C.fkine(sol.q[None])[0] - Tep[0]).max() < 5e-3
    ur = rtb.models.UR10()
    Tu = ur.eval(rng.uniform(-2, 2, (64, 6)))
    q, s, *_ = ur.ik_nr(Tu, None, 30, 100, 1e-6, False, None, True, 0.05)
    assert s.mean() > 0.95


def test_ik_restarts_match_oracle_stream():
    """With the documented counter-based restart generator the whole multi-start run is
    reproducible: same (seed,row,search,joint) draws as oracle_kin.c, so counters agree."""
    z = np.load(os.path.join(G, "panda_ik.npz"))
    e = rtb.models.Panda().ets()
    C = orc.Chain(e.describe())
    for sem, fn in ((0, "ik"), (1, "ikine")):
        for jl in (True, False):
            want = C.ik_lm(z["Tep"], q0=None, joint_limits=jl, k=1.0, seed=7, semantics=sem, rng_per_row=True)
            got = e._ik(dev(z["Tep"]), None, 30, 100, 1e-6, None, jl, 1.0, "chan", 7, sem, True, None)[:5]
            q, s, it, sr, E = (host(x) for x in got)
            assert s.mean() == want[1].mean() == 1.0
            same = (it == want[2]) & (sr == want[3])
            assert same.mean() >= 0.97, f"sem {sem} jl {jl}: {same.mean():.3f}"
            np.testing.assert_allclose(q[same], want[0][same], atol=1e-6)
    # reference statistics with its own (unseeded) restarts: same success rate, similar search count
    q, s, it, sr, E = (host(x) for x in e.ik_LM(dev(z["Tep"]), joint_limits=True, k=1.0, seed=3))
    assert s.mean() == z["rs_success"].mean() == 1.0
    assert abs(sr.mean() - z["rs_search"].mean()) < 0.5


def test_ik_two_phase_restarts_equal_sequential_semantics():
    """Batches >= 1024 run the restarts of hard problems in parallel (8 searches at a time per problem,
    csrc/b2k_ik.cuh k_ik_restarts).  Because the restart draws are counter-based this must report
    exactly what the sequential loops report: compare against the oracle's sequential run."""
    z = np.load(os.path.join(G, "panda_ik.npz"))
    e = rtb.models.Panda().ets()
    C = orc.Chain(e.describe())
    Tep = np.tile(z["Tep"], (8, 1, 1))  # 1536 targets: same poses, different rows -> different restart draws
    for sem in (0, 1):
        for jl, slimit, ilimit in ((True, 100, 30), (True, 3, 10), (False, 20, 15)):
            want = C.ik_lm(Tep, q0=None, ilimit=ilimit, slimit=slimit, joint_limits=jl, k=1.0, seed=21, semantics=sem,
                           rng_per_row=True)
            got = e._ik(dev(Tep), None, ilimit, slimit, 1e-6, None, jl, 1.0, "chan", 21, sem, True, None)[:5]
            q, s, it, sr, E = (host(x) for x in got)
            assert (s == want[1]).mean() >= 0.995, (sem, jl, slimit)
            same = (s == want[1]) & (it == want[2]) & (sr == want[3])
            assert same.mean() >= 0.97, f"sem {sem} jl {jl} slimit {slimit}: {same.mean():.3f}"
            ok = same & (s == 1)
            np.testing.assert_allclose(q[ok], want[0][ok], atol=1e-6)
            fail = same & (s == 0)
            if fail.any():  # failures report the same leftover q / residual as the sequential loop
                np.testing.assert_allclose(q[fail], want[0][fail], atol=1e-6)
                np.testing.assert_allclose(E[fail], want[4][fail], rtol=1e-6, atol=1e-9)


def test_ik_fp32_outcomes():
    """Config 4 protocol at reduced size: fp32, reachable targets, chan k=0.1 and k=1.0."""
    e = rtb.models.Panda().ets()
    C = orc.Chain(e.describe())
    rng = np.random.default_rng(2)
    qs = rng.uniform(-np.pi, np.pi, (20000, 7))
    Tep = C.fkine(qs)
    for k, jl in ((0.1, False), (1.0, True)):
        q, s, it, sr, E = (host(x) for x in e.ik_LM(dev(Tep, np.float32), joint_limits=jl, k=k, seed=5))
        assert s.mean() > 0.999
        ok = s == 1
        assert (E[ok] < 1e-6).all()
        err = np.abs(C.fkine(q.astype(np.float64)) - Tep).max(axis=(1, 2))
        assert np.percentile(err[ok], 99.9) < 5e-3  # E < 1e-6 <=> ||e|| < 1.4e-3
        if jl:
            assert (np.abs(q[ok]) <= np.pi + 1e-6).all()
    sol = e.ikine_LM(Tep[:500].astype(np.float32), seed=1)
    assert sol.success and sol.q.shape == (500, 7) and sol.searches >= 500


def test_config4_full_size_100k():
    """BASELINE config 4 at full size: 100 000 reachable Panda targets (Tep = FK(q*), q* ~ U(-pi, pi), seed 2), fp32,
    ilimit 30, slimit 100, tol 1e-6, both protocols of SURVEY 8d (notebook: chan 0.1 without the limit check; API
    default: chan 1.0 with it).  Every target must be solved, every solution must solve the pose, and -- the restart
    stream being counter-based -- the fp64 run must report the oracle's sequential-loop counters on a sampled subset."""
    e = rtb.models.Panda().ets()
    C = orc.Chain(e.describe())
    N = 100_000
    qs = np.random.default_rng(2).uniform(-np.pi, np.pi, (N, 7))
    Tep = C.fkine(qs)
    for k, jl in ((0.1, False), (1.0, True)):
        q, s, it, sr, E = (host(x) for x in e.ik_LM(dev(Tep, np.float32), joint_limits=jl, k=k, seed=5))
        assert s.all(), f"k={k}: {int((s == 0).sum())} of {N} targets unsolved"
        assert (E < 1e-6).all()
        err = np.abs(C.fkine(q.astype(np.float64)) - Tep).max(axis=(1, 2))
        assert err.max() < 5e-3  # E < 1e-6 <=> |e| < 1.5e-3; fp32 FK noise on top
        if jl:
            assert (np.abs(q) <= np.pi + 1e-6).all()
        # fp64, same seed: counters of the sequential reference loop, row for row, on a subset (oracle: ~30 us / solve)
        q64, s64, it64, sr64, E64 = (host(x) for x in e.ik_LM(dev(Tep), joint_limits=jl, k=k, seed=5))
        assert s64.all()
        # restart r of row i is keyed by (seed, i, r): the first M rows of the batch are rows 0..M-1 for the oracle too
        M = 3000
        wq, ws, wit, wsr, wE = C.ik_lm(Tep[:M], q0=None, joint_limits=jl, k=k, seed=5, semantics=0, rng_per_row=True)
        same = (s64[:M] == ws) & (it64[:M] == wit) & (sr64[:M] == wsr)
        assert same.mean() >= IK_COUNTER_PARITY, f"k={k}: {same.mean():.4f} of rows reproduce the sequential loop's counters"
        np.testing.assert_allclose(q64[:M][same], wq[same], atol=1e-4)  # both ends stop at E < tol: q agrees to ~sqrt(tol) at worst
        # iteration statistics of the fp32 run track the fp64 run (same problems, same draws up to rounding)
        assert abs(it.mean() - it64.mean()) < 0.05 * it64.mean()
        assert abs(sr.mean() - sr64.mean()) < 0.05 * sr64.mean()


# ------------------------------------------------------------------ oracle on fresh inputs, edge sizes
@pytest.mark.parametrize("N", [1, 2, 31, 32, 33, 1000, 100001])
def test_sizes_and_ragged_tiles(N):
    e = rtb.models.Panda().ets()
    C = orc.Chain(e.describe())
    Q = np.random.default_rng(N).uniform(-np.pi, np.pi, (N, 7))
    sq = (lambda a: a[0]) if N == 1 else (lambda a: a)  # a (1,n) q is ONE configuration (fknm.cpp:970-975)
    T, J = e.fkine_jacob0(dev(Q))
    np.testing.assert_allclose(host(T), sq(C.fkine(Q)), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(J), sq(C.jacob0(Q)), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(e.jacobe(dev(Q))), sq(C.jacobe(Q)), rtol=1e-10, atol=1e-12)
    for dt in (np.float32,):
        Qr = ref_inputs(Q, dt)
        T32, J32 = e.fkine_jacob0(dev(Q, dt))
        np.testing.assert_allclose(host(T32), sq(C.fkine(Qr)), **TOL[dt])
        np.testing.assert_allclose(host(J32), sq(C.jacob0(Qr)), **TOL[dt])
    puma = rtb.models.Puma560()
    q, qd, qdd = Q[:, :6], np.cos(Q[:, :6]), np.sin(Q[:, :6])
    want = orc.rne(6, 0, puma._pack_rne(), -puma.gravity, q, qd, qdd)
    if N == 1:  # rne keeps (N, n) for 2-D input (DHRobot.py:1416-1424)
        np.testing.assert_allclose(host(puma.rne(dev(q), dev(qd), dev(qdd))), want, rtol=1e-10, atol=1e-10)
    else:
        np.testing.assert_allclose(host(puma.rne(dev(q), dev(qd), dev(qdd))), want, rtol=1e-10, atol=1e-10)


def test_sincos_accuracy():
    """The in-house sincos (csrc/b2k_trig.cuh) against extended-precision libm."""
    L = rtb._lib.lib()
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-np.pi, np.pi, 400000), rng.uniform(-100, 100, 200000),
                        rng.uniform(-1e5, 1e5, 200000), rng.uniform(-1e9, 1e9, 1000),
                        np.array([0.0, -0.0, np.pi / 2, np.pi, -np.pi, 1e-300, 105614.9, 105615.1, 1e22])])
    ld = np.longdouble
    for dt, lim in ((np.float64, 2.0), (np.float32, 2.5)):
        xd = dev(x, dt)
        s, c = torch.empty_like(xd), torch.empty_like(xd)
        rtb._lib.check(L.b2k_selftest_sincos(0 if dt == np.float32 else 1, xd.data_ptr(), xd.numel(), s.data_ptr(),
                                             c.data_ptr(), torch.cuda.current_stream().cuda_stream))
        xr = host(xd).astype(ld)
        rs, rc = np.sin(xr), np.cos(xr)
        eps = np.finfo(dt).eps
        # error in ulps of the result, with an absolute floor of one ulp(1) near the zeros of sin / cos
        us = np.abs(host(s).astype(ld) - rs) / np.maximum(np.abs(rs) * eps, ld(eps) * eps)
        uc = np.abs(host(c).astype(ld) - rc) / np.maximum(np.abs(rc) * eps, ld(eps) * eps)
        small = np.abs(xr) < 100
        assert float(us[small].max()) < lim and float(uc[small].max()) < lim, (dt, float(us[small].max()), float(uc[small].max()))
        assert float(np.abs(host(s).astype(ld) - rs).max()) < 4 * eps and float(np.abs(host(c).astype(ld) - rc).max()) < 4 * eps


def test_empty_batch():
    e = rtb.models.Panda().ets()
    q = torch.empty((0, 7), dtype=torch.float64, device="cuda")
    assert tuple(e.eval(q).shape) == (0, 4, 4)
    assert tuple(e.jacob0(q).shape) == (0, 6, 7)


def test_wide_q_and_permuted_jindex():
    """q may be wider than n and jindices need not be 0..n-1 (reference methods.cpp:338, appendix C.13)."""
    ET = rtb.ET
    e = ET.Rz(jindex=4) * ET.tx(0.3) * ET.Ry(jindex=0, flip=True) * ET.tz(jindex=2) * ET.Rx(0.4) * ET.Rx(jindex=5)
    C = orc.Chain(e.describe())
    Q = np.random.default_rng(1).uniform(-2, 2, (777, 9))
    np.testing.assert_allclose(host(e.eval(dev(Q))), C.fkine(Q), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(e.jacob0(dev(Q))), C.jacob0(Q), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(e.jacobe(dev(Q))), C.jacobe(Q), rtol=1e-10, atol=1e-12)
    with pytest.raises(ValueError):
        e.eval(dev(Q[:, :5]))  # too narrow for jindex 5
    # IK on a chain whose jindices are not 0..n-1: q0 / q come in chain joint order (q[ets.jindices], IK.py:216-240,346)
    ed = ET.Rz() * ET.tx(0.3) * ET.Ry(flip=True) * ET.tz() * ET.Rx(0.4) * ET.Rx()  # the same chain, densely numbered
    qs = np.random.default_rng(2).uniform(-1, 1, (64, 4))
    Tep = orc.Chain(ed.describe()).fkine(qs)
    q0 = qs + 0.05
    a = [host(x) for x in e.ik_LM(dev(Tep), q0=dev(q0), slimit=1, joint_limits=False, k=0.1)]
    b = [host(x) for x in ed.ik_LM(dev(Tep), q0=dev(q0), slimit=1, joint_limits=False, k=0.1)]
    assert a[1].all()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    Qw = np.zeros((64, 6))
    Qw[:, [4, 0, 2, 5]] = a[0]  # scatter the chain-order solution back into the robot-wide q
    np.testing.assert_allclose(C.fkine(Qw), Tep, atol=5e-3)
    sol = e.ikine_LM(Tep[:8], q0=q0[0], joint_limits=False, seed=3)
    assert sol.success and sol.q.shape == (8, 4)
    dup = ET.Rz(jindex=0) * ET.tx(0.3) * ET.Ry(jindex=0)
    with pytest.raises(ValueError, match="share a jindex"):
        dup.ik_LM(np.eye(4))


def test_api_shapes_and_types():
    panda = rtb.models.Panda()
    e = panda.ets()
    q = np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7])
    assert e.eval(q).shape == (4, 4) and isinstance(e.eval(q), np.ndarray)
    assert e.eval(q[None, :]).shape == (4, 4)  # (1,n) is ONE configuration (fknm.cpp:970-975)
    assert e.eval(q[:, None]).shape == (4, 4)  # (n,1) too (fknm.cpp:976-981)
    assert e.eval(np.tile(q, (5, 1))).shape == (5, 4, 4)
    assert len(e.fkine(np.tile(q, (5, 1)))) == 5
    t = e.eval(torch.from_numpy(q).cuda())
    assert isinstance(t, torch.Tensor) and t.is_cuda and tuple(t.shape) == (4, 4)
    f = e.eval(np.tile(q, (3, 1)).astype(np.float32))
    assert f.dtype == np.float32
    with pytest.raises(TypeError):
        e.eval("abc")
    with pytest.raises(TypeError):
        e.eval(np.array(["a"] * 7, dtype=object))
    with pytest.raises(ValueError):
        e.eval(q, base=np.eye(3))
    # base on the pose but not on the Jacobian (RobotKinematics.py:94 vs :158)
    panda.base = ch.trotz(0.5) @ ch.transl(1, 2, 3)
    T0 = e.eval(q)
    np.testing.assert_allclose(panda.fkine(q).A, panda.base.A @ T0, atol=1e-13)
    np.testing.assert_allclose(panda.jacob0(q), e.jacob0(q), atol=0)
    np.testing.assert_allclose(panda.fkine(q, include_base=False).A, T0, atol=0)
    # DHRobot: base rotation IS in jacob0 (DHRobot.py:1186)
    ur = rtb.models.UR10()
    q6 = q[:6]
    J_nobase = ur.jacob0(q6)
    ur.base = ch.trotx(0.7)
    R = ur.base.A[:3, :3]
    blk = np.zeros((6, 6)); blk[:3, :3] = R; blk[3:, 3:] = R
    np.testing.assert_allclose(ur.jacob0(q6), blk @ J_nobase, atol=1e-13)


def test_host_pipeline_matches_device_path():
    """The pipelined host-buffer front end (chunks over several streams) returns the same bits."""
    e = rtb.models.Panda().ets()
    N = 300_001  # more than two 128k-row chunks, ragged tail
    Q = np.random.default_rng(4).uniform(-np.pi, np.pi, (N, 7))
    Th, Jh = e.fkine_jacob0(Q)
    Td, Jd = e.fkine_jacob0(dev(Q))
    assert np.array_equal(Th, host(Td)) and np.array_equal(Jh, host(Jd))
    qp = rtb.pinned_empty((N, 7)); qp[:] = Q
    Tp = rtb.pinned_empty((N, 4, 4)); Jp = rtb.pinned_empty((N, 6, 7))
    e.fkine_jacob0_into(qp, Tp, Jp)
    assert np.array_equal(Tp, Th) and np.array_equal(Jp, Jh)
    puma = rtb.models.Puma560()
    q, qd, qdd = Q[:, :6], np.cos(Q[:, :6]), np.sin(Q[:, :6])
    assert np.array_equal(puma.rne(q, qd, qdd), host(puma.rne(dev(q), dev(qd), dev(qdd))))


# ------------------------------------------------------------------ properties at full BASELINE sizes
def test_full_size_properties_panda_1M():
    """Config 2 at full size: 1M rows, seed 0, fp64.  Size-independent checks + an oracle subset."""
    e = rtb.models.Panda().ets()
    N = 1_000_000
    Q = np.random.default_rng(0).uniform(-np.pi, np.pi, (N, 7))
    q = dev(Q)
    T, J = e.fkine_jacob0(q)
    # (i) fused == separate kernels, bit for bit
    assert torch.equal(T, e.eval(q)) and torch.equal(J, e.jacob0(q))
    # (ii) rotation blocks orthonormal, bottom row exact
    R = T[:, :3, :3]
    assert (R @ R.transpose(1, 2) - torch.eye(3, dtype=T.dtype, device="cuda")).abs().max().item() < 1e-13
    assert torch.equal(T[:, 3, :], torch.tensor([0.0, 0, 0, 1], dtype=T.dtype, device="cuda").expand(N, 4))
    # (iii) jacobe == blkdiag(R^T, R^T) jacob0 (tests/test_ETS.py:396-398)
    Je = e.jacobe(q)
    Rt = R.transpose(1, 2)
    JeX = torch.cat([Rt @ J[:, :3, :], Rt @ J[:, 3:, :]], dim=1)
    assert (Je - JeX).abs().max().item() < 1e-13
    # (iv) periodicity: q + 2 pi gives the same pose to rounding
    T2 = e.eval(q + 2 * np.pi)
    assert (T2 - T).abs().max().item() < 1e-12
    # (v) a 64k random subset + the first/last rows against the oracle
    idx = np.unique(np.r_[0, N - 1, np.random.default_rng(9).integers(0, N, 65536)])
    C = orc.Chain(e.describe())
    np.testing.assert_allclose(host(T[idx]), C.fkine(Q[idx]), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(host(J[idx]), C.jacob0(Q[idx]), rtol=1e-10, atol=1e-12)
    # (vi) linear rows of J0 vs central differences of the pose (tests/test_jacob.py:27-39)
    h = 1e-6
    sub = q[:4096]
    for j in (0, 3, 6):
        dq = torch.zeros(7, dtype=q.dtype, device="cuda"); dq[j] = h
        dp = (e.eval(sub + dq)[:, :3, 3] - e.eval(sub - dq)[:, :3, 3]) / (2 * h)
        assert (dp - J[:4096, :3, j]).abs().max().item() < 1e-7


def test_full_size_properties_puma_rne_1M():
    """Config 3 at full size: linearity of tau in qdd (tau = M(q) qdd + h(q,qd)) and in gravity."""
    puma = rtb.models.Puma560()
    N = 1_000_000
    rng = np.random.default_rng(1)
    ql = puma.qlim
    q = dev(rng.uniform(ql[0], ql[1], (N, 6)))
    qd = dev(rng.normal(size=(N, 6)))
    a, b = dev(rng.normal(size=(N, 6))), dev(rng.normal(size=(N, 6)))
    qd[-1000:] = 0.0  # Coulomb qd == 0 branch (ne.c:487-490)
    z = torch.zeros_like(a)
    t_ab, t_a, t_b, t_0 = (puma.rne(q, qd, x) for x in (a + b, a, b, z))
    scale = t_ab.abs().max().item()
    assert (t_ab - t_a - t_b + t_0).abs().max().item() < 1e-11 * scale
    # gravity enters linearly: tau(g) - tau(0) doubles when g doubles
    g = np.array([0, 0, -9.81])
    d1 = puma.rne(q, qd, a, gravity=g) - puma.rne(q, qd, a, gravity=[0, 0, 0])
    d2 = puma.rne(q, qd, a, gravity=2 * g) - puma.rne(q, qd, a, gravity=[0, 0, 0])
    assert (d2 - 2 * d1).abs().max().item() < 1e-10 * scale
    idx = np.r_[0, N - 1, np.random.default_rng(3).integers(0, N, 20000)]
    ref = orc.rne(6, 0, puma._pack_rne(), -puma.gravity, host(q[idx]), host(qd[idx]), host(a[idx]))
    np.testing.assert_allclose(host(t_a[idx]), ref, rtol=1e-10, atol=1e-10)


def test_full_size_ur10_fp32():
    """Config 5's per-GPU shard: UR10 DH chain, 1M rows, fp32."""
    e = rtb.models.UR10().ets()
    N = 1 << 20
    Q = np.random.default_rng(3).uniform(-np.pi, np.pi, (N, 6)).astype(np.float32)
    T, J = e.fkine_jacob0(dev(Q, np.float32))
    idx = np.r_[0, N - 1, np.random.default_rng(5).integers(0, N, 30000)]
    C = orc.Chain(e.describe())
    Qr = Q[idx].astype(np.float64)
    np.testing.assert_allclose(host(T[idx]), C.fkine(Qr), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(host(J[idx]), C.jacob0(Qr), rtol=1e-4, atol=1e-5)


def test_launch_counter_moves():
    e = rtb.models.Panda().ets()
    n0 = rtb.launch_count()
    e.eval(dev(np.zeros((10, 7))))
    assert rtb.launch_count() == n0 + 1


def test_jtraj_producer():
    """jtraj on the device (SURVEY 8f-3): the reference's own test properties (tests/test_trajectory.py:420-520)
    and the restated numpy formula, for the `t: int` and time-vector forms, with boundary velocities."""
    q1 = np.r_[1, 2, 3, 4, 5, 6].astype(float)
    q2 = -q1
    tg = rtb.jtraj(q1, q2, 11)
    assert tg.q.shape == tg.qd.shape == tg.qdd.shape == (11, 6) and len(tg) == 11 and tg.naxes == 6
    assert np.allclose(tg.q[0], q1) and np.allclose(tg.q[-1], q2) and np.allclose(tg.q[5], 0)
    assert np.allclose(tg.qd[0], 0) and np.allclose(tg.qd[-1], 0)
    assert np.allclose(tg.qdd[0], 0) and np.allclose(tg.qdd[-1], 0) and np.allclose(tg.qdd[5], 0)
    tv, q, qd, qdd = orc.jtraj(q1, q2, 11)
    np.testing.assert_allclose(tg.t, tv)
    for a, b in ((tg.q, q), (tg.qd, qd), (tg.qdd, qdd)):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12)
    # time vector + boundary velocities, on the device, feeding FK without leaving it
    t = np.linspace(0, 2.5, 5001)
    v0, v1 = 0.1 * q1, -0.2 * q1
    tg = rtb.jtraj(q1, q2, dev(t), qd0=v0, qd1=v1)
    assert tg.q.is_cuda
    tv, q, qd, qdd = orc.jtraj(q1, q2, t, v0, v1)
    for a, b in ((tg.q, q), (tg.qd, qd), (tg.qdd, qdd)):
        np.testing.assert_allclose(host(a), b, rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(host(tg.qd[0]), v0, atol=1e-12)
    np.testing.assert_allclose(host(tg.qd[-1]), v1, atol=1e-10)
    puma = rtb.models.Puma560()
    T = puma.ets().eval(tg.q)
    np.testing.assert_allclose(host(T), orc.Chain(puma.ets().describe()).fkine(q), rtol=1e-9, atol=1e-10)
    tau = puma.rne(tg.q, tg.qd, tg.qdd)  # the whole q, qd, qdd -> torque pipeline stays in HBM
    assert tau.is_cuda and tau.shape == (5001, 6)
    tg32 = rtb.jtraj(q1, q2, 1000, dtype=np.float32, device=True)
    np.testing.assert_allclose(host(tg32.q), orc.jtraj(q1, q2, 1000)[1], rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError):
        rtb.jtraj(q1, q2[:5], 10)
    with pytest.raises(ValueError):
        rtb.jtraj(q1, q2, 10, qd0=[1, 2])


def test_angle_axis_and_p_servo():
    """Batched fknm.Angle_Axis against the compiled-reference fixture (corner cases of ik.cpp:261-277) and p_servo
    (tools/p_servo.py:46-106, angle-axis method): v = gain .* e, arrived = sum|e| < threshold."""
    z = np.load(os.path.join(G, "angle_axis.npz"))
    e = rtb.angle_axis(z["Te"], z["Tep"])
    np.testing.assert_allclose(e, z["e"], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(rtb.angle_axis(z["Te"][5], z["Tep"][5]), z["e"][5], rtol=1e-10, atol=1e-12)
    one = rtb.angle_axis(dev(z["Te"]), dev(z["Tep"][3]))  # a single target for every row
    want = np.stack([orc.angle_axis(a, z["Tep"][3]) for a in z["Te"]])
    np.testing.assert_allclose(host(one), want, rtol=1e-10, atol=1e-12)
    e32 = rtb.angle_axis(z["Te"].astype(np.float32), z["Tep"].astype(np.float32))
    far = np.abs(z["e"]).max(axis=1) < 3.0  # away from the angle = pi discontinuity, where fp32 rounding picks a branch
    np.testing.assert_allclose(e32[far], z["e"][far], rtol=2e-3, atol=2e-3)
    gain = np.array([1, 2, 3, 0.5, 0.25, 4.0])
    v, arrived = rtb.p_servo(z["Te"], z["Tep"], gain=gain, threshold=0.4, method="angle-axis")
    np.testing.assert_allclose(v, z["e"] * gain, rtol=1e-10, atol=1e-12)
    assert (arrived == (np.abs(z["e"]).sum(axis=1) < 0.4)).all()
    v1, a1 = rtb.p_servo(z["Te"][0], z["Tep"][0], gain=2.0, method="angle-axis")
    assert v1.shape == (6,) and a1 is True
    panda = rtb.models.Panda()
    Q = dev(np.random.default_rng(1).uniform(-2, 2, (4096, 7)))
    T = panda.ets().eval(Q)
    v, arr = rtb.p_servo(T, T[7], gain=1.5, method="angle-axis")  # servo every pose of the batch towards one target, all on the device
    assert v.is_cuda and v.shape == (4096, 6) and bool(arr[7]) and float(v[7].abs().max()) == 0.0
    with pytest.raises(ValueError):
        rtb.p_servo(z["Te"][0], z["Tep"][0], method="quaternion")


def test_c_program_through_the_c_abi(tmp_path):
    """examples/cabi_host.c: a plain C program (no Python, no torch, no CUDA headers) linked against libb2kin.so
    builds a 3R chain, calls b2k_fkine_jacob0_host and prints the rows; compare them with the oracle."""
    import subprocess

    root = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
    libdir = os.path.join(root, "robotics-toolbox-python_b200", "lib")
    exe = str(tmp_path / "cabi_host")
    subprocess.run(["gcc", "-O2", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "cabi_host.c"),
                    "-L", libdir, "-lb2kin", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe], check=True)
    r = subprocess.run([exe, "3001"], check=True, capture_output=True, text=True)
    rows = np.array([[float(x) for x in ln.split()] for ln in r.stdout.strip().splitlines()])
    assert rows.shape == (3001, 3 + 16 + 18)
    links = [dict(d=0.4, a=0.0, alpha=np.pi / 2), dict(d=0.0, a=0.35, alpha=0.0), dict(d=0.1, a=0.25, alpha=-np.pi / 2)]
    e = rtb.DHRobot([rtb.RevoluteDH(**lk) for lk in links]).ets()
    C = orc.Chain(e.describe())
    Q = rows[:, :3]
    np.testing.assert_allclose(rows[:, 3:19].reshape(-1, 4, 4), C.fkine(Q), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(rows[:, 19:].reshape(-1, 6, 3), C.jacob0(Q), rtol=1e-10, atol=1e-12)


def test_quintic_trapezoidal_mtraj_producers():
    """quintic / trapezoidal / mtraj on the device (SURVEY 8f-3) against the restated numpy formulas and the
    reference tests' properties (tests/test_trajectory.py:19-153, 209-260): int and time-vector forms,
    boundary velocities, explicit V with its two error cases, multi-axis form."""
    for targ in (11, np.linspace(0, 1, 11), np.linspace(0, 2.5, 1001)):
        for args in ((1, 2), (1, 2, -1, 1), (2, -0.5, 0.3, 0.0)):
            tg = rtb.quintic(args[0], args[1], targ, *args[2:])
            t, s, sd, sdd = orc.quintic(args[0], args[1], targ, *args[2:])
            assert tg.s.shape == s.shape and tg.naxes == 1
            np.testing.assert_allclose(tg.t, t)
            scale = max(1.0, np.abs(sdd).max())
            for a, b in ((tg.s, s), (tg.sd, sd), (tg.sdd, sdd)):
                np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-9 * scale)
        for V in (None, 0.12 if isinstance(targ, int) else 1.2 * 1.0 / float(np.max(targ))):
            tg = rtb.trapezoidal(1, 2, targ, V)
            t, s, sd, sdd, tb = orc.trapezoidal(1, 2, targ, V)
            for a, b in ((tg.s, s), (tg.sd, sd), (tg.sdd, sdd)):
                np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12)
            assert abs(tg.tblend - tb) < 1e-12
    tg = rtb.quintic(1, 2, 11)
    assert np.all(np.diff(tg.s) > 0) and abs(tg.s[5] - 1.5) < 1e-9 and abs(tg.sdd.sum()) < 1e-9
    tg = rtb.trapezoidal(1, 2, 11)
    assert np.all(np.diff(tg.s) > 0) and abs(tg.s[5] - 1.5) < 1e-12 and abs(tg.sd[0]) < 1e-12
    assert rtb.trapezoidal(2, 2, 11).sd.max() == 0.0  # q0 == qf: V = 0, tb = inf
    with pytest.raises(ValueError, match="V too small"):
        rtb.trapezoidal(1, 2, 11, 0.01)
    with pytest.raises(ValueError, match="V too big"):
        rtb.trapezoidal(1, 2, 11, 1.0)
    with pytest.raises(TypeError):
        rtb.quintic(1, 2, 3.5)
    # multi-axis
    q0, qf = np.array([1.0, -2.0, 0.5, 3.0]), np.array([2.0, 1.0, 0.5, -1.0])
    for f, o in ((rtb.quintic, orc.quintic), (rtb.trapezoidal, orc.trapezoidal)):
        tg = rtb.mtraj(f, q0, qf, 50, device=True)
        assert tg.q.is_cuda and tg.q.shape == (50, 4) and tg.name == "mtraj" and not tg.istime
        for j in range(4):
            ref = o(q0[j], qf[j], 50)
            np.testing.assert_allclose(host(tg.q[:, j]), ref[1], rtol=1e-9, atol=1e-9)
            np.testing.assert_allclose(host(tg.qd[:, j]), ref[2], rtol=1e-9, atol=1e-9)
            np.testing.assert_allclose(host(tg.qdd[:, j]), ref[3], rtol=1e-9, atol=1e-9)
    tg32 = rtb.mtraj(rtb.quintic, q0, qf, dev(np.linspace(0, 2, 300), np.float32))
    np.testing.assert_allclose(host(tg32.q[:, 0]), orc.quintic(q0[0], qf[0], np.linspace(0, 2, 300))[1], rtol=1e-4, atol=1e-4)
    with pytest.raises(TypeError):
        rtb.mtraj("quintic", q0, qf, 10)
    with pytest.raises(ValueError):
        rtb.mtraj(rtb.quintic, q0, qf[:3], 10)
