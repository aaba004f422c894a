"""GPU parity of the rows widened in round 2 (SURVEY 8f): singular-value manipulability measures, ..."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import chains as ch  # noqa: E402
from oracle import oracle as orc  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jacfun_ref  # noqa: E402


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def host(t):
    return t.cpu().numpy()


def test_manipulability_minsingular_and_invcondition():
    """ETS.manipulability(method="minsingular" | "invcondition") (ETS.py:1789-1796) against numpy's svd / cond on the
    oracle's Jacobians: Panda (6x7: wide), a 4-joint chain (6x4: tall), axis subsets, a singular configuration."""
    rng = np.random.default_rng(12)
    panda = rtb.models.Panda().ets()
    C = orc.Chain(panda.describe())
    Q = rng.uniform(-2.5, 2.5, (500, 7))
    Q[0] = 0.0  # Panda at zero is singular
    J = C.jacob0(Q)
    for axes, mask in (("all", [True] * 6), ("trans", [True] * 3 + [False] * 3), ("rot", [False] * 3 + [True] * 3),
                       ([True, False, True, False, True, True], [True, False, True, False, True, True])):
        for method in ("minsingular", "invcondition"):
            got = host(panda.manipulability(dev(Q), method=method, axes=axes))
            np.testing.assert_allclose(got, orc.manip_svd(J, mask, method), rtol=1e-9, atol=1e-12, err_msg=f"{axes} {method}")
    assert panda.manipulability(Q[0], method="minsingular") < 1e-10
    # from a given J, numpy in -> numpy out, one configuration -> float
    m = panda.manipulability(J=J[5], method="invcondition")
    assert isinstance(m, float) and abs(m - orc.manip_svd(J[5], kind="invcondition")[0]) < 1e-12
    ET = rtb.ET
    e4 = ET.Rz() * ET.tx(0.3) * ET.Ry() * ET.tz(0.2) * ET.Rx() * ET.tx(0.1) * ET.Rz()
    C4 = orc.Chain(e4.describe())
    Q4 = rng.uniform(-2, 2, (300, 4))
    for method in ("minsingular", "invcondition"):
        np.testing.assert_allclose(host(e4.manipulability(dev(Q4), method=method)), orc.manip_svd(C4.jacob0(Q4), kind=method),
                                   rtol=1e-9, atol=1e-12)
    got32 = host(panda.manipulability(dev(Q[1:], np.float32), method="minsingular"))
    np.testing.assert_allclose(got32, orc.manip_svd(J[1:], kind="minsingular"), rtol=2e-3, atol=2e-5)
    with pytest.raises(ValueError):
        panda.manipulability(Q[1], method="asada")


def test_jacob0_analytical_all_representations():
    """ETS.jacob0_analytical (ETS.py:1570-1626) for rpy/xyz, rpy/zyx, eul, exp against the oracle's restatement of
    rotvelxform, and -- independently of any restatement -- against the finite-difference derivative of the
    representation of the pose the product itself computes."""
    rng = np.random.default_rng(21)
    panda = rtb.models.Panda()
    e = panda.ets()
    C = orc.Chain(e.describe())
    Q = rng.uniform(-2, 2, (400, 7))
    T, J = C.fkine(Q), C.jacob0(Q)
    for rep in ("rpy/xyz", "rpy/zyx", "eul", "exp"):
        Ja = host(e.jacob0_analytical(dev(Q), representation=rep))
        want = orc.jacob0_analytical(T, J, rep)
        ok = np.abs(want).max(axis=(1, 2)) < 1e4  # rows next to the representation's singularity: 1/cos(pitch) etc. blow up
        np.testing.assert_allclose(Ja[ok], want[ok], rtol=1e-8, atol=1e-9, err_msg=rep)
        one = e.jacob0_analytical(Q[3], representation=rep)
        assert isinstance(one, np.ndarray) and one.shape == (6, 7)
        np.testing.assert_allclose(one, want[3], rtol=1e-8, atol=1e-9)
    # finite differences through the product's own FK
    h = 1e-6
    Ja = host(e.jacob0_analytical(dev(Q[:50]), representation="rpy/zyx"))
    for j in (0, 3, 6):
        dq = np.zeros(7); dq[j] = h
        gp = np.stack([orc.tr2rpy(t, "zyx") for t in host(e.eval(dev(Q[:50] + dq)))])
        gm = np.stack([orc.tr2rpy(t, "zyx") for t in host(e.eval(dev(Q[:50] - dq)))])
        d = (gp - gm + np.pi) % (2 * np.pi) - np.pi
        good = np.abs(d).max(axis=1) < 1e-3
        np.testing.assert_allclose(Ja[:50][good][:, 3:, j], d[good] / (2 * h), rtol=1e-4, atol=1e-5)
    with pytest.raises(ValueError):
        e.jacob0_analytical(Q[0], representation="quaternion")
    # analytical jacob0_dot: the reference differentiates jacob0_analytical numerically (Robot.py:1090-1092)
    qd = rng.normal(size=(50, 7))
    Jd = host(e.jacob0_dot(dev(Q[:50]), dev(qd), representation="rpy/xyz"))
    hh = 1e-5
    num = (orc.jacob0_analytical(C.fkine(Q[:50] + hh * qd), C.jacob0(Q[:50] + hh * qd), "rpy/xyz")
           - orc.jacob0_analytical(C.fkine(Q[:50] - hh * qd), C.jacob0(Q[:50] - hh * qd), "rpy/xyz")) / (2 * hh)
    ok = np.abs(num).max(axis=(1, 2)) < 1e3
    np.testing.assert_allclose(Jd[ok], num[ok], rtol=1e-4, atol=1e-4)


def test_p_servo_rpy_method():
    """tools/p_servo.py:80-106 with the reference's default method='rpy' (error in the end-effector frame)."""
    rng = np.random.default_rng(22)
    C = orc.Chain(ch.panda_ets())
    Te, Tep = C.fkine(rng.uniform(-2, 2, (300, 7))), C.fkine(rng.uniform(-2, 2, (300, 7)))
    gain = np.array([1, 2, 3, 0.5, 0.25, 4.0])
    v, arrived = rtb.p_servo(Te, Tep, gain=gain, threshold=2.5)  # default method is rpy, as in the reference
    wv, wa = orc.p_servo_rpy(Te, Tep, gain, 2.5)
    np.testing.assert_allclose(v, wv, rtol=1e-10, atol=1e-11)
    assert (arrived == wa).all() and 0 < arrived.sum() < 300
    v1, a1 = rtb.p_servo(Te[0], Te[0], gain=2.0)
    assert v1.shape == (6,) and a1 is True and np.abs(v1).max() < 1e-12
    vd, ad = rtb.p_servo(dev(Te), dev(Tep[5]), gain=1.5, method="rpy")
    wv, wa = orc.p_servo_rpy(Te, Tep[5], 1.5, 0.1)
    np.testing.assert_allclose(host(vd), wv, rtol=1e-10, atol=1e-11)
    v32, _ = rtb.p_servo(Te.astype(np.float32), Tep.astype(np.float32), gain=1.0)
    far = np.abs(np.abs(orc.p_servo_rpy(Te, Tep, 1.0, 0.1)[0][:, 3:]) - np.pi).min(axis=1) > 0.05  # away from the +-pi wrap
    np.testing.assert_allclose(v32[far], orc.p_servo_rpy(Te, Tep, 1.0, 0.1)[0][far], rtol=2e-3, atol=2e-3)


def test_ctraj_feeds_ik_on_the_device():
    """tools.trajectory.ctraj (trajectory.py:782-841): the pose batch is produced in HBM and consumed there by ik_LM."""
    rng = np.random.default_rng(23)
    panda = rtb.models.Panda().ets()
    C = orc.Chain(panda.describe())
    qa = rng.uniform(-1.5, 1.5, 7)
    qb = qa + rng.uniform(-0.4, 0.4, 7)  # a short move: the straight Cartesian line stays inside the workspace
    T0, T1 = C.fkine(qa)[0], C.fkine(qb)[0]
    s = np.r_[rng.uniform(0, 1, 300), 0.0, 1.0, -0.2, 1.3]
    P = rtb.ctraj(T0, T1, s=s)
    np.testing.assert_allclose(P.A, orc.ctraj_poses(T0, T1, s), rtol=1e-10, atol=1e-12)
    for n in (2, 25, 100):  # ctraj(T0, T1, n): trapezoidal path fraction
        Pn = rtb.ctraj(T0, T1, n)
        sn = orc.trapezoidal(0, 1, n)[1]
        np.testing.assert_allclose(Pn.A, orc.ctraj_poses(T0, T1, sn), rtol=1e-9, atol=1e-11)
    t = np.linspace(0, 4, 33)
    np.testing.assert_allclose(rtb.ctraj(T0, T1, t).A, orc.ctraj_poses(T0, T1, orc.trapezoidal(0, 1, t / t.max())[1]), rtol=1e-9, atol=1e-11)
    # opposite-hemisphere quaternions take the shorter arc; identical orientations interpolate the translation only
    T2 = T0.copy(); T2[:3, 3] += [0.1, -0.2, 0.3]
    np.testing.assert_allclose(rtb.ctraj(T0, T2, s=[0.25, 0.5]).A[0, :3, :3], T0[:3, :3], atol=1e-12)
    Td = rtb.ctraj(T0, T1, 200, device=True)
    assert Td.is_cuda and Td.shape == (200, 4, 4)
    q, ok, it, sr, E = panda.ik_LM(Td, q0=dev(qa), joint_limits=False, k=0.1)
    okh = host(ok).astype(bool)
    assert okh.all()
    np.testing.assert_allclose(C.fkine(host(q))[okh], host(Td)[okh], atol=5e-3)
    with pytest.raises(TypeError):
        rtb.ctraj(T0, T1)


def test_mstraj_sample_table():
    """tools.trajectory.mstraj (trajectory.py:852-1152): plan on the host, samples on the device; against the numpy
    restatement of the reference loop, both timing modes, initial / final velocities, scalar and per-segment tacc."""
    via = np.array([[0.0, 0.0, 0.2], [1.0, 0.5, -0.4], [1.0, 2.0, 0.0], [-0.5, 2.0, 0.9], [0.3, -1.0, 0.9]])
    cases = [dict(dt=0.1, tacc=0.4, qdmax=[1.0, 0.8, 0.5]), dict(dt=0.05, tacc=0.2, qdmax=1.5),
             dict(dt=0.1, tacc=0.0, qdmax=[1.0, 0.8, 0.5]), dict(dt=0.2, tacc=0.5, tsegment=[2.0, 3.0, 2.5, 4.0]),
             dict(dt=0.1, tacc=[0.2, 0.4, 0.6, 0.3], qdmax=2.0, qd0=[0.1, 0.0, -0.1], qdf=[0.0, 0.2, 0.0]),
             dict(dt=0.1, tacc=0.3, qdmax=1.0, q0=[0.5, 0.5, 0.5])]
    for kw in cases:
        tr = rtb.mstraj(via, **kw)
        t, q, arrive = orc.mstraj(via, **kw)
        assert tr.q.shape == q.shape, (kw, tr.q.shape, q.shape)
        np.testing.assert_allclose(tr.q, q, rtol=1e-10, atol=1e-12, err_msg=str(kw))
        np.testing.assert_allclose(tr.t, t, atol=1e-12)
        np.testing.assert_allclose(tr.arrive, arrive, atol=1e-12)
        assert len(tr.info) == (len(via) if "q0" in kw else len(via) - 1) + 1
    trd = rtb.mstraj(via, dt=0.1, tacc=0.4, qdmax=[1.0, 0.8, 0.5], device=True)
    assert trd.q.is_cuda
    tr32 = rtb.mstraj(via, dt=0.1, tacc=0.4, qdmax=[1.0, 0.8, 0.5], dtype=np.float32)
    np.testing.assert_allclose(tr32.q, orc.mstraj(via, dt=0.1, tacc=0.4, qdmax=[1.0, 0.8, 0.5])[1], rtol=1e-5, atol=1e-6)
    with pytest.raises(ValueError):
        rtb.mstraj(via, dt=0.1, tacc=0.2, qdmax=1.0, tsegment=[1, 1, 1, 1])
    with pytest.raises(ValueError):
        rtb.mstraj(via, dt=0.1, tacc=0.2)


def test_fdyn_device_integrator_follows_scipy_rk45():
    """DynamicsMixin.fdyn (Dynamics.py:185-422): the device-resident Dormand-Prince integrator against the reference's
    procedure restated with scipy.integrate.RK45 and the oracle's accel -- same accepted steps, same states."""
    full = rtb.models.Puma560()
    puma = full.nofriction()  # Coulomb friction off, as the reference's fdyn example does (the integrators chatter at qd = 0)
    assert (puma._pack_rne().reshape(6, 24)[:, 22:] == 0).all() and (full._pack_rne().reshape(6, 24)[:, 22:] != 0).any()
    assert puma._pack_rne().reshape(6, 24)[0, 21] == full._pack_rne().reshape(6, 24)[0, 21] != 0  # viscous friction kept
    n = 6
    L, g = puma._pack_rne(), puma.gravity
    rne = lambda q, qd, qdd, grav: orc.rne(n, 0, L, -np.asarray(grav, dtype=float), q, qd, qdd)  # noqa: E731
    acc = lambda q, qd, tau: orc.dyn_accel(rne, n, q, qd, tau, g)[0]  # noqa: E731
    q0 = puma.qn
    # zero torque, the reference's default call: the arm falls under gravity
    tg = puma.fdyn(0.4, q0)
    t, q, qd = orc.fdyn(acc, n, 0.4, q0)
    assert tg.t.shape == t.shape, (tg.t.shape, t.shape)
    np.testing.assert_allclose(tg.t, t, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(tg.q, q, rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(tg.qd, qd, rtol=1e-6, atol=1e-8)
    # uniform output grid (interp1d), tighter tolerances, an initial velocity
    sa = dict(rtol=1e-6, atol=1e-9)
    qd0 = np.array([0.1, -0.2, 0.3, 0.0, 0.1, 0.0])
    tg = puma.fdyn(0.3, q0, qd0=qd0, solver_args=sa, dt=0.01)
    t, q, qd = orc.fdyn(acc, n, 0.3, q0, qd0=qd0, solver_args=sa, dt=0.01)
    np.testing.assert_allclose(tg.t, t, atol=1e-14)
    np.testing.assert_allclose(tg.q, q, rtol=1e-7, atol=1e-9)
    np.testing.assert_allclose(tg.qd, qd, rtol=1e-6, atol=1e-8)
    # constant torque and the PD law
    tau = np.array([5.0, -20.0, 3.0, 0.5, 0.2, 0.1])
    tg = puma.fdyn(0.2, q0, Q=tau, solver_args=sa)
    t, q, qd = orc.fdyn(acc, n, 0.2, q0, torque_fn=lambda t, q, qd: tau, solver_args=sa)
    assert tg.t.shape == t.shape
    np.testing.assert_allclose(tg.q, q, rtol=1e-7, atol=1e-9)
    kp, kd = np.array([80, 120, 60, 10, 10, 5.0]), np.array([8, 10, 6, 1, 1, 0.5])
    tg = puma.fdyn(0.3, q0, Q=("pd", kp, kd, puma.qz), solver_args=sa, dt=0.02)
    t, q, qd = orc.fdyn(acc, n, 0.3, q0, torque_fn=lambda t, q, qd: kp * (puma.qz - q) - kd * qd, solver_args=sa, dt=0.02)
    np.testing.assert_allclose(tg.q, q, rtol=1e-7, atol=1e-9)
    # the reference's callable route (scipy on the host, this robot's accel kernel as the right-hand side)
    tgc = puma.fdyn(0.2, q0, Q=lambda robot, t, q, qd: tau, solver_args=sa)
    t, q, qd = orc.fdyn(acc, n, 0.2, q0, torque_fn=lambda t, q, qd: tau, solver_args=sa)
    assert tgc.t.shape == t.shape
    np.testing.assert_allclose(tgc.q, q, rtol=1e-7, atol=1e-9)
    # an ensemble: every lane integrates its own initial state with its own step sizes
    rng = np.random.default_rng(5)
    Q0 = q0 + rng.uniform(-0.3, 0.3, (200, 6))
    ens = puma.fdyn(0.2, dev(Q0), solver_args=sa, dt=0.02)
    assert ens.q.is_cuda and ens.q.shape == (200, 10, 6)
    for i in (0, 57, 199):
        t, q, qd = orc.fdyn(acc, n, 0.2, Q0[i], solver_args=sa, dt=0.02)
        np.testing.assert_allclose(ens.q[i].cpu().numpy(), q, rtol=1e-7, atol=1e-9)
    steps = puma.fdyn(0.2, Q0[:8], solver_args=sa)
    assert steps.t.shape == (8, 4096) and (steps.count > 3).all() and np.isnan(steps.t[0, steps.count[0]:]).all()
    for i in (0, 7):
        t, q, qd = orc.fdyn(acc, n, 0.2, Q0[i], solver_args=sa)
        assert steps.count[i] == len(t)
        np.testing.assert_allclose(steps.q[i, :len(t)], q, rtol=1e-7, atol=1e-9)
    with pytest.raises(RuntimeError, match="max_steps"):
        puma.fdyn(0.5, q0, solver_args=dict(rtol=1e-10, atol=1e-12), max_steps=8)
    with pytest.raises(ValueError):
        puma.fdyn(0.1, q0, solver="Radau")


def test_fkine_all_reference_literals_and_dh_link_products():
    """DHRobot.fkine_all (DHRobot.py:1018-1064): the literal frames of the reference's own test (tests/test_DHRobot.py:
    638-710, DH Panda at q = 1..7, 4 decimals) and, for batches, the running product base * A1 ... Ak of the DH link
    transforms restated independently in oracle/chains.py."""
    panda = rtb.models.DH.Panda()
    q = np.arange(1.0, 8.0)
    T = panda.fkine_all(q)
    assert T.shape == (8, 4, 4)
    lit = {
        0: np.eye(4),
        1: [[0.5403, -0.8415, 0, 0], [0.8415, 0.5403, 0, 0], [0, 0, 1, 0.333], [0, 0, 0, 1]],
        2: [[-0.2248, -0.4913, -0.8415, 0], [-0.3502, -0.7651, 0.5403, 0], [-0.9093, 0.4161, 0, 0.333], [0, 0, 0, 1]],
        3: [[0.1038, 0.8648, 0.4913, 0.1552], [0.4229, -0.4855, 0.7651, 0.2418], [0.9002, 0.1283, -0.4161, 0.2015], [0, 0, 0, 1]],
        4: [[-0.4397, -0.2425, -0.8648, 0.1638], [-0.8555, -0.1801, 0.4855, 0.2767], [-0.2735, 0.9533, -0.1283, 0.2758], [0, 0, 0, 1]],
        5: [[-0.9540, -0.1763, -0.2425, 0.107], [0.2229, -0.9581, -0.1801, 0.2781], [-0.2006, -0.2258, 0.9533, 0.6644], [0, 0, 0, 1]],
        6: [[-0.8482, -0.4994, 0.1763, 0.107], [0.2643, -0.1106, 0.9581, 0.2781], [-0.4590, 0.8593, 0.2258, 0.6644], [0, 0, 0, 1]],
        7: [[-0.5236, 0.6902, 0.4994, 0.08575], [0.8287, 0.5487, 0.1106, 0.3132], [-0.1977, 0.4718, -0.8593, 0.5321], [0, 0, 0, 1]],
    }
    for k, want in lit.items():
        np.testing.assert_array_almost_equal(T[k], np.asarray(want, dtype=float), decimal=4)
    rng = np.random.default_rng(12)
    for robot, links, mdh in ((panda, ch.panda_mdh_links(), True), (rtb.models.Puma560(), ch.puma560_links(), False)):
        n = robot.n
        Q = rng.uniform(-np.pi, np.pi, (257, n))
        base = ch.transl(0.1, -0.2, 0.3) @ ch.trotz(0.4)
        robot.base = base
        got = robot.fkine_all(dev(Q))
        assert got.is_cuda and tuple(got.shape) == (257, n + 1, 4, 4)
        got = got.cpu().numpy()
        for i in (0, 100, 256):
            Tk = base.copy()
            np.testing.assert_allclose(got[i, 0], Tk, atol=1e-14)
            for k in range(n):
                Tk = Tk @ ch.dh_A(links[k], Q[i, k], mdh=mdh)
                np.testing.assert_allclose(got[i, k + 1], Tk, rtol=1e-10, atol=1e-12)
        # the last frame is fkine without the tool
        np.testing.assert_allclose(got[:, n], robot.eval(dev(Q)).cpu().numpy() @ np.linalg.inv(robot.tool.A), rtol=1e-10, atol=1e-12)
        host = robot.fkine_all(Q[:5].astype(np.float32))
        assert isinstance(host, np.ndarray) and host.dtype == np.float32 and host.shape == (5, n + 1, 4, 4)
        np.testing.assert_allclose(host, got[:5], rtol=1e-4, atol=1e-5)
        robot.base = None


def test_fkine_all_of_a_branched_urdf_robot():
    """Robot.fkine_all (Robot.py:638-700): frame i = pose of link number i, every branch, static links included; each
    frame against the product of link.A(q) from the base link down (the reference's recursion)."""
    import os

    rob = rtb.Robot.URDF(os.path.join(os.path.dirname(__file__), "golden", "urdf", "two_arm.urdf"))
    rng = np.random.default_rng(13)
    Q = rng.uniform(-1.5, 1.5, (65, rob.n))
    got = rob.fkine_all(dev(Q)).cpu().numpy()
    assert got.shape == (65, len(rob.links) + 1, 4, 4)
    for i in (0, 64):
        np.testing.assert_allclose(got[i, 0], np.eye(4), atol=1e-15)
        for k, link in enumerate(rob.links):
            T, l, chain = np.eye(4), link, []
            while l is not None:
                chain.append(l)
                l = l.parent
            for l in reversed(chain):
                T = T @ l.A(Q[i, l.jindex] if l.isjoint else 0.0)
            np.testing.assert_allclose(got[i, k + 1], T, rtol=1e-10, atol=1e-12, err_msg=link.name)
    one = rob.fkine_all(Q[0])
    assert one.shape == (len(rob.links) + 1, 4, 4)
    np.testing.assert_allclose(one, got[0], rtol=1e-12, atol=1e-13)


def test_hessian_every_joint_count_grid_stride_and_alignment():
    """k_hessian (b2k_extra.cu): every instantiated joint count, both dtypes, more rows than one wave of warps (each warp
    walks several rows with its per-thread index table), a ragged last block, and an output pointer that is only
    element-aligned (scalar-store path) -- against the vectorised restatement, itself checked against oracle.hessian."""
    from importlib import import_module
    B = import_module("b2kin")._buffers
    lib = rtb._lib.lib()
    rng = np.random.default_rng(77)
    Jc = rng.normal(size=(3, 6, 5))
    for k in range(3):
        np.testing.assert_allclose(jacfun_ref.hessian_batch(Jc)[k], orc.hessian(Jc[k]), rtol=0, atol=1e-15)
    for n in range(1, 11):
        N = 9001 if n not in (6, 7) else 150_003
        J = rng.normal(size=(N, 6, n))
        ref = jacfun_ref.hessian_batch(J)
        for dt, tol in ((np.float64, dict(rtol=0, atol=1e-14)), (np.float32, dict(rtol=0, atol=2e-6))):
            Jd = dev(J, dt)
            H = torch.full((N * 6 * n * n + 1,), float("nan"), dtype=Jd.dtype, device="cuda")
            for off in (0, 1):  # off = 1: rows start one element past a 16-byte boundary
                out = H[off:off + N * 6 * n * n]
                out.fill_(float("nan"))
                rtb._lib.check(lib.b2k_hessian(B.code(np.dtype(dt)), n, B.ptr(Jd), N, B.ptr(out), B.stream_ptr(Jd)))
                np.testing.assert_allclose(host(out).reshape(N, n, 6, n), ref.astype(dt) if dt == np.float32 else ref, **tol,
                                           err_msg=f"n={n} {dt.__name__} offset={off}")


def test_pose_kernels_on_element_aligned_arrays():
    """The pose consumers / producers take 16-byte vector loads and stores when the arrays allow it; a C-ABI caller may
    hand over arrays that are only element-aligned.  Both code paths against the same restatements: p_servo("rpy"),
    p_servo("angle-axis") on pose batches that start one element past a 16-byte boundary, ctraj into such an array."""
    B = rtb._buffers
    lib = rtb._lib.lib()
    rng = np.random.default_rng(91)
    Ch = orc.Chain(ch.panda_ets())
    N = 3001
    Te, Tep = Ch.fkine(rng.uniform(-2, 2, (N, 7))), Ch.fkine(rng.uniform(-2, 2, (N, 7)))
    gain = np.array([1, 2, 3, 0.5, 0.25, 4.0])
    T0, T1 = Te[0], Tep[0]
    A0, A1 = np.ascontiguousarray(T0), np.ascontiguousarray(T1)
    s = rng.uniform(-0.1, 1.1, N)
    for dt, tol in ((np.float64, dict(rtol=1e-9, atol=1e-11)), (np.float32, dict(rtol=2e-3, atol=2e-3))):
        code = B.code(np.dtype(dt))
        bufE = torch.zeros(N * 16 + 1, dtype=B.tdtype(np.dtype(dt)), device="cuda")
        bufP = torch.zeros(N * 16 + 1, dtype=bufE.dtype, device="cuda")
        res = {}
        for off in (0, 1):
            e_, p_ = bufE[off:off + N * 16], bufP[off:off + N * 16]
            e_.copy_(dev(Te, dt).reshape(-1)); p_.copy_(dev(Tep, dt).reshape(-1))
            for name, fn in (("rpy", lib.b2k_p_servo_rpy), ("aa", lib.b2k_p_servo)):
                v = torch.empty(N * 6, dtype=bufE.dtype, device="cuda")
                arrived = torch.empty(N, dtype=torch.int32, device="cuda")
                rtb._lib.check(fn(code, B.ptr(e_), B.ptr(p_), N, 16, rtb._lib.dptr(gain), 2.5, B.ptr(v),
                                  B.ptr(arrived), B.stream_ptr(v)))
                res[name, off] = (host(v).reshape(N, 6), host(arrived))
            out = torch.full((N * 16 + 1,), float("nan"), dtype=bufE.dtype, device="cuda")
            sd = dev(s, dt)
            rtb._lib.check(lib.b2k_ctraj(code, rtb._lib.dptr(A0), rtb._lib.dptr(A1), B.ptr(sd), N,
                                         B.ptr(out[off:]), B.stream_ptr(sd)))
            res["ctraj", off] = host(out[off:off + N * 16]).reshape(N, 4, 4)
        for name in ("rpy", "aa"):  # the two load paths do the same arithmetic
            np.testing.assert_array_equal(res[name, 0][0], res[name, 1][0])
            np.testing.assert_array_equal(res[name, 0][1], res[name, 1][1])
        np.testing.assert_array_equal(res["ctraj", 0], res["ctraj", 1])
        wv, wa = orc.p_servo_rpy(Te, Tep, gain, 2.5)
        far = np.abs(np.abs(wv[:, 3:] / gain[3:]) - np.pi).min(axis=1) > 0.05  # away from the +-pi wrap (fp32)
        np.testing.assert_allclose(res["rpy", 1][0][far], wv[far], **tol)
        if dt == np.float64:
            np.testing.assert_array_equal(res["rpy", 1][1], wa)
            np.testing.assert_allclose(res["ctraj", 1], orc.ctraj_poses(T0, T1, s), rtol=1e-10, atol=1e-12)
        else:
            np.testing.assert_allclose(res["ctraj", 1], orc.ctraj_poses(T0, T1, s), rtol=1e-4, atol=1e-5)
