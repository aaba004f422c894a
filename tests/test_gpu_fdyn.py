"""GPU sweep of the device forward-dynamics integrator (k_fdyn in csrc/b2k_rne_spec.cu behind DHRobot.fdyn and
Robot.fdyn) against scipy's RK45 on the oracle's accel (tests/fdyn_ref.py): every joint count, DH and MDH, prismatic
joints, motor inertia, gear ratio, viscous and Coulomb friction, rigid-body trees up to 16 joints, every gravity pattern
(each one a different generated program), the four torque laws, the step-control options, both output modes, ensembles
that straddle a block of 64 lanes, fp32, and the C ABI's argument checks.

In fp64 the device takes scipy's accepted steps: the same count, t to 1e-9, q and qd to rounding accumulated over the
steps.  fp32 takes its own steps, so it is held to the error scipy itself makes at the same tolerances."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import oracle as orc  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fdyn_ref as R  # noqa: E402

ET, ETS, Link, Robot = rtb.ET, rtb.ETS, rtb.Link, rtb.Robot
URDF_DIR = os.path.join(os.path.dirname(__file__), "golden", "urdf")
TQ, TQD = dict(rtol=1e-7, atol=1e-9), dict(rtol=1e-6, atol=1e-8)  # fp64 q / qd against scipy on the oracle
TREE_TQ, TREE_TQD = dict(rtol=1e-6, atol=1e-8), dict(rtol=1e-5, atol=1e-7)  # trees: the oracle is a numpy recursion
TIGHT = dict(rtol=1e-10, atol=1e-12)
# The error estimate is a difference of O(h f) terms, so the rounding by which the device's accel differs from the
# oracle's reaches the step-size factor amplified by about |f| h / tolerance: step sequences are compared at these
# tolerances (as in test_gpu_widened_r2's Puma case), with t to 1e-7 (fast, stiff cases drift by a few 1e-8; a wrong
# error coefficient or step rule moves the steps by 1e-4 or more); tighter cases are compared on a grid.
STEPS = dict(rtol=1e-6, atol=1e-9)


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


# ------------------------------------------------------------------ robots from a seed
def dh_arm(rng, n, mdh, prismatic=(), coulomb=False):
    """A random DH / MDH arm with motor inertia, gear ratio and viscous friction on every joint; translational joints
    at the indices in `prismatic`; Coulomb friction when asked."""
    links = []
    for j in range(n):
        kw = dict(a=float(rng.choice([0.0, rng.uniform(-0.4, 0.4)])), alpha=float(rng.choice([0.0, np.pi / 2, -np.pi / 2, rng.uniform(-1, 1)])),
                  m=float(rng.uniform(0.5, 4)), r=rng.uniform(-0.2, 0.2, 3).tolist(),
                  I=rng.uniform(0.02, 0.3, 3).tolist() + rng.uniform(-0.005, 0.005, 3).tolist(), Jm=float(rng.uniform(1e-4, 3e-4)),
                  G=float(rng.choice([-1, 1]) * rng.uniform(20, 100)), B=float(rng.uniform(1e-3, 3e-3)),
                  Tc=[float(rng.uniform(0.1, 0.4)), float(-rng.uniform(0.1, 0.4))] if coulomb else [0.0, 0.0])
        if j in prismatic:
            mk = rtb.PrismaticMDH if mdh else rtb.PrismaticDH
            links.append(mk(theta=float(rng.uniform(-1, 1)), offset=float(rng.uniform(-0.2, 0.2)), **kw))
        else:
            mk = rtb.RevoluteMDH if mdh else rtb.RevoluteDH
            links.append(mk(d=float(rng.choice([0.0, rng.uniform(-0.4, 0.4)])), offset=float(rng.choice([0.0, rng.uniform(-1, 1)])), **kw))
    return rtb.DHRobot(links)


def tree_robot(rng, n):
    """A random branched tree with translational and flipped joints and massless static links; every centre of mass
    off every axis, so the inertia matrix (mass and centre of mass only, Robot.rne) is regular."""
    links = []
    for j in range(n):
        parent = None if j == 0 else links[int(rng.integers(0, len(links)))]
        consts = ETS()
        for _ in range(int(rng.integers(0, 3))):
            kind = int(rng.integers(0, 6))
            val = float(rng.choice([np.pi / 2, -np.pi / 2, rng.uniform(-1, 1)])) if kind < 3 else float(rng.uniform(-0.4, 0.4))
            consts = consts * getattr(ET, ("Rx", "Ry", "Rz", "tx", "ty", "tz")[kind])(val)
        joint = getattr(ET, ("Rx", "Ry", "Rz", "tx", "ty", "tz")[int(rng.integers(0, 6))])(flip=bool(rng.integers(0, 2)))
        links.append(Link(consts * joint, name=f"j{j}", parent=parent, m=float(rng.uniform(0.5, 3)),
                          r=(rng.uniform(0.1, 0.3, 3) * rng.choice([-1, 1], 3)).tolist()))
        if rng.random() < 0.3:
            links.append(Link(ETS(ET.tx(float(rng.uniform(-0.2, 0.2)))), name=f"s{j}", parent=links[-1]))
    return Robot(links)


def regular(make, rne_of, n, T, q0_of, seed, **kw):
    """The first robot from `seed` on whose zero-torque reference trajectory cond(M) < 1e6."""
    rng = np.random.default_rng(seed)
    for _ in range(20):
        rob = make(rng)
        q0 = q0_of(rng)
        acc = R.tree_accel(rob) if isinstance(rob, Robot) else R.dh_accel(rob)
        ref = R.fdyn(acc, n, T, q0, **kw)
        if R.max_cond(rne_of(rob), n, ref.q) < 1e6:
            return rob, q0, ref
    raise AssertionError("no well-conditioned robot")


def check_steps(got, ref, label, tq=TQ, tqd=TQD):
    assert isinstance(got.t, np.ndarray) and got.t.shape == ref.t.shape, (label, got.t.shape, ref.t.shape)
    np.testing.assert_allclose(got.t, ref.t, rtol=1e-7, atol=1e-12, err_msg=label)
    np.testing.assert_allclose(got.q, ref.q, **tq, err_msg=label)
    np.testing.assert_allclose(got.qd, ref.qd, **tqd, err_msg=label)


def check_grid(got, ref, label, tq=TQ, tqd=TQD):
    assert np.shape(got.t) == ref.t.shape, (label, np.shape(got.t), ref.t.shape)
    np.testing.assert_allclose(got.t, ref.t, rtol=0, atol=1e-14, err_msg=label)
    np.testing.assert_allclose(got.q, ref.q, **tq, err_msg=label)
    np.testing.assert_allclose(got.qd, ref.qd, **tqd, err_msg=label)


def pd(kp, kd, qs):
    return lambda t, q, qd: kp * (qs - q) - kd * qd  # noqa: E731


# ------------------------------------------------------------------ DH / MDH arms at every joint count
GRAVITY = ("argument", "attribute", "zero", "base")  # rotated per joint count


@pytest.mark.parametrize("n", range(1, 11))
def test_dh_arms_every_joint_count(n):
    """Random arms, DH at odd n and MDH at even n: zero torque on the solver's steps at default tolerances; then a
    gravity variant (a general vector as argument, a partly zero one as attribute, zero, or a rotated base) with a
    torque law and an initial velocity on a grid that does not divide T, at tight tolerances where n is small."""
    mdh = n % 2 == 0
    rob, q0, ref = regular(lambda rng: dh_arm(rng, n, mdh), R.dh_rne, n, 0.25, lambda rng: rng.uniform(-1.5, 1.5, n), 500 + n)
    check_steps(rob.fdyn(0.25, q0), ref, f"n={n} default")
    rng = np.random.default_rng(n)
    qd0 = rng.uniform(-1, 1, n)
    which = GRAVITY[n % 4]
    kw = {}
    if which == "argument":
        g = np.array([0.5, -1.0, 3.0])
        kw = dict(gravity=g)
        acc = R.dh_accel(rob, g)
    elif which == "attribute":
        rob.gravity = [0.0, 4.0, -9.81]
        acc = R.dh_accel(rob)
    elif which == "zero":
        kw = dict(gravity=[0, 0, 0])
        acc = R.dh_accel(rob, [0, 0, 0])
    else:
        c, s = np.cos(0.6), np.sin(0.6)
        base = np.eye(4)
        base[:3, :3] = np.array([[1, 0, 0], [0, c, -s], [0, s, c]]) @ np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        base[:3, 3] = [0.1, 0.2, 0.3]
        rob.base = base
        assert np.count_nonzero(R.dh_gravity(rob)) == 3
        acc = R.dh_accel(rob)
    tau = rng.normal(size=n)
    Q = [tau, ("pd", 30.0, 3.0, np.zeros(n)), ("pd", rng.uniform(10, 60, n), rng.uniform(1, 5, n), rng.uniform(-1, 1, n))][n % 3]
    law = (lambda t, q, qd: tau) if n % 3 == 0 else pd(*Q[1:])
    sa = TIGHT if n <= 4 else dict(rtol=1e-8, atol=1e-10)
    T, dt = 0.2, 0.03
    ref = R.fdyn(acc, n, T, q0, qd0=qd0, torque=law, solver_args=sa, dt=dt)
    check_grid(rob.fdyn(T, q0, qd0=qd0, Q=Q, solver_args=sa, dt=dt, **kw), ref, f"n={n} {which} {Q}")
    # the same case on the solver's steps
    ref = R.fdyn(acc, n, T, q0, qd0=qd0, torque=law, solver_args=STEPS)
    check_steps(rob.fdyn(T, q0, qd0=qd0, Q=Q, solver_args=STEPS, **kw), ref, f"n={n} {which} steps")


def test_prismatic_mixes():
    """Translational joints: a DH arm whose FIRST joint is prismatic and an MDH arm with a prismatic joint inside
    the chain; the MDH prismatic-first arm is refused (its M is not symmetric under the kept reference treatment)."""
    for n, mdh, pris, seed in ((4, False, (0, 2), 41), (5, True, (1, 3), 42)):
        rob, q0, ref = regular(lambda rng: dh_arm(rng, n, mdh, pris), R.dh_rne, n, 0.25, lambda rng: rng.uniform(-0.5, 0.5, n), seed)
        assert all((l.sigma == 1) == (j in pris) for j, l in enumerate(rob.links))
        check_steps(rob.fdyn(0.25, q0), ref, f"prismatic n={n} mdh={mdh}")
        qd0 = np.linspace(-0.5, 0.5, n)
        ref = R.fdyn(R.dh_accel(rob), n, 0.2, q0, qd0=qd0, solver_args=TIGHT, dt=0.02)
        check_grid(rob.fdyn(0.2, q0, qd0=qd0, solver_args=TIGHT, dt=0.02), ref, f"prismatic n={n} grid")
    bad = dh_arm(np.random.default_rng(3), 3, True, (0,))
    with pytest.raises(ValueError, match="prismatic first joint"):
        bad.fdyn(0.1, np.zeros(3))


def test_coulomb_friction_away_from_zero_velocity():
    """Coulomb friction is a step in qd at 0 where adaptive integrators chatter (the reference too): start every joint
    well away from rest and check on the reference that no velocity changes sign within T."""
    for n, mdh, seed in ((3, False, 61), (5, True, 62)):
        rng = np.random.default_rng(seed)
        rob = dh_arm(rng, n, mdh, coulomb=True)
        assert (rob._pack_rne().reshape(n, 24)[:, 22:] != 0).all()
        q0, qd0 = rng.uniform(-1, 1, n), rng.choice([-1, 1], n) * rng.uniform(2, 3, n)
        acc = R.dh_accel(rob, [0, 0, 0])
        ref = R.fdyn(acc, n, 0.1, q0, qd0=qd0)
        assert R.keeps_velocity_signs(R.fdyn(acc, n, 0.1, q0, qd0=qd0, solver_args=TIGHT, dt=0.002).qd)
        check_steps(rob.fdyn(0.1, q0, qd0=qd0, gravity=[0, 0, 0]), ref, f"coulomb n={n}")
        ref = R.fdyn(acc, n, 0.1, q0, qd0=qd0, solver_args=TIGHT, dt=0.01)
        check_grid(rob.fdyn(0.1, q0, qd0=qd0, gravity=[0, 0, 0], solver_args=TIGHT, dt=0.01), ref, f"coulomb n={n} grid")


# ------------------------------------------------------------------ trees
@pytest.mark.parametrize("case", [1, 3, 7, 12, 16, "urdf"])
def test_tree_robots(case):
    """Robot.fdyn on random branched trees up to the 16-joint maximum and on two_arm.urdf."""
    if case == "urdf":
        rob = Robot.URDF(os.path.join(URDF_DIR, "two_arm.urdf"))
        n = rob.n
        rng = np.random.default_rng(71)
        q0 = rng.uniform(-0.5, 0.5, n)
        for l in rob.links:  # point masses on their own joint axes make M singular; move them off-axis
            if l.isjoint:
                l.r = (rng.uniform(0.1, 0.3, 3) * rng.choice([-1, 1], 3)).tolist()
                l.m = max(float(l.m), 0.5)
        rob = Robot(rob.links)
        ref = R.fdyn(R.tree_accel(rob), n, 0.2, q0)
        assert R.max_cond(R.tree_rne(rob), n, ref.q) < 1e6
    else:
        n = case
        rob, q0, ref = regular(lambda rng: tree_robot(rng, n), R.tree_rne, n, 0.2, lambda rng: rng.uniform(-1, 1, n), 700 + n)
    assert rob.n == n
    check_steps(rob.fdyn(0.2, q0), ref, f"tree {case}", TREE_TQ, TREE_TQD)
    rng = np.random.default_rng(n)
    tau, qd0, g = rng.normal(size=n), rng.uniform(-1, 1, n), np.array([0.0, -2.0, -9.81])
    ref = R.fdyn(R.tree_accel(rob, g), n, 0.2, q0, qd0=qd0, torque=lambda t, q, qd: tau, solver_args=dict(rtol=1e-7, atol=1e-10), dt=0.03)
    check_grid(rob.fdyn(0.2, q0, qd0=qd0, Q=tau, gravity=g, solver_args=dict(rtol=1e-7, atol=1e-10), dt=0.03), ref, f"tree {case} grid",
               TREE_TQ, TREE_TQD)


# ------------------------------------------------------------------ torque laws, initial velocities
def test_torque_laws_and_initial_velocity_forms():
    n = 4
    rob, q0, _ = regular(lambda rng: dh_arm(rng, n, False), R.dh_rne, n, 0.2, lambda rng: rng.uniform(-1, 1, n), 81)
    acc = R.dh_accel(rob)
    rng = np.random.default_rng(82)
    Bn = 5
    Q0 = q0 + rng.uniform(-0.5, 0.5, (Bn, n))
    QD0 = rng.uniform(-1, 1, (Bn, n))
    TAU = rng.normal(scale=5, size=(Bn, n))
    sa = dict(rtol=1e-7, atol=1e-10)
    T, dt = 0.2, 0.02
    # (B, n) torques per trajectory, from a host array and from a device tensor
    ens_h = rob.fdyn(T, Q0, qd0=QD0, Q=TAU, solver_args=sa, dt=dt)
    ens_d = rob.fdyn(T, dev(Q0), qd0=dev(QD0), Q=dev(TAU), solver_args=sa, dt=dt)
    assert isinstance(ens_h.q, np.ndarray) and ens_d.q.is_cuda
    assert np.array_equal(ens_h.q, ens_d.q.cpu().numpy()) and np.array_equal(ens_h.qd, ens_d.qd.cpu().numpy())
    for i in range(Bn):
        ref = R.fdyn(acc, n, T, Q0[i], qd0=QD0[i], torque=lambda t, q, qd, i=i: TAU[i], solver_args=sa, dt=dt)
        check_grid(type(ref)(ens_h.t, ens_h.q[i], ens_h.qd[i], *ref[3:]), ref, f"tau_rows row {i}")
    # (n,) constant torque; PD with scalar and per-joint gains; no torque
    kp, kd = rng.uniform(20, 80, n), rng.uniform(2, 6, n)
    for Q, law in ((TAU[0], lambda t, q, qd: TAU[0]), (("pd", 50.0, 4.0, q0), pd(50.0, 4.0, q0)),
                   (("pd", kp, kd, np.zeros(n)), pd(kp, kd, np.zeros(n))), (None, None)):
        ref = R.fdyn(acc, n, T, Q0[1], qd0=QD0[1], torque=law, solver_args=STEPS)
        check_steps(rob.fdyn(T, Q0[1], qd0=QD0[1], Q=Q, solver_args=STEPS), ref, f"torque {Q}")
    # qd0: None, (n,) broadcast to every row, (1, n) broadcast, (B, n)
    for qd0, rows in ((None, np.zeros((Bn, n))), (QD0[2], np.tile(QD0[2], (Bn, 1))), (QD0[2:3], np.tile(QD0[2], (Bn, 1))), (QD0, QD0)):
        ens = rob.fdyn(T, Q0, qd0=qd0, solver_args=sa, dt=dt)
        for i in (0, Bn - 1):
            ref = R.fdyn(acc, n, T, Q0[i], qd0=rows[i], solver_args=sa, dt=dt)
            check_grid(type(ref)(ens.t, ens.q[i], ens.qd[i], *ref[3:]), ref, f"qd0 {np.shape(qd0)} row {i}")
    # the callable route: scipy on the host around this robot's accel kernel
    tau = TAU[3]
    got = rob.fdyn(T, q0, Q=lambda robot, t, q, qd: tau, solver_args=STEPS)
    check_steps(got, R.fdyn(acc, n, T, q0, torque=lambda t, q, qd: tau, solver_args=STEPS), "callable Q")


# ------------------------------------------------------------------ step control
def test_step_control_options():
    n = 6
    rob, q0, _ = regular(lambda rng: dh_arm(rng, n, False), R.dh_rne, n, 0.2, lambda rng: rng.uniform(-1, 1, n), 91)
    acc = R.dh_accel(rob)
    T = 0.2
    # a max_step that binds
    ref = R.fdyn(acc, n, T, q0, solver_args=dict(max_step=0.01))
    assert ref.steps.max() <= 0.01 * (1 + 1e-12) and ref.accepted >= T / 0.01
    check_steps(rob.fdyn(T, q0, solver_args=dict(max_step=0.01)), ref, "max_step")
    # a given first step (no automatic selection), small and too large for the tolerance
    for fs in (1e-4, 0.15):
        ref = R.fdyn(acc, n, T, q0, solver_args=dict(STEPS, first_step=fs))
        assert ref.steps[0] <= fs
        check_steps(rob.fdyn(T, q0, solver_args=dict(STEPS, first_step=fs)), ref, f"first_step {fs}")
    assert R.fdyn(acc, n, T, q0, solver_args=dict(STEPS, first_step=0.15)).rejected > 0
    # rejected steps without a given first step: a stiff PD law from a large initial velocity
    law = ("pd", 4000.0, 20.0, np.zeros(n))
    qd0 = np.full(n, 6.0)
    ref = R.fdyn(acc, n, T, q0, qd0=qd0, torque=pd(*law[1:]))
    assert ref.rejected > 0, ref.rejected
    check_steps(rob.fdyn(T, q0, qd0=qd0, Q=law), ref, "rejections")
    # tight tolerances, on a grid
    ref = R.fdyn(acc, n, T, q0, qd0=qd0, solver_args=TIGHT, dt=0.01)
    check_grid(rob.fdyn(T, q0, qd0=qd0, solver_args=TIGHT, dt=0.01), ref, "tight")


def test_solver_args_follow_scipy():
    """first_step <= 0 or > T, rtol under scipy's floor and a vector atol are handled as scipy handles them (or, for a
    vector atol the device cannot take, refused with a ValueError)."""
    from scipy import integrate

    n = 3
    rob, q0, _ = regular(lambda rng: dh_arm(rng, n, False), R.dh_rne, n, 0.2, lambda rng: rng.uniform(-1, 1, n), 95)
    f = lambda t, y: -y  # noqa: E731
    for fs, msg in ((0.0, "must be positive"), (-1e-3, "must be positive"), (0.3, "exceeds bounds")):
        with pytest.raises(ValueError, match=msg):
            integrate.RK45(f, 0.0, np.ones(2 * n), 0.2, first_step=fs)
        with pytest.raises(ValueError, match=msg):
            rob.fdyn(0.2, q0, solver_args=dict(first_step=fs))
    eps = np.finfo(float).eps
    with pytest.warns(UserWarning, match="rtol"):
        integrate.RK45(f, 0.0, np.ones(2 * n), 0.2, rtol=1e-16)
    with pytest.warns(UserWarning, match="rtol"):
        low = rob.fdyn(0.2, q0, solver_args=dict(rtol=1e-16, atol=1e-12), max_steps=20000)
    floor = rob.fdyn(0.2, q0, solver_args=dict(rtol=100 * eps, atol=1e-12), max_steps=20000)
    assert np.array_equal(low.t, floor.t) and np.array_equal(low.q, floor.q) and np.array_equal(low.qd, floor.qd)
    integrate.RK45(f, 0.0, np.ones(2 * n), 0.2, atol=np.full(2 * n, 1e-6))  # scipy takes a vector atol
    with pytest.raises(ValueError, match="scalar"):
        rob.fdyn(0.2, q0, solver_args=dict(atol=np.full(2 * n, 1e-6)))


# ------------------------------------------------------------------ output modes
def test_output_modes():
    n = 3
    rob, q0, _ = regular(lambda rng: dh_arm(rng, n, True), R.dh_rne, n, 0.3, lambda rng: rng.uniform(-1, 1, n), 101)
    acc = R.dh_accel(rob)
    sa = dict(rtol=1e-8, atol=1e-10)
    # grids: T/dt not an integer; T/dt that looks like one (0.3/0.1 -> 3 samples); last sample on T; a single sample
    for T, dt, M in ((0.3, 0.07, 5), (0.3, 0.1, 3), (2.1, 0.3, 8), (0.2, 0.2, 1), (0.2, 0.5, 1)):
        ref = R.fdyn(acc, n, T, q0, solver_args=sa, dt=dt)
        assert len(ref.t) == M
        got = rob.fdyn(T, q0, solver_args=sa, dt=dt)
        check_grid(got, ref, f"grid T={T} dt={dt}")
        ens = rob.fdyn(T, np.stack([q0, q0]), solver_args=sa, dt=dt)
        assert ens.q.shape == (2, M, n) and np.array_equal(ens.q[1], got.q) and np.array_equal(ens.t, ref.t)
    # steps: one trajectory trimmed to its count; an ensemble padded with NaN past each row's count
    rng = np.random.default_rng(102)
    Q0 = np.stack([q0, q0 + 0.3, q0 - 0.2])
    QD0 = np.array([np.zeros(n), np.full(n, 4.0), rng.uniform(-1, 1, n)])
    ens = rob.fdyn(0.3, Q0, qd0=QD0, solver_args=STEPS)
    assert ens.t.shape == (3, 4096) and ens.q.shape == (3, 4096, n)
    for i in range(3):
        ref = R.fdyn(acc, n, 0.3, Q0[i], qd0=QD0[i], solver_args=STEPS)
        c = int(ens.count[i])
        assert c == len(ref.t)
        check_steps(type(ref)(ens.t[i, :c], ens.q[i, :c], ens.qd[i, :c], *ref[3:]), ref, f"ensemble steps row {i}")
        assert np.isnan(ens.t[i, c:]).all() and np.isnan(ens.q[i, c:]).all() and np.isnan(ens.qd[i, c:]).all()
    # max_steps: exceeded by one row -> RuntimeError; exactly enough for every row -> no error
    big = int(ens.count.max())
    assert ens.count.min() < big
    with pytest.raises(RuntimeError, match="max_steps"):
        rob.fdyn(0.3, Q0, qd0=QD0, solver_args=STEPS, max_steps=big - 1)
    fit = rob.fdyn(0.3, Q0, qd0=QD0, solver_args=STEPS, max_steps=big)
    assert fit.t.shape == (3, big) and np.array_equal(fit.count, ens.count)
    assert np.array_equal(fit.q, ens.q[:, :big], equal_nan=True)


# ------------------------------------------------------------------ ensembles
@pytest.mark.parametrize("Bn", [1, 63, 64, 65, 200])
def test_ensembles_mix_busy_and_quiet_lanes(Bn):
    """Every warp mixes lanes that need many steps (large velocity, large torque) with lanes that sit in static
    equilibrium (qd0 = 0, torque = gravity load).  Sampled rows against their own scipy run, and bit for bit against a
    one-trajectory call on that row: the same program in the same lane position, so any difference is a leak between
    lanes or a row indexed wrongly."""
    n = 3
    rob, q0, _ = regular(lambda rng: dh_arm(rng, n, False), R.dh_rne, n, 0.2, lambda rng: rng.uniform(-1, 1, n), 111)
    acc, rne = R.dh_accel(rob), R.dh_rne(rob)
    rng = np.random.default_rng(112 + Bn)
    Q0 = q0 + rng.uniform(-0.5, 0.5, (Bn, n))
    busy = rng.random(Bn) < 0.5
    busy[0] = True
    if Bn > 1:
        busy[-1] = False
    QD0 = np.where(busy[:, None], rng.choice([-1, 1], (Bn, n)) * rng.uniform(20, 30, (Bn, n)), 0.0)
    TAU = np.where(busy[:, None], rng.normal(scale=300, size=(Bn, n)), orc.dyn_gravload(rne, n, Q0, rob.gravity))
    T, sa = 0.2, STEPS
    ens = rob.fdyn(T, dev(Q0), qd0=dev(QD0), Q=dev(TAU), solver_args=sa)
    assert ens.q.is_cuda and ens.t.shape == (Bn, 4096)
    count = ens.count.cpu().numpy()
    t, q, qd = (x.cpu().numpy() for x in (ens.t, ens.q, ens.qd))
    assert (~busy).sum() == 0 or count[busy].min() > count[~busy].max()
    rows = sorted({0, Bn // 2, Bn - 1} | ({31, 32, 63, 64} & set(range(Bn))))
    for i in rows:
        ref = R.fdyn(acc, n, T, Q0[i], qd0=QD0[i], torque=lambda tt, a, b, i=i: TAU[i], solver_args=sa)
        c = int(count[i])
        assert c == len(ref.t), (i, c, len(ref.t))
        # busy lanes move at 20-30 rad/s, so the few 1e-10 s by which step times drift move q by up to 1e-8
        check_steps(type(ref)(t[i, :c], q[i, :c], qd[i, :c], *ref[3:]), ref, f"B={Bn} row {i} busy={busy[i]}",
                    dict(rtol=1e-7, atol=2e-8), dict(rtol=1e-6, atol=2e-7))
        one = rob.fdyn(T, Q0[i], qd0=QD0[i], Q=TAU[i:i + 1], solver_args=sa)
        assert np.array_equal(one.t, t[i, :c]) and np.array_equal(one.q, q[i, :c]) and np.array_equal(one.qd, qd[i, :c]), i
        assert np.isnan(t[i, c:]).all()
    # the same ensemble on a grid: numpy in, numpy out; every row bit for bit its one-trajectory run
    grid = rob.fdyn(T, Q0, qd0=QD0, Q=TAU, solver_args=sa, dt=0.03)
    assert isinstance(grid.q, np.ndarray) and grid.q.shape == (Bn, 7, n)
    for i in rows:
        one = rob.fdyn(T, Q0[i], qd0=QD0[i], Q=TAU[i:i + 1], solver_args=sa, dt=0.03)
        assert np.array_equal(one.q, grid.q[i]) and np.array_equal(one.qd, grid.qd[i]), i


# ------------------------------------------------------------------ fp32
def fp32_case(rob, acc, n, q0, qd0, T, dt, Q=None, torque=None, **kw):
    """The fp32 device run (rtol 1e-4, atol 1e-7, its own steps) against a true solution on the grid: its error must
    stay within 20 times scipy's own error at those tolerances, plus 1e-4 max(1, |x|)."""
    q0 = np.asarray(q0, np.float32).astype(np.float64)
    qd0 = np.asarray(qd0, np.float32).astype(np.float64)
    loose = dict(rtol=1e-4, atol=1e-7)
    true = R.fdyn(acc, n, T, q0, qd0=qd0, torque=torque, solver_args=TIGHT, dt=dt)
    sp = R.fdyn(acc, n, T, q0, qd0=qd0, torque=torque, solver_args=loose, dt=dt)
    a = rob.fdyn(T, q0, qd0=qd0, Q=Q, solver_args=loose, dt=dt, dtype=np.float32, **kw)
    b = rob.fdyn(T, q0.astype(np.float32), qd0=qd0.astype(np.float32), Q=Q, solver_args=loose, dt=dt, **kw)
    for got in (a, b):
        assert got.q.dtype == np.float32 and got.q.shape == true.q.shape, (got.q.dtype, got.q.shape, true.q.shape)
        np.testing.assert_allclose(got.t, true.t, rtol=1e-6, atol=1e-7)
        for x, y, z in ((got.q, true.q, sp.q), (got.qd, true.qd, sp.qd)):
            err, bar = np.abs(x - y).max(), 20 * np.abs(z - y).max() + 1e-4 * max(1.0, np.abs(y).max())
            assert err <= bar, (err, bar)
    return true


@pytest.mark.parametrize("case", ["dh2", "dh6", "dh9", "tree5"])
def test_fp32(case):
    if case == "tree5":
        n = 5
        rob, q0, _ = regular(lambda rng: tree_robot(rng, n), R.tree_rne, n, 0.3, lambda rng: rng.uniform(-1, 1, n), 121)
        acc = R.tree_accel(rob)
    else:
        n = int(case[2:])
        rob, q0, _ = regular(lambda rng: dh_arm(rng, n, n == 6), R.dh_rne, n, 0.3, lambda rng: rng.uniform(-1, 1, n), 120 + n)
        acc = R.dh_accel(rob)
    qd0 = np.random.default_rng(n).uniform(-1, 1, n)
    fp32_case(rob, acc, n, q0, qd0, 0.3, 0.02)
    # ensemble in fp32: a CUDA tensor in gives a tensor out; a single trajectory comes back as numpy
    ens = rob.fdyn(0.3, dev(np.stack([q0, q0]), np.float32), solver_args=dict(rtol=1e-4, atol=1e-7), dt=0.02)
    assert ens.q.is_cuda and ens.q.dtype == torch.float32
    one = rob.fdyn(0.3, dev(q0, np.float32), solver_args=dict(rtol=1e-4, atol=1e-7), dt=0.02)
    assert isinstance(one.q, np.ndarray) and np.array_equal(one.q, ens.q[1].cpu().numpy())


def test_grid_ending_on_T_in_both_dtypes():
    """np.arange(0, 2.1, 0.3) has 8 samples and the last one is T itself; in fp32 7 * 0.3f rounds above (float)2.1,
    so the last sample is never reached by a step: it must still be written, from the state at T."""
    n = 2
    rob, q0, _ = regular(lambda rng: dh_arm(rng, n, False), R.dh_rne, n, 0.3, lambda rng: rng.uniform(-1, 1, n), 131)
    acc = R.dh_accel(rob, [0, 0, 0])
    law = ("pd", 20.0, 5.0, np.zeros(n))
    T, dt = 2.1, 0.3
    assert len(np.arange(0, T, dt)) == 8 and np.float32(7) * np.float32(dt) > np.float32(T)
    sa = dict(rtol=1e-8, atol=1e-10)
    ref = R.fdyn(acc, n, T, q0, torque=pd(*law[1:]), solver_args=sa, dt=dt)
    check_grid(rob.fdyn(T, q0, Q=law, gravity=[0, 0, 0], solver_args=sa, dt=dt), ref, "fp64 T=2.1 dt=0.3")
    true = fp32_case(rob, acc, n, q0, np.zeros(n), T, dt, Q=law, torque=pd(*law[1:]), gravity=[0, 0, 0])
    q32 = np.asarray(q0, np.float32)
    ens = rob.fdyn(T, np.stack([q32, q32, q32]), Q=law, gravity=[0, 0, 0], solver_args=dict(rtol=1e-4, atol=1e-7), dt=dt)
    assert ens.q.shape == (3, 8, n) and np.isfinite(ens.q).all() and np.isfinite(ens.qd).all()
    one = rob.fdyn(T, q32, Q=law, gravity=[0, 0, 0], solver_args=dict(rtol=1e-4, atol=1e-7), dt=dt)
    assert np.array_equal(one.q, ens.q[2]) and np.array_equal(one.qd, ens.qd[2])
    assert np.abs(ens.q[:, -1] - true.q[-1]).max() < 1e-3


# ------------------------------------------------------------------ C ABI argument checks
def test_c_abi_rejects_bad_arguments_before_any_launch():
    lib = rtb._lib.lib()
    n = 3
    arm = dh_arm(np.random.default_rng(141), n, False)
    tree = tree_robot(np.random.default_rng(142), n)
    handles = {"b2k_rne_fdyn": arm._rne_handle(), "b2k_tree_fdyn": tree._tree_handle()}
    q0 = dev(np.zeros((2, n)))
    M = 4
    out_t, out_q, out_qd = dev(np.zeros((2, M))), dev(np.zeros((2, M, n))), dev(np.zeros((2, M, n)))
    cnt, st = torch.zeros(2, dtype=torch.int32, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    g = np.array([0.0, 0.0, 9.81])
    tau = np.ones(n)
    tau_rows = dev(np.ones((2, n)))
    vp = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
    good = dict(dtype=1, T=0.1, mode=1, tau=tau, tau_rows=None, rtol=1e-3, atol=1e-6, max_step=np.inf, first_step=0.0, dt=0.05, grid=1, M=2)
    bad = [dict(handle=None), dict(dtype=7), dict(mode=4), dict(tau=None), dict(mode=2, tau_rows=None), dict(M=0), dict(dt=0.0),
           dict(dt=-0.1), dict(max_step=0.0), dict(rtol=0.0), dict(atol=-1e-9)]
    for name, h in handles.items():
        fn = getattr(lib, name)

        def call(handle=h, **kw):
            a = dict(good, **kw)
            return fn(handle, a["dtype"], vp(q0), None, 2, a["T"], rtb._lib.dptr(g), a["mode"], rtb._lib.dptr(a["tau"]),
                      None if a["tau_rows"] is None else vp(a["tau_rows"]), None, None, None, a["rtol"], a["atol"], a["max_step"],
                      a["first_step"], a["dt"], a["grid"], a["M"], vp(out_t), vp(out_q), vp(out_qd), vp(cnt), vp(st), None)

        for kw in bad:
            n0 = rtb.launch_count()
            assert call(**kw) == -1, (name, kw)
            assert rtb.launch_count() == n0, (name, kw)
        n0 = rtb.launch_count()
        assert call() == 0 and call(mode=2, tau_rows=tau_rows) == 0
        assert rtb.launch_count() == n0 + 2
        torch.cuda.synchronize()
        assert (st == 0).all() and (cnt == 2).all()
