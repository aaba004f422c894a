"""DHRobot.rollout / Robot.rollout on the GPU against the float64 RK4 restatement of tests/rollout_ref.py.

Bounds, relative to the largest entry of the reference (at least 1): states fp64 1e-10, fp32 1e-3 (K <= 10).  A and B:
fp64 against the complex step of the tree's whole RK4 map 1e-9; against the DH chained reference 1e-6, the accuracy of
its Richardson-differenced accel_derivatives (about 1e-8 relative) carried through four stages; fp32 1e-3 max(1,
kappa(M) / 100).  The reference runs Python recursions per state, so large batches are checked on the rows around the
64-lane block edges, the first and the last rows."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import rollout_ref as ref  # noqa: E402

URDF_DIR = os.path.join(os.path.dirname(__file__), "golden", "urdf")
DH = ("Puma560", "PandaMDH", "UR10")
TREES = ("two_arm", "panda_ets", "random9", "random16")


def random_robot(rng, n):
    """A branched tree of revolute joints (the last one prismatic) with point masses off every joint axis, so that M is
    well conditioned."""
    ET, ETS, Link = rtb.ET, rtb.ETS, rtb.Link
    links = []
    for j in range(n):
        parent = None if j == 0 else links[int(rng.integers(0, len(links)))]
        consts = ETS()
        for _ in range(int(rng.integers(0, 3))):
            kind = int(rng.integers(0, 6))
            val = float(rng.choice([np.pi / 2, -np.pi / 2, rng.uniform(-1, 1)])) if kind < 3 else float(rng.uniform(-0.4, 0.4))
            consts = consts * getattr(ET, ("Rx", "Ry", "Rz", "tx", "ty", "tz")[kind])(val)
        axis = int(rng.integers(0, 3)) + (3 if j == n - 1 else 0)
        joint = getattr(ET, ("Rx", "Ry", "Rz", "tx", "ty", "tz")[axis])(flip=bool(rng.integers(0, 2)))
        links.append(Link(consts * joint, name=f"j{j}", parent=parent, m=float(rng.uniform(0.5, 3)),
                          r=(rng.uniform(0.05, 0.2, 3) * rng.choice([-1, 1], 3)).tolist()))
    return rtb.Robot(links)


def robot_of(name):
    if name in DH:
        return getattr(rtb.models, name)()
    if name == "two_arm":
        return rtb.Robot.URDF(os.path.join(URDF_DIR, "two_arm.urdf"))
    if name == "panda_ets":  # the kinematic Panda with point masses off the joint axes, so that M is regular
        r = rtb.models.Panda()
        for k, l in enumerate(r.links):
            l.m, l.r = 1.0 + 0.2 * k, [0.03, -0.02, 0.05]
        return r
    n = int(name[6:])
    return random_robot(np.random.default_rng(40 + n), n)


def model_of(rob):
    if isinstance(rob, rtb.DHRobot):
        return ref.dh(rob._pack_rne(), rob.mdh, rob._kernel_gravity(None))
    return ref.tree(rob.tree_description(), rob.gravity)


def inputs(rob, N, K, rng, dt=np.float64):
    n = rob.n
    q0, qd0 = rng.uniform(-1.5, 1.5, (N, n)), rng.uniform(-1, 1, (N, n))
    qd0[:, 0] = np.where(rng.uniform(size=N) < 0.5, 0.3, -0.3)  # the Coulomb step stays away from the samples
    tau = rng.normal(size=(N, K, n))
    return tuple(a.astype(dt).astype(np.float64) for a in (q0, qd0, tau))


def cuda(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()


def edge_rows(N):
    return sorted({0, N - 1} | {i for e in range(64, N, 64) for i in (e - 1, e) if i < N})[:8]


def check(got, want, tol):
    got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    assert got.shape == want.shape, (got.shape, want.shape)
    assert np.all(np.isfinite(got))
    err = float(np.abs(got.astype(np.float64) - want).max()) / max(1.0, float(np.abs(want).max()))
    assert err <= tol, (err, tol)


def kappa_max(rob, q):
    if isinstance(rob, rtb.DHRobot):
        M = ref.dref.inertia(rob._pack_rne(), rob.mdh, q)
    else:
        M = [ref.tref.inertia(rob.tree_description(), x) for x in q]
    return max(np.linalg.cond(m) for m in M)


@pytest.mark.parametrize("name", DH + TREES)
@pytest.mark.parametrize("N,K", [(1, 1), (63, 2), (65, 2), (4097, 2), (64, 50)])
def test_states_and_sensitivities_fp64(name, N, K):
    rob = robot_of(name)
    rng = np.random.default_rng(N + K)
    q0, qd0, tau = inputs(rob, N, K, rng)
    h = 0.01 if K <= 2 else 0.002  # 0.1 s: the light links of two_arm and the Panda are fast under random torques
    out = rob.rollout(cuda(q0, np.float64), cuda(tau, np.float64), h, qd0=cuda(qd0, np.float64), sensitivities=True)
    rows = edge_rows(N)
    if K == 50:
        rows = rows[:2]
    model = model_of(rob)
    sens = K <= 2
    wq, wqd, wA, wB = ref.rollout(model, q0[rows], qd0[rows], tau[rows], h, sensitivities=sens and isinstance(rob, rtb.DHRobot))
    check(out.q[rows], wq, 1e-10)
    check(out.qd[rows], wqd, 1e-10)
    if not sens:
        return
    if isinstance(rob, rtb.DHRobot):
        check(out.A[rows], wA, 1e-6)
        check(out.B[rows], wB, 1e-6)
    else:  # the complex step of each step's whole map, at the device's own states
        x = np.concatenate([wq, wqd], axis=2)
        for k in range(K):
            A, B = ref.complex_step(model[0], x[:, k], tau[rows, k], h)
            check(out.A[rows, k], A, 1e-9)
            check(out.B[rows, k], B, 1e-9)


@pytest.mark.parametrize("name", DH + ("two_arm", "random16"))
def test_fp32(name):
    rob = robot_of(name)
    rng = np.random.default_rng(7)
    N, K = 65, 10
    q0, qd0, tau = inputs(rob, N, K, rng, np.float32)
    out = rob.rollout(cuda(q0, np.float32), cuda(tau, np.float32), 0.01, qd0=cuda(qd0, np.float32), sensitivities=True)
    assert out.q.dtype == torch.float32 and out.A.dtype == torch.float32
    rows = edge_rows(N)
    o64 = rob.rollout(cuda(q0[rows], np.float64), cuda(tau[rows], np.float64), 0.01, qd0=cuda(qd0[rows], np.float64),
                      sensitivities=True)
    kap = kappa_max(rob, q0[rows])
    check(out.q[rows], o64.q.cpu().numpy(), 1e-3)
    check(out.qd[rows], o64.qd.cpu().numpy(), 1e-3)
    check(out.A[rows, :2], o64.A[:, :2].cpu().numpy(), 1e-3 * max(1.0, kap / 100))
    check(out.B[rows, :2], o64.B[:, :2].cpu().numpy(), 1e-3 * max(1.0, kap / 100))
    wq, wqd, _, _ = ref.rollout(model_of(rob), q0[rows[:2]], qd0[rows[:2]], tau[rows[:2]], 0.01, sensitivities=False)
    check(out.q[rows[:2]], wq, 1e-3)
    check(out.qd[rows[:2]], wqd, 1e-3)


@pytest.mark.parametrize("name", DH + ("two_arm", "random16"))
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_states_only_and_sensitivities_programs_give_identical_states(name, dt):
    rob = robot_of(name)
    q0, qd0, tau = inputs(rob, 1000, 50, np.random.default_rng(3), dt)
    a = rob.rollout(cuda(q0, dt), cuda(tau, dt), 0.002, qd0=cuda(qd0, dt))
    b = rob.rollout(cuda(q0, dt), cuda(tau, dt), 0.002, qd0=cuda(qd0, dt), sensitivities=True)
    assert a.A is None and a.B is None
    bits = torch.int64 if dt == np.float64 else torch.int32  # bit patterns: equal NaNs count as equal
    assert torch.equal(a.q.view(bits), b.q.view(bits)) and torch.equal(a.qd.view(bits), b.qd.view(bits))


@pytest.mark.parametrize("name", DH + TREES)
def test_one_step_composed_from_the_public_accel_and_accel_derivatives(name):
    rob = robot_of(name)
    n, h = rob.n, 0.02
    q0, qd0, tau = inputs(rob, 5, 1, np.random.default_rng(11))
    out = rob.rollout(q0, tau, h, qd0=qd0, sensitivities=True)
    t = tau[:, 0]
    acc = lambda q, qd: rob.accel(q, qd, t)  # noqa: E731
    x = np.concatenate([q0, qd0], axis=1)
    I = np.eye(2 * n)
    ks, dx, du = [], [], []
    for c in (0.0, 0.5, 0.5, 1.0):
        xs = x if not ks else x + c * h * ks[-1]
        aq, aqd, at = rob.accel_derivatives(xs[:, :n], xs[:, n:], t)
        J = np.zeros((5, 2 * n, 2 * n))
        J[:, :n, n:] = np.eye(n)
        J[:, n:, :n], J[:, n:, n:] = aq, aqd
        dx.append(J @ (I if not ks else I + c * h * dx[-1]))
        du.append(J @ (np.zeros((5, 2 * n, n)) if not ks else c * h * du[-1]) + np.concatenate([np.zeros((5, n, n)), at], 1))
        ks.append(np.concatenate([xs[:, n:], acc(xs[:, :n], xs[:, n:])], axis=1))
    xn = x + h / 6 * (ks[0] + 2 * ks[1] + 2 * ks[2] + ks[3])
    check(out.q[:, 1], xn[:, :n], 1e-10)
    check(out.qd[:, 1], xn[:, n:], 1e-10)
    check(out.A[:, 0], I + h / 6 * (dx[0] + 2 * dx[1] + 2 * dx[2] + dx[3]), 1e-10)
    check(out.B[:, 0], h / 6 * (du[0] + 2 * du[1] + 2 * du[2] + du[3]), 1e-10)


@pytest.mark.parametrize("name", ("Puma560", "random9"))
def test_long_rollout_matches_fdyn(name):
    rob = robot_of(name)
    if isinstance(rob, rtb.DHRobot):
        rob = rob.nofriction()
    n, h, K = rob.n, 1e-3, 200
    rng = np.random.default_rng(5)
    q0, qd0, t = rng.uniform(-1, 1, (4, n)), rng.uniform(-0.5, 0.5, (4, n)), rng.normal(size=(4, n))
    out = rob.rollout(q0, np.repeat(t[:, None], K, axis=1), h, qd0=qd0)
    # fdyn interpolates its steps linearly onto the grid: max_step h / 10 keeps that below 1e-8 of the motion here
    fd = rob.fdyn(K * h, q0, Q=t, qd0=qd0, dt=h, solver_args={"rtol": 1e-10, "atol": 1e-12, "max_step": h / 10})
    assert fd.q.shape == (4, K, n)
    check(out.q[:, :K], fd.q, 1e-6)
    check(out.qd[:, :K], fd.qd, 1e-6)


def test_input_forms():
    rob = robot_of("Puma560")
    n, K = rob.n, 3
    q0, qd0, tau = inputs(rob, 4, K, np.random.default_rng(2))
    full = rob.rollout(q0, tau, 0.01, qd0=qd0, sensitivities=True)
    assert isinstance(full.q, np.ndarray) and full.q.shape == (4, K + 1, n) and full.A.shape == (4, K, 2 * n, 2 * n)
    assert full.B.shape == (4, K, 2 * n, n)
    np.testing.assert_array_equal(full.t, np.arange(K + 1) * 0.01)
    np.testing.assert_array_equal(full.q[:, 0], q0)
    one = rob.rollout(q0[1], tau[1], 0.01, qd0=qd0[1], sensitivities=True)  # single trajectory: no N axis
    assert one.q.shape == (K + 1, n) and one.A.shape == (K, 2 * n, 2 * n)
    np.testing.assert_array_equal(one.q, full.q[1])
    np.testing.assert_array_equal(one.B, full.B[1])
    shared = rob.rollout(q0, tau[2], 0.01, qd0=qd0)  # one torque sequence for every trajectory
    per = rob.rollout(q0, np.repeat(tau[2][None], 4, axis=0), 0.01, qd0=qd0)
    np.testing.assert_array_equal(shared.q, per.q)
    ten = rob.rollout(cuda(q0, np.float64), cuda(tau, np.float64), 0.01, qd0=cuda(qd0, np.float64), sensitivities=True)
    assert ten.q.is_cuda and ten.A.is_cuda
    np.testing.assert_array_equal(ten.A.cpu().numpy(), full.A)
    rest = rob.rollout(q0, tau, 0.01)  # qd0=None: at rest
    np.testing.assert_array_equal(rest.q, rob.rollout(q0, tau, 0.01, qd0=np.zeros((4, n))).q)
    bq = rob.rollout(q0[0], tau, 0.01, qd0=qd0[0])  # one initial state broadcast over per-trajectory torques
    assert bq.q.shape == (4, K + 1, n)
    bv = rob.rollout(q0[0], tau[2], 0.01, qd0=qd0, sensitivities=True)  # batched qd0 only: every trajectory comes back
    assert bv.q.shape == (4, K + 1, n) and bv.A.shape == (4, K, 2 * n, 2 * n)
    np.testing.assert_array_equal(bv.q, rob.rollout(np.repeat(q0[:1], 4, axis=0), tau[2], 0.01, qd0=qd0).q)


def test_empty_batch_launches_nothing():
    rob = robot_of("Puma560")
    n0 = rtb.launch_count()
    out = rob.rollout(np.zeros((0, 6)), np.zeros((2, 6)), 0.01, sensitivities=True)
    assert out.q.shape == (0, 3, 6) and out.A.shape == (0, 2, 12, 12)
    assert rtb.launch_count() == n0
