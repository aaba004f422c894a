"""Robot.rne_derivatives / accel_derivatives on the GPU against the complex-step reference of tests/tree_derivs_ref.py,
and against the independent DH derivative kernel on a Puma built both ways.

Tolerances, relative to the largest entry of the reference (at least 1), as tests/test_gpu_rne_derivs.py sets them:
inverse mode fp64 1e-9, fp32 1e-3; forward mode fp64 1e-8 and fp32 1e-3, both widened by max(1, kappa(M) / 100) because
M^-1 carries the condition number of M.  The reference costs 2n Python recursions per state, so a batch is checked on
its first and last rows, the rows around each tile edge, and a random sample."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import rne_derivs_ref as DR  # noqa: E402
import tree_derivs_ref as ref  # noqa: E402
from oracle import chains as ch  # noqa: E402
from test_gpu_tree import random_robot  # noqa: E402

ET, ETS, Link, Robot = rtb.ET, rtb.ETS, rtb.Link, rtb.Robot
URDF_DIR = os.path.join(os.path.dirname(__file__), "golden", "urdf")


def cuda(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()


def rows_to_check(N, rng):
    r = {0, N - 1} | {i for e in range(32, N, 32) for i in (e - 1, e) if i < N}
    r |= set(int(i) for i in rng.integers(0, N, 6))
    return sorted(r)[:24]


def check(got, want, dt, forward=False, kappa=1.0):
    got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    assert got.shape == want.shape
    assert np.all(np.isfinite(got))
    scale = max(float(np.abs(want).max()), 1.0)
    tol = (1e-3 if dt == np.float32 else (1e-8 if forward else 1e-9)) * (max(1.0, kappa / 100) if forward else 1.0)
    err = float(np.abs(got.astype(np.float64) - want).max()) / scale
    assert err <= tol, (err, tol)


def puma_ets(bump=0.0):
    """The Puma560 DH table as an ETS robot (rotational inertia, motor and friction terms stripped, as Robot.rne has none);
    `bump` adds to every mass and centre-of-mass coordinate so that M is regular.  Returns (Robot, packed DH table)."""
    dh = ch.puma560_links()
    for l in dh:
        l.update(I=[0, 0, 0, 0, 0, 0], Jm=0.0, B=0.0, Tc=[0.0, 0.0], G=1.0, m=l["m"] + bump,
                 r=(np.asarray(l["r"], dtype=float) + bump / 10).tolist())
    links, prev = [], ETS()
    for j, l in enumerate(dh):
        post = ETS()
        for kind, v in (("tz", l["d"]), ("tx", l["a"]), ("Rx", l["alpha"])):
            if v != 0:
                post = post * getattr(ET, kind)(v)
        Tpost = np.eye(4)
        for et in post:
            Tpost = Tpost @ et.A()
        r_in = Tpost[:3, :3] @ np.asarray(l["r"], dtype=float) + Tpost[:3, 3]
        links.append(Link(prev * ET.Rz(), name=f"l{j}", parent=links[-1] if links else None, m=l["m"], r=r_in))
        prev = post
    links.append(Link(prev, name="tool", parent=links[-1]))
    return Robot(links), ch.pack_rne(dh)


def robot_of(case, rng):
    if case == "urdf":
        return Robot.URDF(os.path.join(URDF_DIR, "two_arm.urdf"))
    if case == "random7":
        return random_robot(rng, 7, True)
    return puma_ets(0.5)[0]


def run(rob, N, dt, rng, grav=None, form="tensor"):
    n = rob.n
    tree = rob.tree_description()
    g = rob.gravity if grav is None else np.asarray(grav, dtype=np.float64)
    q, qd, x = rng.uniform(-2, 2, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
    q, qd, x = (a.astype(dt).astype(np.float64) for a in (q, qd, x))  # the reference sees the inputs the kernel sees
    if form == "tensor":
        args = [cuda(a, dt) for a in (q, qd, x)]
    elif form == "numpy":
        args = [a.astype(dt) for a in (q, qd, x)]
    else:  # one state
        args = [a[0].astype(dt) for a in (q, qd, x)]
    dq, dqd = rob.rne_derivatives(*args, gravity=grav)
    fwd = rob.accel_derivatives(*args, gravity=grav)
    for o in (dq, dqd) + tuple(fwd):
        assert (torch.is_tensor(o) and o.is_cuda) if form == "tensor" else isinstance(o, np.ndarray)
        assert o.dtype == (torch.float64 if dt == np.float64 else torch.float32) if form == "tensor" else o.dtype == dt
        assert tuple(o.shape) == ((n, n) if form == "single" else (N, n, n))
    if form == "single":
        dq, dqd, fwd = dq[None], dqd[None], tuple(o[None] for o in fwd)
    regular = list(tree["jindex"]) == list(range(n))
    for i in rows_to_check(N if form != "single" else 1, rng):
        wq, wqd = ref.rne_derivatives(tree, q[i], qd[i], x[i], g)
        check(dq[i], wq, dt)
        check(dqd[i], wqd, dt)
        if regular:
            M = ref.inertia(tree, q[i])
            kappa = np.linalg.cond(M, p=np.inf)
            if kappa < 1e8:
                for got, want in zip(fwd, ref.accel_derivatives(tree, q[i], qd[i], x[i], g)):
                    check(got[i], want, dt, forward=True, kappa=kappa)


@pytest.mark.parametrize("case", ["urdf", "random7", "puma_ets"])
@pytest.mark.parametrize("N", [1, 31, 32, 33, 4097])
def test_named_robots_against_the_complex_step_reference(case, N):
    rng = np.random.default_rng({"urdf": 1, "random7": 2, "puma_ets": 3}[case] * 10000 + N)
    rob = robot_of(case, np.random.default_rng(40))
    run(rob, N, np.float64, rng, grav=None if N != 33 else [0.4, -0.3, -9.81])
    if N in (33, 4097):
        run(rob, N, np.float32, rng)


@pytest.mark.parametrize("form", ["numpy", "single"])
def test_numpy_and_single_state_forms(form):
    rng = np.random.default_rng(5)
    rob = robot_of("puma_ets", rng)
    run(rob, 40, np.float64, rng, form=form)
    run(rob, 40, np.float32, rng, form=form)


@pytest.mark.parametrize("n", range(1, 17))
def test_random_sweep_every_joint_count_both_dtypes(n):
    rng = np.random.default_rng(600 + n)
    rob = random_robot(rng, n, n % 2 == 1)
    assert rob.n == n
    for dt in (np.float64, np.float32):
        run(rob, 33, dt, rng)


def test_shape_and_type_errors_as_rne():
    rob = robot_of("puma_ets", np.random.default_rng(0))
    q = np.zeros((3, 6))
    with pytest.raises(ValueError):
        rob.rne_derivatives(q[:, :5], q, q)
    with pytest.raises(ValueError):
        rob.accel_derivatives(q, q[:2], q)
    with pytest.raises(TypeError):
        rob.rne_derivatives("q", q, q)
    assert rob.rne_kernel_info(op="rne_derivatives").startswith("k_rne_deriv_spec<double,tree n=6,mode=7>")
    assert rob.rne_kernel_info(np.float32, op="accel_derivatives").startswith("k_rne_deriv_spec<float,tree n=6,mode=8>")


def test_two_formulations_one_robot_agree_with_the_dh_derivative_kernel():
    """The Puma as an ETS tree (generated kernels) and as a DH table (the generic k_rne_deriv): same derivatives."""
    for bump in (0.0, 0.5):
        rob, L = puma_ets(bump)
        dh = DR.dhrobot(L, 0)
        rng = np.random.default_rng(8)
        N = 500
        q, qd, x = rng.uniform(-3, 3, (N, 6)), rng.normal(size=(N, 6)), rng.normal(size=(N, 6))
        args = [cuda(a, np.float64) for a in (q, qd, x)]
        for got, want in zip(rob.rne_derivatives(*args), dh.rne_derivatives(*args)):
            want = want.cpu().numpy()
            np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=1e-9 * max(1, np.abs(want).max()))
        if bump:  # a regular M (the stripped Puma's wrist masses sit on their joint axes)
            kappa = max(np.linalg.cond(M, p=np.inf) for M in rob.inertia(q))
            for got, want in zip(rob.accel_derivatives(*args), dh.accel_derivatives(*args)):
                want = want.cpu().numpy()
                np.testing.assert_allclose(got.cpu().numpy(), want, rtol=0, atol=1e-8 * max(1, kappa / 100) * max(1, np.abs(want).max()))
