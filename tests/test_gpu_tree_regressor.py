"""Robot.rne_regressor / regressor_gram / identify on the GPU: the generated regressor kernel against the reference of
tests/tree_regressor_ref.py (10n restated rne calls per state), the identity Y pi = rne on named and random robots and on
a handle with full rigid-body inertias, the gram against a float64 einsum over the materialised Y, and identification.

Tolerances relative to max(|ref|, 1): fp64 1e-9, fp32 1e-3.  The reference is slow, so a batch is checked on its first
and last rows, the rows around each tile edge and a random sample."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import tree_regressor_ref as ref  # noqa: E402
from test_codegen_cpu import tree_handle  # noqa: E402
from test_gpu_tree import random_robot  # noqa: E402
from test_gpu_tree_derivs import puma_ets, rows_to_check  # noqa: E402

URDF_DIR = os.path.join(os.path.dirname(__file__), "golden", "urdf")


def cuda(x, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()


def states(rng, N, n, dt=np.float64):
    q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
    return tuple(a.astype(dt).astype(np.float64) for a in (q, qd, qdd))  # the reference sees the inputs the kernel sees


def check_rows(rob, Y, q, qd, qdd, grav, dt, rng):
    tree = rob.tree_description()
    g = rob.gravity if grav is None else np.asarray(grav, dtype=np.float64)
    Y = Y.cpu().numpy() if torch.is_tensor(Y) else Y
    assert np.all(np.isfinite(Y))
    tol = 1e-3 if dt == np.float32 else 1e-9
    for i in rows_to_check(len(q), rng):
        want = ref.regressor(tree, q[i], qd[i], qdd[i], g)
        err = np.abs(Y[i].astype(np.float64) - want).max() / max(1.0, np.abs(want).max())
        assert err <= tol, (i, err)
        for r in range(rob.n):  # the structural zeros are exact
            assert np.all(Y[i, r, np.repeat(~ref.below(tree, r), 10)] == 0)


@pytest.mark.parametrize("n", range(1, 17))
def test_random_trees_every_joint_count_against_the_reference(n):
    rng = np.random.default_rng(1100 + n)
    rob = random_robot(rng, n, n % 2 == 1)
    assert rob.n == n
    for dt in (np.float64, np.float32):
        for grav in (None, [0.6, -1.1, -9.5]):
            q, qd, qdd = states(rng, 33, n, dt)
            Y = rob.rne_regressor(cuda(q, dt), cuda(qd, dt), cuda(qdd, dt), gravity=grav)
            assert Y.dtype == (torch.float64 if dt == np.float64 else torch.float32) and tuple(Y.shape) == (33, n, 10 * n)
            check_rows(rob, Y, q, qd, qdd, grav, dt, rng)


@pytest.mark.parametrize("N", [1, 31, 32, 33, 1000])
def test_batch_sizes_and_tile_edges(N):
    rng = np.random.default_rng(1200 + N)
    for rob in (Robot_urdf(), random_robot(np.random.default_rng(41), 16, True)):
        for dt in (np.float64, np.float32):
            q, qd, qdd = states(rng, N, rob.n, dt)
            grav = None if dt == np.float64 else [0.3, 0.2, -9.81]
            check_rows(rob, rob.rne_regressor(cuda(q, dt), cuda(qd, dt), cuda(qdd, dt), gravity=grav), q, qd, qdd, grav, dt, rng)


def Robot_urdf():
    return rtb.Robot.URDF(os.path.join(URDF_DIR, "two_arm.urdf"))


@pytest.mark.parametrize("case", ["urdf", "puma_ets", "random9", "random16"])
def test_regressor_times_dynamic_parameters_is_rne(case):
    rng = np.random.default_rng(13)
    rob = {"urdf": Robot_urdf, "puma_ets": lambda: puma_ets(0.3)[0], "random9": lambda: random_robot(rng, 9, True),
           "random16": lambda: random_robot(rng, 16, False)}[case]()
    n = rob.n
    q, qd, qdd = (cuda(a) for a in states(rng, 5000, n))
    for grav in (None, [0.4, -0.3, -9.7]):
        tau = rob.rne(q, qd, qdd, gravity=grav).cpu().numpy()
        Y = rob.rne_regressor(q, qd, qdd, gravity=grav).cpu().numpy()
        got = Y @ rob.dynamic_parameters()
        np.testing.assert_allclose(got, tau, rtol=0, atol=1e-10 * max(1.0, np.abs(tau).max()))


def full_inertia_tree(rng, n):
    """A random robot's kinematics with full rigid-body group inertias (Ib not a point mass's): a handle made through the
    C ABI, which Robot.rne's point masses cannot express."""
    rob = random_robot(rng, n, True)
    tree = rob.tree_description()
    tree["I6"] = [ref.rigid_body_inertia(rng) for _ in range(n)]
    return rob, tree, tree_handle(tree)


def tree_rne(h, q, qd, qdd, agrav):
    tau = torch.empty_like(q)
    rtb._lib.check(rtb._lib.lib().b2k_tree_rne(h, rtb._lib.F64 if q.dtype == torch.float64 else rtb._lib.F32, q.data_ptr(),
                                               qd.data_ptr(), qdd.data_ptr(), q.shape[0], rtb._lib.dptr(agrav), tau.data_ptr(),
                                               None))
    torch.cuda.synchronize()
    return tau


def test_full_rigid_body_inertias_through_the_c_abi():
    rng = np.random.default_rng(17)
    rob, tree, h = full_inertia_tree(rng, 8)
    q, qd, qdd = (cuda(a) for a in states(rng, 2000, 8))
    tau = tree_rne(h, q, qd, qdd, -rob.gravity).cpu().numpy()
    Yc = torch.empty((2000, 8, 80), dtype=torch.float64, device="cuda")
    rtb._lib.check(rtb._lib.lib().b2k_tree_regressor(h, rtb._lib.F64, q.data_ptr(), qd.data_ptr(), qdd.data_ptr(), 2000,
                                                     rtb._lib.dptr(-rob.gravity), Yc.data_ptr(), None))
    Y = Yc.cpu().numpy()
    np.testing.assert_array_equal(Y, rob.rne_regressor(q, qd, qdd).cpu().numpy())  # Y does not depend on the inertias
    np.testing.assert_allclose(Y @ ref.dynamic_parameters(tree), tau, rtol=0, atol=1e-10 * max(1.0, np.abs(tau).max()))
    rtb._lib.lib().b2k_tree_destroy(h)


def test_regressor_is_bit_identical_after_the_masses_change():
    rng = np.random.default_rng(19)
    rob = random_robot(rng, 7, True)
    q, qd, qdd = (cuda(a) for a in states(rng, 777, 7))
    Y0 = rob.rne_regressor(q, qd, qdd).cpu().numpy()
    pi0 = rob.dynamic_parameters()
    for link in rob.links:
        link.m = 2 * link.m + 0.1
    assert not np.array_equal(rob.dynamic_parameters(), pi0)
    Y1 = rob.rne_regressor(q, qd, qdd).cpu().numpy()
    assert Y0.tobytes() == Y1.tobytes()
    tau = rob.rne(q, qd, qdd).cpu().numpy()
    np.testing.assert_allclose(Y1 @ rob.dynamic_parameters(), tau, rtol=0, atol=1e-10 * max(1.0, np.abs(tau).max()))


@pytest.mark.parametrize("n", [6, 16])
@pytest.mark.parametrize("N", [4095, 4096, 4097, 10000])
def test_gram_against_an_einsum_over_the_materialised_regressor(n, N):
    rng = np.random.default_rng(1300 + n + N)
    rob = random_robot(np.random.default_rng(60 + n), n, True)
    q, qd, qdd = (cuda(a) for a in states(rng, N, n))
    tau = rob.rne(q, qd, qdd) + 0.01 * torch.randn(N, n, dtype=torch.float64, device="cuda")
    Y = rob.rne_regressor(q, qd, qdd).cpu().numpy()
    t = tau.cpu().numpy()
    for w in (None, rng.uniform(0.2, 2.0, n)):
        ww = np.ones(n) if w is None else w
        G, b, s = rob.regressor_gram(q, qd, qdd, tau, weights=w)
        Gw = np.einsum("rip,i,riq->pq", Y, ww, Y)
        bw = np.einsum("rip,i,ri->p", Y, ww, t)
        sw = float(np.einsum("ri,i,ri->", t, ww, t))
        assert np.array_equal(G, G.T)
        np.testing.assert_allclose(G, Gw, rtol=0, atol=1e-11 * np.abs(Gw).max())
        np.testing.assert_allclose(b, bw, rtol=0, atol=1e-11 * np.abs(bw).max())
        assert abs(s - sw) <= 1e-11 * sw
        G2, b2, s2 = rob.regressor_gram(q, qd, qdd, tau, weights=w)
        assert G.tobytes() == G2.tobytes() and b.tobytes() == b2.tobytes() and s == s2
    # fp32 Y, fp64 sums
    G32, _, _ = rob.regressor_gram(q.float(), qd.float(), qdd.float(), tau.float())
    Gw = np.einsum("rip,riq->pq", Y, Y)
    np.testing.assert_allclose(G32, Gw, rtol=0, atol=1e-4 * np.abs(Gw).max())


def rms_floor(s, count):
    """What rms = sqrt((s - 2 pi.b + pi.G.pi) / count) resolves: about sqrt(eps) times the rms of tau."""
    return np.sqrt(16 * np.finfo(np.float64).eps * s / count)


def test_identify_on_torques_of_full_rigid_body_inertias():
    rng = np.random.default_rng(23)
    rob, tree, h = full_inertia_tree(rng, 7)
    n, N = 7, 20000
    q, qd, qdd = (cuda(a) for a in states(rng, N, n, np.float32))
    tau = tree_rne(h, q, qd, qdd, -rob.gravity)
    res = rob.identify(q, qd, qdd, tau)
    G, b, s = rob.regressor_gram(q, qd, qdd, tau)
    assert res.rms <= rms_floor(s, tau.numel()), (res.rms, rms_floor(s, tau.numel()))
    d = res.pi - ref.dynamic_parameters(tree)
    assert np.max(np.abs(G @ d)) <= 1e-7 * np.max(np.abs(b))
    # the rank is that of the stacked regressor with identify's zero columns and unit scaling
    qs, qds, qdds = (x[:400] for x in (q, qd, qdd))
    Ys = rob.rne_regressor(qs, qds, qdds).cpu().numpy().reshape(-1, 10 * n)
    norms = np.linalg.norm(Ys, axis=0)
    nz = norms > 16 * np.finfo(np.float64).eps * norms.max()
    sv = np.linalg.svd(Ys[:, nz] / norms[nz], compute_uv=False)
    small = rob.identify(qs, qds, qdds, tree_rne(h, qs, qds, qdds, -rob.gravity))
    assert small.rank == int(np.sum(sv ** 2 > 1e-10 * sv[0] ** 2))
    # float32: with an rcond above its rounding, no identifiable parameter is lost
    r32 = rob.identify(q.float(), qd.float(), qdd.float(), tau.float(), rcond=1e-5)
    assert r32.rank == res.rank, (r32.rank, res.rank)
    g = np.diag(G)
    nzg = g > 0
    assert np.max(np.abs(G @ (r32.pi - ref.dynamic_parameters(tree)))[nzg] / np.sqrt(g[nzg] * s)) < 1e-4
    rtb._lib.lib().b2k_tree_destroy(h)


@pytest.mark.parametrize("form", ["numpy", "single"])
def test_numpy_and_single_state_forms(form):
    rng = np.random.default_rng(29)
    rob = puma_ets(0.2)[0]
    q, qd, qdd = states(rng, 40, 6)
    for dt in (np.float64, np.float32):
        args = [a.astype(dt) for a in (q, qd, qdd)] if form == "numpy" else [a[0].astype(dt) for a in (q, qd, qdd)]
        Y = rob.rne_regressor(*args)
        assert isinstance(Y, np.ndarray) and Y.dtype == dt
        assert Y.shape == ((40, 6, 60) if form == "numpy" else (6, 60))
        Yd = rob.rne_regressor(*(cuda(a, dt) for a in (q, qd, qdd))).cpu().numpy()
        np.testing.assert_array_equal(Y if form == "numpy" else Y[None], Yd if form == "numpy" else Yd[:1])
        G, b, s = rob.regressor_gram(*args, args[0] * 0 + 1)
        assert G.shape == (60, 60) and b.shape == (60,) and isinstance(s, float)


def test_shape_errors_and_empty_batches():
    rob = puma_ets(0.2)[0]
    n0 = rtb.launch_count()
    x = cuda(np.zeros((4, 6)))
    with pytest.raises(ValueError):
        rob.rne_regressor(x, x, cuda(np.zeros((4, 5))))
    with pytest.raises(ValueError):
        rob.rne_regressor(x, x[:3], x)
    with pytest.raises(TypeError):
        rob.rne_regressor("q", x, x)
    with pytest.raises(ValueError):
        rob.regressor_gram(x, x, x, cuda(np.zeros((3, 6))))
    with pytest.raises(ValueError):
        rob.regressor_gram(x, x, x, x, weights=np.ones(5))
    with pytest.raises(ValueError, match="weights"):
        rob.regressor_gram(x, x, x, x, weights=-np.ones(6))
    e = cuda(np.zeros((0, 6)))
    assert tuple(rob.rne_regressor(e, e, e).shape) == (0, 6, 60)
    G, b, s = rob.regressor_gram(e, e, e, e)
    assert not G.any() and not b.any() and s == 0.0
    torch.cuda.synchronize()
    assert rtb.launch_count() == n0
    assert rob.rne_kernel_info(op="rne_regressor").startswith("k_rne_regressor_spec<double,tree n=6,mode=10>")
    assert rob.rne_kernel_info(np.float32, op="rne_regressor").startswith("k_rne_regressor_spec<float,tree n=6,mode=10>")
