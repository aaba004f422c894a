"""DHRobot.rne_derivatives / accel_derivatives on the GPU against the float64 finite-difference reference of
tests/rne_derivs_ref.py, and against the identities of rigid-body dynamics checked on the GPU outputs themselves.

Tolerances, relative to the largest entry of the reference (at least 1): fp64 1e-9; fp32 1e-3.  The forward-mode
reference differentiates accel, whose own rounding leaves its differences good to about 1e-9, so fp64 is compared to
1e-8 there.  The forward-mode results carry the
condition number kappa of M through M^-1 (the kernel's solve and the reference's differences of accel), so for them both
are widened by max(1, kappa / 100).  An MDH arm whose first joint is prismatic and whose M is singular (one such joint
without armature inertia) has no accel, and its forward derivatives are not compared."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import rne_derivs_ref as R  # noqa: E402
from oracle import chains as ch  # noqa: E402

TOL = {np.float64: 1e-9, np.float32: 1e-3}
G_CUSTOM = np.array([1.5, -2.0, -9.81])  # a robot gravity; the kernel receives minus it
FEXT = np.array([3.0, -1.0, 2.0, 0.4, -0.3, 0.2])
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst error / tolerance per (dtype, op):")
    for k in sorted(WORST, key=str):
        print(f"  {k[0]:8s} {k[1]:18s} {WORST[k]:.3g}")


def kappa(M):
    return np.linalg.cond(M, p=np.inf)


def check(key, got, want, dt, widen=None):
    got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    assert np.all(np.isfinite(got)), key
    scale = max(float(np.max(np.abs(want))), 1.0)  # an identically-zero block (a 1-joint arm) is compared absolutely
    tol = (TOL[dt] if widen is None or dt == np.float32 else 1e-8) * (np.maximum(1.0, widen / 100)[:, None, None] if widen is not None else 1.0)
    err = np.abs(got.astype(np.float64) - want) / scale
    ratio = float(np.max(err / tol))
    WORST[(np.dtype(dt).name, key[0])] = max(WORST.get((np.dtype(dt).name, key[0]), 0.0), ratio)
    assert ratio <= 1.0, (key, ratio)


def cuda(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()


def run_case(L, mdh, dt, gravity, fext, N=33, seed=0):
    rob = R.dhrobot(L, mdh)
    q, qd, qdd, tq = R.states(L, N, seed)
    if dt == np.float32:  # the reference sees the inputs the kernel sees
        q, qd, qdd, tq = (x.astype(np.float32).astype(np.float64) for x in (q, qd, qdd, tq))
    g = -(rob.gravity if gravity is None else gravity)
    dq, dqd = rob.rne_derivatives(cuda(q, dt), cuda(qd, dt), cuda(qdd, dt), gravity=gravity, fext=fext)
    rq, rqd = R.rne_derivatives(L, mdh, g, q, qd, qdd, fext)
    check(("rne_derivatives", "dq"), dq, rq, dt)
    check(("rne_derivatives", "dqd"), dqd, rqd, dt)
    M = R.inertia(L, mdh, q)
    if fext is None and np.all(np.linalg.matrix_rank(M) == M.shape[-1]):
        fq, fqd, ft = rob.accel_derivatives(cuda(q, dt), cuda(qd, dt), cuda(tq, dt), gravity=gravity)
        aq, aqd, at = R.accel_derivatives(L, mdh, g, q, qd, tq)
        k = kappa(M)
        check(("accel_derivatives", "dq"), fq, aq, dt, k)
        check(("accel_derivatives", "dqd"), fqd, aqd, dt, k)
        check(("accel_derivatives", "dtau"), ft, at, dt, k)


@pytest.mark.parametrize("pris", [False, True], ids=["rev", "pris"])
@pytest.mark.parametrize("mdh", [0, 1], ids=["dh", "mdh"])
@pytest.mark.parametrize("n", range(1, 11))
def test_every_joint_count_convention_and_joint_mix(n, mdh, pris):
    """Friction on / off x default / custom gravity x tip wrench on / off (rne_derivatives only) x fp64 / fp32."""
    tables = [R.robot(n, mdh, pris, fr, 1000 * n + 100 * mdh + 10 * pris + fr) for fr in (False, True)]
    if mdh and pris and n > 1:  # also prismatic joints behind a revolute first one
        tables += [R.revolute_first(L) for L in tables]
    for L in tables:
        for gravity in (None, G_CUSTOM):
            for fext in (None, FEXT):
                for dt in (np.float64, np.float32):
                    run_case(L, mdh, dt, gravity, fext, seed=n)


def _batch_robots():
    return [("puma560", ch.pack_rne(ch.puma560_links()), 0), ("panda_mdh", ch.pack_rne(ch.panda_mdh_links()), 1),
            ("mdh7_pris", R.robot(7, 1, True, True, 7), 1)]


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name,L,mdh", _batch_robots(), ids=[r[0] for r in _batch_robots()])
def test_tile_edges_through_the_c_abi(name, L, mdh, dt):
    """N around the 32-row tile: every row written, nothing past the last one (a NaN-filled guard row behind it)."""
    lib = rtb._lib.lib()
    h = rtb._lib.vp()
    Lc = np.ascontiguousarray(L, dtype=np.float64)
    n = len(Lc) // 24
    rtb._lib.check(lib.b2k_rne_create(n, mdh, rtb._lib.dptr(Lc), C.byref(h)))
    g = np.array([0.0, 0.0, 9.81])
    try:
        for N in (1, 31, 32, 33, 4097):
            q, qd, qdd, tq = R.states(Lc, N, N)
            q, qd, qdd, tq = (x.astype(dt).astype(np.float64) for x in (q, qd, qdd, tq))
            outs = [torch.full((N + 1, n, n), float("nan"), dtype=torch.float64 if dt == np.float64 else torch.float32,
                               device="cuda") for _ in range(3)]
            ins = [cuda(x, dt) for x in (q, qd, qdd, tq)]
            code = 1 if dt == np.float64 else 0
            rtb._lib.check(lib.b2k_rne_derivatives(h, code, ins[0].data_ptr(), ins[1].data_ptr(), ins[2].data_ptr(), N,
                                                   rtb._lib.dptr(g), None, outs[0].data_ptr(), outs[1].data_ptr(), None))
            rq, rqd = R.rne_derivatives(Lc, mdh, g, q, qd, qdd)
            check(("rne_derivatives", name, N), outs[0][:N], rq, dt)
            check(("rne_derivatives", name, N), outs[1][:N], rqd, dt)
            for o in outs[:2]:
                assert torch.isnan(o[N]).all()
            outs = [o.fill_(float("nan")) for o in outs]
            rtb._lib.check(lib.b2k_rne_accel_derivatives(h, code, ins[0].data_ptr(), ins[1].data_ptr(), ins[3].data_ptr(), N,
                                                         rtb._lib.dptr(g), *[o.data_ptr() for o in outs], None))
            want = R.accel_derivatives(Lc, mdh, g, q, qd, tq)
            k = kappa(R.inertia(Lc, mdh, q))
            for o, w in zip(outs, want):
                check(("accel_derivatives", name, N), o[:N], w, dt, k)
                assert torch.isnan(o[N]).all()
    finally:
        lib.b2k_rne_destroy(h)


def test_numpy_tensor_and_single_state_shapes():
    puma = rtb.models.Puma560()
    L = puma._pack_rne()
    q, qd, qdd, tq = R.states(L, 5, 11)
    dq, dqd = puma.rne_derivatives(q, qd, qdd)
    assert isinstance(dq, np.ndarray) and dq.shape == (5, 6, 6) and dqd.shape == (5, 6, 6)
    d1 = puma.rne_derivatives(q[2], qd[2], qdd[2])
    assert isinstance(d1[0], np.ndarray) and d1[0].shape == (6, 6)
    np.testing.assert_array_equal(d1[0], dq[2])
    np.testing.assert_array_equal(d1[1], dqd[2])
    t = puma.rne_derivatives(cuda(q[2], np.float64), cuda(qd[2], np.float64), cuda(qdd[2], np.float64))
    assert torch.is_tensor(t[0]) and t[0].is_cuda and tuple(t[0].shape) == (6, 6)
    np.testing.assert_array_equal(t[0].cpu().numpy(), dq[2])
    f = puma.accel_derivatives(q, qd, tq)
    assert len(f) == 3 and all(isinstance(x, np.ndarray) and x.shape == (5, 6, 6) for x in f)
    f1 = puma.accel_derivatives(cuda(q[0], np.float64), cuda(qd[0], np.float64), cuda(tq[0], np.float64))
    assert all(torch.is_tensor(x) and x.is_cuda and tuple(x.shape) == (6, 6) for x in f1)
    for a, b in zip(f1, f):
        np.testing.assert_array_equal(a.cpu().numpy(), b[0])
    f32 = puma.rne_derivatives(q, qd, qdd, dtype=np.float32)
    assert f32[0].dtype == np.float32
    with pytest.raises(ValueError):
        puma.rne_derivatives(q[:, :5], qd[:, :5], qdd[:, :5])
    with pytest.raises(ValueError):
        puma.accel_derivatives(q, qd[:4], tq)


def test_identities_hold_on_the_gpu_outputs():
    """Quadratic velocity terms, a symmetric gravity-load derivative, and the forward / inverse relations, on the
    kernels' own outputs (fp64), for DH and MDH arms with friction."""
    for name, L, mdh in [("puma", ch.pack_rne(ch.puma560_links()), 0), ("panda_mdh", ch.pack_rne(ch.panda_mdh_links()), 1),
                         ("dh8_pris", R.robot(8, 0, True, True, 81), 0), ("mdh6_rev", R.robot(6, 1, False, True, 61), 1)]:
        rob = R.dhrobot(L, mdh)
        n = rob.n
        q, qd, qdd, tq = R.states(L, 64, 5)
        _, dqd = rob.rne_derivatives(q, qd, qdd, gravity=G_CUSTOM)
        lhs = np.einsum("rik,rk->ri", dqd, qd)
        rhs = 2 * (R.rne(L, mdh, np.zeros(3), q, qd, np.zeros_like(q)) + R.friction(L, qd)) + R.viscous(L) * qd
        assert np.max(np.abs(lhs - rhs)) <= 1e-10 * np.max(np.abs(rhs)), name
        z = np.zeros_like(q)
        dq0, _ = rob.rne_derivatives(q, z, z)
        assert np.max(np.abs(dq0 - np.swapaxes(dq0, 1, 2))) <= 1e-10 * np.max(np.abs(dq0)), name
        fq, fqd, ft = rob.accel_derivatives(q, qd, tq, gravity=G_CUSTOM)
        M = rob.inertia(q)
        k = max(1.0, float(np.max(kappa(M))) / 100)
        assert np.max(np.abs(ft @ M - np.eye(n))) <= 1e-10 * k, name
        iq, iqd = rob.rne_derivatives(q, qd, rob.accel(q, qd, tq, gravity=G_CUSTOM), gravity=G_CUSTOM)
        Minv = np.linalg.inv(M)
        assert np.max(np.abs(fq + Minv @ iq)) <= 1e-9 * k * np.max(np.abs(fq)), name
        assert np.max(np.abs(fqd + Minv @ iqd)) <= 1e-9 * k * np.max(np.abs(fqd)), name


def test_coulomb_friction_adds_nothing_even_at_zero_rate():
    """Rates with exact 0 and -0.0: the derivatives equal those of the robot without Coulomb friction, bit for bit."""
    L = R.robot(6, 0, True, True, 17)
    rob, nc = R.dhrobot(L, 0), R.dhrobot(L, 0).nofriction(coulomb=True, viscous=False)
    q, qd, qdd, tq = R.states(L, 64, 9)
    qd[::3, 1] = 0.0
    qd[1::3, 4] = -0.0
    for a, b in zip(rob.rne_derivatives(q, qd, qdd), nc.rne_derivatives(q, qd, qdd)):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_same_results_with_and_without_the_specialised_path(monkeypatch, dt):
    """The robot-specialised path declines both ops: B2K_RNE_SPEC=0 and the default setting run the same kernel."""
    puma = rtb.models.Puma560()
    q, qd, qdd, tq = (cuda(x, dt) for x in R.states(puma._pack_rne(), 257, 3))
    res = {}
    for setting in ("0", None):
        if setting is None:
            monkeypatch.delenv("B2K_RNE_SPEC", raising=False)
        else:
            monkeypatch.setenv("B2K_RNE_SPEC", setting)
        res[setting] = puma.rne_derivatives(q, qd, qdd) + puma.accel_derivatives(q, qd, tq)
        assert puma.rne_kernel_info(op="rne_derivatives").startswith("generic k_rne_deriv<")
    for a, b in zip(res["0"], res[None]):
        assert torch.equal(a, b)
