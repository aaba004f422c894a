"""GPU tests of the operational-space dynamics (reference DynamicsMixin.inertia_x / coriolis_x / gravload_x / accel_x):
the device pipeline against the oracle's per-row numpy restatement, the operational-space equation of motion on device
outputs, precomputed operands, singular rows and placement."""
import os
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import oracle as orc  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import opspace_ref as ops  # noqa: E402

URDF = os.path.join(os.path.dirname(__file__), "golden", "urdf", "macro_arm.urdf.xacro")
REPS = ("rpy/xyz", "rpy/zyx", "eul", "exp")


def dev(a, dt=np.float64, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)


def host(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def close(got, want, rtol):
    """|got - want| <= rtol * (largest |entry| of the row's want), row by row"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    g, w = got.reshape(len(got), -1), want.reshape(len(want), -1)
    scale = np.maximum(np.abs(w).max(1, keepdims=True), 1e-300)
    err = (np.abs(g - w) / scale).max()
    assert err <= rtol, f"max row-relative error {err:.3g} > {rtol}"


class Case:
    def __init__(self, name, friction_free=False):
        self.name = name
        if name == "tree":
            rob = rtb.Robot.URDF(URDF)
            tree = rob.tree_description()
            self.rne = self.rne_nf = lambda a, b, c, g: orc.tree_rne(tree, np.atleast_2d(a), np.atleast_2d(b), np.atleast_2d(c), g)
        else:
            rob = {"puma": rtb.models.Puma560, "ur10": rtb.models.UR10, "panda_mdh": rtb.models.PandaMDH}[name]()
            if friction_free:
                rob = rob.nofriction(coulomb=True, viscous=True)
            n, mdh, L = rob.n, rob.mdh, rob._pack_rne()
            Lnf = orc.nofriction_L(L)
            self.rne = lambda q, qd, qdd, g: orc.rne(n, mdh, L, -np.asarray(g, dtype=float), q, qd, qdd)
            self.rne_nf = lambda q, qd, qdd, g: orc.rne(n, mdh, Lnf, -np.asarray(g, dtype=float), q, qd, qdd)
        self.rob, self.n = rob, rob.n
        self.chain = orc.Chain(rob.ets().describe())
        self.g = np.asarray(rob.gravity, dtype=float)


def sample_rows(N, rng, k=40):
    idx = {0, 30, 31, 32, N - 1} | set(rng.choice(N, min(N, k), replace=False).tolist())
    return np.array(sorted(i for i in idx if 0 <= i < N))


CASES = [("puma", False), ("puma", True), ("ur10", False), ("ur10", True), ("panda_mdh", True), ("tree", True)]


@pytest.mark.parametrize("N", [1, 31, 33, 1000, 100001])
@pytest.mark.parametrize("name,pinv", CASES)
def test_parity_with_the_oracle_fp64(name, pinv, N):
    c = Case(name)
    rob, n = c.rob, c.n
    rng = np.random.default_rng(zlib.crc32(f"{name}{pinv}{N}".encode()))
    q = rng.uniform(-2.5, 2.5, (N, n))
    qd, xd, w = rng.normal(size=(N, n)), rng.normal(size=(N, 6)), rng.normal(size=(N, 6)) * 5
    qt, qdt, xdt, wt = dev(q), dev(qd), dev(xd), dev(w)
    rows = sample_rows(N, rng)
    rows = rows[np.linalg.cond(ops.ja(c.chain, q[rows])) < 1e4]
    assert len(rows) >= min(N, 10) // 2
    qs = q[rows]
    for rep in REPS:
        Mx = host(rob.inertia_x(qt, pinv=pinv, representation=rep))
        assert Mx.shape == (N, 6, 6)
        close(Mx[rows], ops.inertia_x(c.rne, c.chain, n, qs, pinv, rep), 1e-8)
    Gx = host(rob.gravload_x(qt, pinv=pinv))
    close(Gx[rows], ops.gravload_x(c.rne, c.chain, n, qs, c.g, pinv), 1e-8)
    Cx = host(rob.coriolis_x(qt, qdt, pinv=pinv))
    close(Cx[rows], ops.coriolis_x(c.rne, c.rne_nf, c.chain, n, qs, qd[rows], pinv), 1e-7)
    xdd = host(rob.accel_x(qt, xdt, wt, pinv=pinv))
    assert xdd.shape == (N, 6)
    close(xdd[rows], ops.accel_x(c.rne, c.chain, n, qs, xd[rows], w[rows], c.g, pinv), 1e-7)


@pytest.mark.parametrize("N", [33, 1000])
@pytest.mark.parametrize("name,pinv", CASES)
def test_parity_with_the_oracle_fp32(name, pinv, N):
    c = Case(name)
    rob, n = c.rob, c.n
    rng = np.random.default_rng(zlib.crc32(f"{name}{pinv}{N}f32".encode()))
    r32 = lambda a: a.astype(np.float32).astype(np.float64)  # noqa: E731
    q, qd = r32(rng.uniform(-2.5, 2.5, (N, n))), r32(rng.normal(size=(N, n)))
    xd, w = r32(rng.normal(size=(N, 6)) * 0.2), r32(rng.normal(size=(N, 6)) * 5)
    rows = sample_rows(N, rng)
    rows = rows[np.linalg.cond(ops.ja(c.chain, q[rows])) < 1e3]
    qs = q[rows]
    f = np.float32
    # the fp32 Jacobi sweeps stop at 1e-6 relative orthogonality (the rule of k_singular_all), so a pseudo-inverse row
    # carries ~1e-6 cond(Ja) of its own on top of fp32 rounding
    tol = 5e-3 if pinv else 2e-3
    Mx = rob.inertia_x(dev(q, f), pinv=pinv)
    assert Mx.dtype == torch.float32
    close(host(Mx)[rows], ops.inertia_x(c.rne, c.chain, n, qs, pinv), tol)
    close(host(rob.gravload_x(dev(q, f), pinv=pinv))[rows], ops.gravload_x(c.rne, c.chain, n, qs, c.g, pinv), tol)
    close(host(rob.coriolis_x(dev(q, f), dev(qd, f), pinv=pinv))[rows],
          ops.coriolis_x(c.rne, c.rne_nf, c.chain, n, qs, qd[rows], pinv, h=1e-3), tol)
    close(host(rob.accel_x(dev(q, f), dev(xd, f), dev(w, f), pinv=pinv))[rows],
          ops.accel_x(c.rne, c.chain, n, qs, xd[rows], w[rows], c.g, pinv, h=1e-3), tol)
    # dtype= on fp64 input selects the fp32 kernels too
    assert rob.inertia_x(q[:3], pinv=pinv, dtype=np.float32).dtype == np.float32


def _opspace_qd(rob, Ja, xd):
    """qd = Ji xd through the C ABI (the first stage accel_x runs)"""
    N = Ja.shape[0]
    qd = torch.empty((N, rob.n), dtype=Ja.dtype, device=Ja.device)
    rtb._lib.check(rtb._lib.lib().b2k_opspace(rtb._lib.F64, rob.n, rtb._lib.OPS_INV, Ja.data_ptr(), None, None, None, None, None,
                                              None, xd.data_ptr(), None, N, None, None, None, None, qd.data_ptr(), None,
                                              torch.cuda.current_stream().cuda_stream))
    return qd


@pytest.mark.parametrize("name", ["puma", "ur10"])
def test_equation_of_motion_on_device_outputs(name):
    """Mx accel_x(q, xd, w) + Cx(q, Ji xd) xd + Gx = w at 100k rows of a friction-free arm"""
    rob = Case(name, friction_free=True).rob
    N = 100_000
    rng = np.random.default_rng({"puma": 11, "ur10": 12}[name])
    qt, xdt, wt = dev(rng.uniform(-2.5, 2.5, (N, 6))), dev(rng.normal(size=(N, 6))), dev(rng.normal(size=(N, 6)) * 10)
    Ja = rob.jacob0_analytical(qt)
    qd = _opspace_qd(rob, Ja, xdt)
    Mx, Cx, Gx = host(rob.inertia_x(qt)), host(rob.coriolis_x(qt, qd)), host(rob.gravload_x(qt))
    xdd = host(rob.accel_x(qt, xdt, wt))
    xd, w = host(xdt), host(wt)
    ok = np.linalg.cond(host(Ja)) < 1e3
    assert ok.sum() > N // 4
    Mxdd = np.einsum("kab,kb->ka", Mx, xdd)
    lhs = Mxdd + np.einsum("kab,kb->ka", Cx, xd) + Gx
    scale = np.maximum.reduce([np.abs(w).max(1), np.abs(Gx).max(1), np.abs(Mxdd).max(1)])
    assert (np.abs(lhs - w).max(1) / scale)[ok].max() < 1e-6


def _launches(fn):
    torch.cuda.synchronize()
    n0 = rtb.launch_count()
    out = host(fn())
    return out, rtb.launch_count() - n0


def test_precomputed_operands_skip_their_producers():
    rob = rtb.models.Puma560()
    rng = np.random.default_rng(5)
    N = 200
    qt, qdt = dev(rng.uniform(-2, 2, (N, 6))), dev(rng.normal(size=(N, 6)))
    Ja, n_ja = _launches(lambda: rob.jacob0_analytical(qt))
    Jd, n_jd = _launches(lambda: rob.jacob0_dot(qt, qdt, representation="rpy/xyz"))
    Cm, n_c = _launches(lambda: rob.coriolis(qt, qdt))
    M, n_m = _launches(lambda: rob.inertia(qt))
    Ji = np.linalg.inv(Ja)
    Mx, n_mx = _launches(lambda: rob.inertia_x(qt))
    Mx_ji, n_mx_ji = _launches(lambda: rob.inertia_x(qt, Ji=Ji))
    close(Mx_ji, Mx, 1e-9)
    assert n_mx == n_ja + n_m + 1 and n_mx_ji == n_m + 1
    Gx, n_gx = _launches(lambda: rob.gravload_x(qt))
    Gx_ji, n_gx_ji = _launches(lambda: rob.gravload_x(qt, Ji=dev(Ji)))
    close(Gx_ji, Gx, 1e-9)
    assert n_gx_ji == n_gx - n_ja
    Cx, n_cx = _launches(lambda: rob.coriolis_x(qt, qdt))
    assert n_cx == n_ja + n_jd + n_c + n_m + 1
    for kw in (dict(Ji=Ji), dict(J=Ja), dict(Jd=Jd), dict(C=Cm), dict(Mx=Mx), dict(Ji=Ji, Jd=Jd, C=Cm, Mx=Mx),
               dict(J=dev(Ja), Jd=dev(Jd), C=dev(Cm), Mx=dev(Mx))):
        got, k = _launches(lambda: rob.coriolis_x(qt, qdt, **kw))
        close(got, Cx, 1e-9)
        skipped = ((n_ja if ("Ji" in kw or "J" in kw) else 0) + (n_jd if "Jd" in kw else 0) + (n_c if "C" in kw else 0)
                   + (n_m if "Mx" in kw else 0))
        assert k == n_cx - skipped, kw
    _, k_all = _launches(lambda: rob.coriolis_x(qt, qdt, Ji=Ji, Jd=Jd, C=Cm, Mx=Mx))
    assert k_all == 1  # nothing but the epilogue
    # single-row operands with a single configuration
    np.testing.assert_allclose(rob.inertia_x(host(qt)[3], Ji=Ji[3]), Mx[3], rtol=1e-9, atol=1e-9 * np.abs(Mx[3]).max())
    with pytest.raises(ValueError):
        rob.inertia_x(qt, Ji=Ji[:5])


def test_a_zero_pivot_gives_nan_on_exactly_that_row():
    rob = rtb.models.Puma560()
    rng = np.random.default_rng(6)
    N = 40
    qt = dev(rng.uniform(-2, 2, (N, 6)))
    Ja = rob.jacob0_analytical(qt).clone()
    Ja[17, :, 2] = 0
    M, G = rob.inertia(qt), rob.gravload(qt)
    L = rtb._lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    for kind in (rtb._lib.OPS_INV, rtb._lib.OPS_PINV):
        Ji, Mx, Gx = (torch.empty(s, dtype=torch.float64, device="cuda") for s in ((N, 6, 6), (N, 6, 6), (N, 6)))
        rtb._lib.check(L.b2k_opspace(rtb._lib.F64, 6, kind, Ja.data_ptr(), None, M.data_ptr(), None, None, G.data_ptr(), None, None,
                                     None, N, Ji.data_ptr(), Mx.data_ptr(), None, Gx.data_ptr(), None, None, st))
        Ji, Mx, Gx = host(Ji), host(Mx), host(Gx)
        others = np.arange(N) != 17
        for a in (Ji, Mx, Gx):
            assert np.isfinite(a[others]).all()
            if kind == rtb._lib.OPS_INV:
                assert np.isnan(a[17]).all()
        want = np.linalg.pinv(host(Ja)) if kind == rtb._lib.OPS_PINV else np.linalg.inv(host(Ja)[others])
        close(Ji if kind == rtb._lib.OPS_PINV else Ji[others], want, 1e-8)


def test_singular_and_shape_errors():
    panda = rtb.models.PandaMDH()
    with pytest.raises(np.linalg.LinAlgError):
        panda.inertia_x(panda.qr)
    assert panda.inertia_x(panda.qr, pinv=True).shape == (6, 6)
    puma = rtb.models.Puma560()
    with pytest.raises(ValueError):
        puma.coriolis_x(np.zeros((4, 6)), np.zeros((3, 6)))
    with pytest.raises(ValueError):
        puma.accel_x(np.zeros((4, 6)), np.zeros(5), np.zeros(6))


def test_placement_numpy_and_devices():
    rob = rtb.models.UR10()
    rng = np.random.default_rng(8)
    q, qd, xd, w = rng.uniform(-2, 2, (50, 6)), rng.normal(size=(50, 6)), rng.normal(size=(50, 6)), rng.normal(size=(50, 6))
    ref = [host(rob.inertia_x(dev(q), pinv=True)), host(rob.coriolis_x(dev(q), dev(qd), pinv=True)),
           host(rob.gravload_x(dev(q), pinv=True)), host(rob.accel_x(dev(q), dev(xd), dev(w), pinv=True))]
    got = [rob.inertia_x(q, pinv=True), rob.coriolis_x(q, qd, pinv=True), rob.gravload_x(q, pinv=True),
           rob.accel_x(q, xd, w, pinv=True)]
    for a, b in zip(got, ref):
        assert isinstance(a, np.ndarray)
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12)
    one = rob.accel_x(q[4], xd[4], w[4], pinv=True)
    assert one.shape == (6,)
    np.testing.assert_allclose(one, ref[3][4], rtol=1e-10, atol=1e-10)
    if torch.cuda.device_count() < 2:
        return
    d1 = "cuda:1"
    got1 = [rob.inertia_x(dev(q, device=d1), pinv=True), rob.coriolis_x(dev(q, device=d1), dev(qd, device=d1), pinv=True),
            rob.gravload_x(dev(q, device=d1), pinv=True), rob.accel_x(dev(q, device=d1), dev(xd, device=d1), dev(w, device=d1), pinv=True)]
    for a, b in zip(got1, ref):
        assert a.device == torch.device(d1)
        np.testing.assert_allclose(host(a), b, rtol=1e-12, atol=1e-12)
