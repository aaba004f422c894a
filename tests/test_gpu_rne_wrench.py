"""DHRobot.rne(..., base_wrench=True) on the GPU: the robot-specialised kernel (B2K_RNE_SPEC=2, which refuses to fall
back) and the generic k_rne_wrench (B2K_RNE_SPEC=0) against the float64 reference of tests/rne_wrench_ref.py, on
Puma560, UR10, the MDH Panda and random DH / MDH tables with n = 1..10 (some with prismatic joints); row counts that
split one call between full specialised tiles and the generic tail; every input form; guard elements around both
outputs; and the whole-robot momentum balance at 100k rows."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import rne_wrench_ref as ref  # noqa: E402
from oracle import chains as ch  # noqa: E402

ROBOTS = ref.robots()
ROWS = (1, 31, 32, 33, 1000 + 17)


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def host(t):
    return t.cpu().numpy()


def robot_of(n, mdh, L, base=None):
    """A DHRobot whose packed link table is exactly L."""
    Lk = np.asarray(L, dtype=np.float64).reshape(n, 24)
    links = [rtb.DHLink(alpha=l[0], a=l[1], theta=l[2], d=l[3], sigma=int(l[4]), mdh=bool(mdh), offset=l[5], m=l[6], r=l[7:10],
                        I=l[10:19].reshape(3, 3), Jm=l[19], G=l[20], B=l[21], Tc=l[22:24]) for l in Lk]
    rob = rtb.DHRobot(links, base=base)
    assert np.array_equal(rob._pack_rne(), np.asarray(L, dtype=np.float64))
    return rob


def max_ulp(a, b):
    """Largest distance in units in the last place between two arrays of one float dtype."""
    it = np.int64 if a.dtype == np.float64 else np.int32
    ia, ib = a.view(it).astype(np.int64), b.view(it).astype(np.int64)
    ia = np.where(ia < 0, np.iinfo(it).min - ia, ia)  # monotone integer order across zero
    ib = np.where(ib < 0, np.iinfo(it).min - ib, ib)
    return int(np.abs(ia - ib).max()) if a.size else 0


def tau_vs_plain(tw, tp, spec):
    """tau of the wrench call against the plain call: the largest ulp difference.  The generic kernels run the same row
    code, so it is 0.  The specialised source of the wrench mode is the plain one plus the wrench lines; NVRTC may then
    fuse a product that the wrench also reads into a different FMA, so there the two agree to rounding."""
    u = max_ulp(tw, tp)
    if spec == "0":
        assert u == 0, u
    else:
        eps = np.finfo(tw.dtype).eps
        np.testing.assert_allclose(tw, tp, rtol=64 * eps, atol=64 * eps * max(1.0, np.abs(tp).max()))
    return u


@pytest.fixture(params=["2", "0"], ids=["specialised", "generic"])
def spec(request, monkeypatch):
    monkeypatch.setenv("B2K_RNE_SPEC", request.param)
    return request.param


@pytest.mark.parametrize("name,n,mdh,L,physical", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_wrench_parity_with_the_reference(spec, name, n, mdh, L, physical):
    rng = np.random.default_rng(sum(map(ord, name)) + int(spec))
    rob = robot_of(n, mdh, L)
    g = rob.gravity
    ulps = {}
    for N in ROWS:
        q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
        qd[-1:] = 0.0
        args = [dev(x) for x in (q, qd, qdd)]
        tau, wb = rob.rne(*args, base_wrench=True)
        want_tau, want_wb = ref.rne_wrench(n, mdh, L, -g, q, qd, qdd)
        np.testing.assert_allclose(host(tau), want_tau, rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(host(wb), want_wb, rtol=1e-9, atol=1e-9 * max(1.0, np.abs(want_wb).max()))
        ulps[N] = tau_vs_plain(host(tau), host(rob.rne(*args)), spec)
        if N == 1017:  # gravity override and a tip wrench
            fx, gv = rng.normal(size=6), np.array([0.5, -1.0, 3.0])
            tau, wb = rob.rne(*args, gravity=gv, fext=fx, base_wrench=True)
            want_tau, want_wb = ref.rne_wrench(n, mdh, L, -gv, q, qd, qdd, fx)
            np.testing.assert_allclose(host(tau), want_tau, rtol=1e-9, atol=1e-9)
            np.testing.assert_allclose(host(wb), want_wb, rtol=1e-9, atol=1e-9 * max(1.0, np.abs(want_wb).max()))
            ulps["fext"] = tau_vs_plain(host(tau), host(rob.rne(*args, gravity=gv, fext=fx)), spec)
            # fp32 on the rounded inputs
            q32, qd32, qdd32 = (x.astype(np.float32) for x in (q, qd, qdd))
            tau32, wb32 = rob.rne(dev(q32, np.float32), dev(qd32, np.float32), dev(qdd32, np.float32), fext=fx, base_wrench=True)
            assert tau32.dtype == torch.float32 and wb32.dtype == torch.float32
            want_tau, want_wb = ref.rne_wrench(n, mdh, L, -g, *(x.astype(np.float64) for x in (q32, qd32, qdd32)), fx)
            np.testing.assert_allclose(host(tau32), want_tau, rtol=5e-4, atol=5e-4 * max(1.0, np.abs(want_tau).max()))
            np.testing.assert_allclose(host(wb32), want_wb, rtol=5e-4, atol=5e-4 * max(1.0, np.abs(want_wb).max()))
            ulps["fp32"] = tau_vs_plain(host(tau32), host(rob.rne(dev(q32, np.float32), dev(qd32, np.float32), dev(qdd32, np.float32), fext=fx)), spec)
    info = rob.rne_kernel_info(op="rne_wrench")
    assert info.startswith("k_rne_spec<" if spec == "2" else "generic"), info
    print(f"\n{name} B2K_RNE_SPEC={spec}: largest ulp difference of tau (wrench call vs plain call) {ulps}")


def test_input_forms_and_result_types(spec):
    puma = robot_of(6, 0, ch.pack_rne(ch.puma560_links()))
    L = puma._pack_rne()
    rng = np.random.default_rng(5)
    N = 5000
    q, qd, qdd = rng.uniform(-3, 3, (N, 6)), rng.normal(size=(N, 6)), rng.normal(size=(N, 6))
    want_tau, want_wb = ref.rne_wrench(6, 0, L, -puma.gravity, q, qd, qdd)
    tau, wb = puma.rne(q, qd, qdd, base_wrench=True)  # numpy: the pipelined host path
    assert isinstance(tau, np.ndarray) and isinstance(wb, np.ndarray) and wb.shape == (N, 6) and wb.dtype == np.float64
    np.testing.assert_allclose(tau, want_tau, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(wb, want_wb, rtol=1e-9, atol=1e-9 * np.abs(want_wb).max())
    np.testing.assert_array_equal(tau, puma.rne(q, qd, qdd))
    t1, w1 = puma.rne(dev(q[7]), dev(qd[7]), dev(qdd[7]), base_wrench=True)  # one state
    assert t1.shape == (6,) and w1.shape == (6,) and w1.is_cuda
    np.testing.assert_allclose(host(w1), want_wb[7], rtol=1e-9, atol=1e-9 * np.abs(want_wb).max())
    t1, w1 = puma.rne(q[7], qd[7], qdd[7], base_wrench=True)
    assert isinstance(w1, np.ndarray) and w1.shape == (6,)
    for empty in (np.zeros((0, 6)), dev(np.zeros((0, 6)))):
        t0, w0 = puma.rne(empty, empty, empty, base_wrench=True)
        assert tuple(t0.shape) == (0, 6) and tuple(w0.shape) == (0, 6)
    # fp32 numpy through the pipeline
    t32, w32 = puma.rne(*(x.astype(np.float32) for x in (q, qd, qdd)), base_wrench=True)
    assert w32.dtype == np.float32
    _, want32 = ref.rne_wrench(6, 0, L, -puma.gravity, *(x.astype(np.float32).astype(np.float64) for x in (q, qd, qdd)))
    np.testing.assert_allclose(w32, want32, rtol=5e-4, atol=5e-4 * np.abs(want32).max())
    # a rotated base: gravity goes into frame 0 as base^T g, and so does the wrench
    Rb = ch.trotz(0.7) @ ch.trotx(-1.1)
    rot = robot_of(6, 0, L, base=Rb)
    _, wbr = rot.rne(dev(q), dev(qd), dev(qdd), base_wrench=True)
    _, want_r = ref.rne_wrench(6, 0, L, -(Rb[:3, :3].T @ rot.gravity), q, qd, qdd)
    np.testing.assert_allclose(host(wbr), want_r, rtol=1e-9, atol=1e-9 * np.abs(want_r).max())


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_no_stray_writes_around_tau_and_wbase(spec, dt):
    """Through the C entry point, both outputs sit between guard elements; every full tile, ragged tail and the split
    between them writes its own rows and nothing else."""
    panda = robot_of(7, 1, ch.pack_rne(ch.panda_mdh_links(), mdh=True))
    lib, code = rtb._lib.lib(), (rtb._lib.F64 if dt == np.float64 else rtb._lib.F32)
    rng = np.random.default_rng(9)
    g = np.ascontiguousarray(-panda.gravity)
    tdt = torch.float64 if dt == np.float64 else torch.float32
    for N in (1, 32, 33, 1017):
        q, qd, qdd = (dev(rng.uniform(-2, 2, (N, 7)), dt) for _ in range(3))
        t_ref, w_ref = panda.rne(q, qd, qdd, base_wrench=True)  # (also builds the robot's handle)
        G = 12  # guard elements on each side (keeps 16-byte alignment for both dtypes)
        tb = torch.full((N * 7 + 2 * G,), float("nan"), dtype=tdt, device="cuda")
        wbuf = torch.full((N * 6 + 2 * G,), float("nan"), dtype=tdt, device="cuda")
        tau, wb = tb[G:G + N * 7], wbuf[G:G + N * 6]
        rtb._lib.check(lib.b2k_rne_wrench(panda._rne_ob, code, q.data_ptr(), qd.data_ptr(), qdd.data_ptr(), N, rtb._lib.dptr(g), None,
                                          tau.data_ptr(), wb.data_ptr(), None))
        torch.cuda.synchronize()
        for buf, inner in ((tb, tau), (wbuf, wb)):
            assert torch.isnan(buf[:G]).all() and torch.isnan(buf[-G:]).all(), N
            assert not torch.isnan(inner).any(), N
        assert torch.equal(tau.view(N, 7), t_ref) and torch.equal(wb.view(N, 6), w_ref)


def test_momentum_balance_at_100k_rows():
    """The wrench of 100k states equals dP/dt and dH_O0/dt of the whole robot plus gravity and the tip wrench, with a
    rotated base -- the physical statement, independent of any recursion."""
    rng = np.random.default_rng(12)
    N = 100_000
    for n, mdh, L in ((6, 0, ch.pack_rne(ch.puma560_links())), (7, 1, ch.pack_rne(ch.panda_mdh_links(), mdh=True))):
        Rb = ch.trotz(rng.uniform(-3, 3)) @ ch.troty(rng.uniform(-1, 1))
        rob = robot_of(n, mdh, L, base=Rb)
        q, qd, qdd = rng.uniform(-2, 2, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
        fx = rng.normal(size=6)
        _, wb = rob.rne(dev(q), dev(qd), dev(qdd), fext=fx, base_wrench=True)
        want = ref.momentum_balance(n, mdh, L, Rb[:3, :3].T @ rob.gravity, q, qd, qdd, fx)
        np.testing.assert_allclose(host(wb), want, rtol=0, atol=2e-6 * np.abs(want).max())
        z = np.zeros_like(q)
        _, w0 = rob.rne(dev(q), dev(z), dev(z), base_wrench=True)
        M = np.asarray(L).reshape(n, 24)[:, 6].sum()
        np.testing.assert_allclose(host(w0)[:, :3], np.broadcast_to(-M * (Rb[:3, :3].T @ rob.gravity), (N, 3)), rtol=1e-12, atol=1e-10)
