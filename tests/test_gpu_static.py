"""DHRobot.gravjac / pay / paycap / friction / payload and Robot.pay on the GPU, against the float64 restatement of
tests/static_ref.py: Puma560, UR10, the MDH Panda with its tool, random DH / MDH tables with n = 1..10 (some with
prismatic joints), a rotated and shifted base; row counts 1, 31, 32, 33, 1017 and 100k; fp64 and fp32; numpy and CUDA
tensors, one wrench and one per row, J given; guard elements around every output; cross-checks against gravload (both
RNE kernels) and jacob0; the payload capacity of 100k Puma poses."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import rne_wrench_ref as wref  # noqa: E402
import static_ref as ref  # noqa: E402
from oracle import chains as ch  # noqa: E402
from oracle import oracle as orc  # noqa: E402

ROBOTS = wref.robots()
ROWS = (1, 31, 32, 33, 1017, 100_000)
BASE = ch.trotz(0.4) @ ch.troty(-0.9) @ ch.transl(0.1, -0.2, 0.3)
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def host(t):
    return t.cpu().numpy()


def setup(name, n, mdh, L):
    """(robot, links, base, tool): every other robot gets a base; the MDH Panda its tool."""
    base = BASE if sum(map(ord, name)) % 2 else None
    tool = ch.panda_mdh_tool() if name == "panda_mdh" else None
    Lk = np.asarray(L, dtype=np.float64).reshape(n, 24)
    links = [rtb.DHLink(alpha=l[0], a=l[1], theta=l[2], d=l[3], sigma=int(l[4]), mdh=bool(mdh), offset=l[5], m=l[6], r=l[7:10],
                        I=l[10:19].reshape(3, 3), Jm=l[19], G=l[20], B=l[21], Tc=l[22:24]) for l in Lk]
    return rtb.DHRobot(links, base=base, tool=tool), ref.links_of(n, L), base, tool


def close(got, want, rel):
    """agreement relative to each row's largest magnitude"""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    scale = np.maximum(1.0, np.abs(want).reshape(want.shape[0], -1).max(axis=1))
    err = np.abs(got - want).reshape(want.shape[0], -1).max(axis=1)
    assert (err <= rel * scale).all(), (err / scale).max()


def sample(N):
    """rows checked against the (slow, per-row) restatement"""
    return np.arange(N) if N <= 64 else np.sort(np.random.default_rng(N).choice(N, 300, replace=False))


def f32(a):
    """values that fp32 holds exactly, so one fp64 reference serves both dtypes"""
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def check_paycap(wm, jt, want_wm, want_jt, tauP, rel):
    """wmax where tau_P is not within rounding of zero (there the quotient is ill-conditioned), NaN rows exactly, and the
    limiting joint where the smallest capacity is not tied with the next to rounding."""
    scale = np.maximum(1.0, np.abs(tauP).max(axis=1, keepdims=True))
    good = np.abs(tauP) > 1e3 * rel * scale
    nan = np.isnan(want_wm).all(axis=1)
    assert (np.isnan(wm).all(axis=1) == nan).all() and (jt[nan] == -1).all()
    g = good & ~nan[:, None]
    np.testing.assert_allclose(wm[g], want_wm[g], rtol=min(1e3 * rel, 1e-2), atol=0)
    srt = np.sort(np.where(good, want_wm, np.inf), axis=1)
    with np.errstate(invalid="ignore"):  # inf - inf where two joints are unloaded
        gap = srt[:, 1] - srt[:, 0] if srt.shape[1] > 1 else np.full(srt.shape[0], np.inf)
    clear = good.all(axis=1) & ~nan & (gap > 1e3 * rel * np.abs(srt[:, 0]))
    np.testing.assert_array_equal(jt[clear], want_jt[clear])


@pytest.mark.parametrize("name,n,mdh,L,physical", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_gravjac_pay_paycap_friction_sweep(name, n, mdh, L, physical):
    rng = np.random.default_rng(sum(map(ord, name)))
    rob, links, base, tool = setup(name, n, mdh, L)
    g = rob.gravity
    tauR = np.stack([rng.uniform(5, 50, n), -rng.uniform(5, 50, n)], axis=1)
    for N in ROWS:
        if N == 100_000 and name not in ("puma560", "panda_mdh", "rand_n10_dh", "prismatic1_n5_mdh"):
            continue
        q = f32(rng.uniform(-3, 3, (N, n)))
        W1, WN = f32(rng.normal(size=6)), f32(rng.normal(size=(N, 6)))
        WN[-1] = 0.0
        qd = f32(rng.normal(size=(N, n)))
        qd[0] = 0.0
        s = sample(N)
        want_t, want_J = ref.gravjac(links, mdh, q[s], g, base, tool)
        want_p1 = {f: ref.pay(links, mdh, W1, q[s], f, base, tool) for f in (0, 1)}
        want_pN = {f: ref.pay(links, mdh, WN[s], q[s], f, base, tool) for f in (0, 1)}
        want_cap = {f: ref.paycap(links, mdh, WN[s], tauR, f, q[s], g, base, tool) for f in (0, 1)}
        nrm = np.linalg.norm(WN[s], axis=1, keepdims=True)
        want_tP = {f: want_pN[f] / np.where(nrm == 0, 1, nrm) for f in (0, 1)}
        want_fr = ref.friction(links, qd[s])
        for dt, rel in ((np.float64, 1e-12), (np.float32, 1e-4)):
            qin = dev(q, dt)

            def rows(x, *tail):  # one row (N = 1) comes back unbatched, as for jacob0
                return np.asarray(host(x) if torch.is_tensor(x) else x).reshape((N,) + tail)

            tau, J0 = rob.gravjac(qin)
            assert tau.dtype == qin.dtype and tuple(J0.shape) == ((N, 6, n) if N > 1 else (6, n))
            close(rows(tau, n)[s], want_t, rel)
            close(rows(J0, 6, n)[s], want_J, rel)
            Jj = rob.jacob0(qin)
            eps = np.finfo(dt).eps
            np.testing.assert_allclose(host(J0), host(Jj), rtol=32 * eps, atol=32 * eps * max(1.0, float(np.abs(host(Jj)).max())))
            for frame in (0, 1):
                close(rows(rob.pay(W1, qin, frame=frame), n)[s], want_p1[frame], rel)  # one wrench for every row
                close(rows(rob.pay(dev(WN, dt), qin, frame=frame), n)[s], want_pN[frame], rel)  # one per row
                Jf = rob.jacobe(qin) if frame == 1 else Jj
                close(rows(rob.pay(W1, J=Jf), n)[s], want_p1[frame], rel)  # J given
                wm, jt = rob.paycap(dev(WN, dt), tauR, frame=frame, q=qin)
                jt = rows(jt)
                check_paycap(rows(wm, n)[s].astype(np.float64), jt[s], *want_cap[frame], want_tP[frame], rel)
                assert jt[-1] == -1
            close(rows(rob.friction(dev(qd, dt)), n)[s], want_fr, rel)
        if N == 33:  # numpy in, numpy out; one row gives unbatched shapes
            tau, J0 = rob.gravjac(q)
            assert isinstance(tau, np.ndarray) and isinstance(J0, np.ndarray)
            close(tau, want_t, 1e-12)
            t1, J1 = rob.gravjac(q[3])
            assert t1.shape == (n,) and J1.shape == (6, n)
            p1 = rob.pay(W1, q[3], frame=0)
            assert isinstance(p1, np.ndarray) and p1.shape == (n,)
            close(p1[None], want_p1[0][3:4], 1e-12)
            wm1, j1 = rob.paycap(W1, tauR, q=q[3])
            assert wm1.shape == (n,) and isinstance(j1, int)
            assert rob.friction(np.zeros(n)).shape == (n,)
            assert isinstance(rob.pay(WN, q, frame=1), np.ndarray)


@pytest.fixture(params=["2", "0"], ids=["specialised", "generic"])
def spec(request, monkeypatch):
    monkeypatch.setenv("B2K_RNE_SPEC", request.param)
    return request.param


@pytest.mark.parametrize("name,n,mdh,L,physical", [r for r in ROBOTS if r[4]], ids=[r[0] for r in ROBOTS if r[4]])
def test_gravjac_tau_is_gravload(spec, name, n, mdh, L, physical):
    rng = np.random.default_rng(sum(map(ord, name)) + 7)
    rob, _, _, _ = setup(name, n, mdh, L)
    for N in (1, 33, 1017):
        q = dev(rng.uniform(-3, 3, (N, n)))
        for gv in (None, np.array([0.4, -2.0, -9.0])):
            tau, _ = rob.gravjac(q, gravity=gv)
            want = host(rob.gravload(q, gravity=gv))
            close(host(tau), want, 1e-12)


def test_puma_qn_reproduces_the_reference_literal(spec):
    kat = json.load(open(os.path.join(GOLDEN, "reference_kats.json")))["puma560_rne"]
    want = next(c["tau"] for c in kat["cases"] if c["qd"] == 0 and c["qdd"] == 0 and "gravity" not in c and "fext" not in c)
    puma = rtb.models.Puma560()
    tau, J0 = puma.gravjac(puma.qn)
    np.testing.assert_array_almost_equal(tau, want, decimal=kat["decimal"])
    np.testing.assert_allclose(J0, puma.jacob0(puma.qn), rtol=1e-14, atol=1e-14)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_no_stray_writes(dt):
    """Through the C entry points, every output sits between guard elements."""
    panda = setup("panda_mdh", 7, 1, ch.pack_rne(ch.panda_mdh_links(), mdh=True))[0]
    L, code = rtb._lib.lib(), (rtb._lib.F64 if dt == np.float64 else rtb._lib.F32)
    tdt = torch.float64 if dt == np.float64 else torch.float32
    rng = np.random.default_rng(9)
    chain, mass = panda.ets()._chain, panda._static_mass_table()
    g = np.ascontiguousarray(panda.gravity)
    tauR = np.ascontiguousarray(np.tile([[40.0, -30.0]], (7, 1)))
    params = np.ascontiguousarray([[l.B, l.G, l.Tc[0], l.Tc[1]] for l in panda.links], dtype=np.float64)
    dp, G = rtb._lib.dptr, 8
    st = torch.cuda.current_stream().cuda_stream

    def guarded(count, kind=tdt):
        fill = float("nan") if kind != torch.int32 else -7
        buf = torch.full((count + 2 * G,), fill, dtype=kind, device="cuda")
        return buf, buf[G:G + count]

    def intact(buf, inner):
        if buf.dtype == torch.int32:
            assert (buf[:G] == -7).all() and (buf[-G:] == -7).all() and not (inner == -7).any()
        else:
            assert torch.isnan(buf[:G]).all() and torch.isnan(buf[-G:]).all() and not torch.isnan(inner).any()

    for N in (1, 31, 32, 33, 1017):
        q = dev(rng.uniform(-2, 2, (N, 7)), dt)
        W = dev(rng.normal(size=(N, 6)) + 0.1, dt)
        tb, tau = guarded(N * 7)
        jb, J = guarded(N * 42)
        rtb._lib.check(L.b2k_gravjac(chain, code, q.data_ptr(), N, 7, dp(mass), dp(g), tau.data_ptr(), J.data_ptr(), st))
        torch.cuda.synchronize()
        intact(tb, tau)
        intact(jb, J)
        t_ref, J_ref = panda.gravjac(q)
        assert torch.equal(tau.view(N, 7), t_ref.reshape(N, 7)) and torch.equal(J.view(N, 6, 7), J_ref.reshape(N, 6, 7))
        for frame in (0, 1):
            pb, p = guarded(N * 7)
            rtb._lib.check(L.b2k_pay(chain, code, q.data_ptr(), N, 7, W.data_ptr(), 6, frame, p.data_ptr(), st))
            torch.cuda.synchronize()
            intact(pb, p)
            wb, wm = guarded(N * 7)
            ib, jt = guarded(N, torch.int32)
            rtb._lib.check(L.b2k_paycap(chain, code, q.data_ptr(), N, 7, dp(mass), dp(g), W.data_ptr(), 6, frame, dp(tauR),
                                        wm.data_ptr(), jt.data_ptr(), st))
            torch.cuda.synchronize()
            intact(wb, wm)
            intact(ib, jt)
        Jb, Jd = guarded(N * 42)
        Jd.copy_(J)
        pb, p = guarded(N * 7)
        rtb._lib.check(L.b2k_pay_jacobian(code, 7, Jd.data_ptr(), W.data_ptr(), 6, N, p.data_ptr(), st))
        fb, f = guarded(N * 7)
        rtb._lib.check(L.b2k_friction(code, 7, dp(params), q.data_ptr(), N, f.data_ptr(), st))
        torch.cuda.synchronize()
        intact(pb, p)
        intact(fb, f)


def test_paycap_at_100k_puma_poses():
    puma = rtb.models.Puma560()
    rng = np.random.default_rng(21)
    N, n = 100_000, 6
    q = dev(rng.uniform(-np.pi, np.pi, (N, n)))
    tauR = np.array([[97.6, -97.6], [186.4, -186.4], [89.4, -89.4], [24.2, -24.2], [20.1, -20.1], [21.3, -21.3]])
    for frame, w in ((0, [0, 0, -1, 0, 0, 0]), (1, [0.3, -0.2, 0.9, 0.05, 0.0, -0.1])):
        wmax, joint = puma.paycap(w, tauR, frame=frame, q=q)
        wmax, joint = host(wmax), host(joint)
        tauB = host(puma.gravjac(q)[0])
        what = np.asarray(w, dtype=np.float64) / np.linalg.norm(w)
        tauP = host(puma.pay(what, q, frame=frame))
        assert (joint >= 0).all()
        rows = np.arange(N)
        s = wmax[rows, joint]
        np.testing.assert_array_equal(np.isinf(wmax), tauP == 0)
        fin = np.isfinite(s)
        t = tauB + s[:, None] * tauP
        lim = np.where(tauP[rows, joint] > 0, tauR[joint, 0], tauR[joint, 1])
        np.testing.assert_allclose(t[rows, joint][fin], lim[fin], rtol=1e-9, atol=1e-9)
        ok = fin & (tauB <= tauR[:, 0]).all(axis=1) & (tauB >= tauR[:, 1]).all(axis=1) & (s >= 0)
        assert ok.sum() > N // 10
        assert (t[ok] <= tauR[:, 0] * (1 + 1e-9) + 1e-9).all() and (t[ok] >= tauR[:, 1] * (1 + 1e-9) - 1e-9).all()
    # joints that a pure world-z force cannot load give +inf: joint 1 of the Puma turns about world z
    wmax, _ = puma.paycap([0, 0, -1, 0, 0, 0], tauR, frame=0, q=q[:100])
    assert np.isinf(host(wmax)[:, 0]).all()


def test_payload_reaches_every_kernel(monkeypatch):
    puma = rtb.models.Puma560()
    rng = np.random.default_rng(4)
    q = rng.uniform(-2, 2, (1017, 6))
    qt = dev(q)
    monkeypatch.setenv("B2K_RNE_SPEC", "2")
    puma.gravload(qt)  # build the specialised kernel for the old mass first
    puma.gravjac(qt)
    puma.payload(2.5, [0, 0, 0.1])
    Lm = puma._pack_rne()
    assert Lm[24 * 5 + 6] == 2.5 and np.array_equal(Lm[24 * 5 + 7:24 * 5 + 10], [0, 0, 0.1])
    want = orc.dyn_gravload(lambda a, b, c, g: orc.rne(6, 0, Lm, g, a, b, c), 6, q, -puma.gravity)
    for sp in ("2", "0"):
        monkeypatch.setenv("B2K_RNE_SPEC", sp)
        close(host(puma.gravload(qt)), want, 1e-12)
        assert puma.rne_kernel_info(op="gravload").startswith("k_rne_spec<" if sp == "2" else "generic")
    close(host(puma.gravjac(qt)[0]), want, 1e-12)
    puma.payload(0)
    assert puma.links[5].m == 0
    want0 = orc.dyn_gravload(lambda a, b, c, g: orc.rne(6, 0, puma._pack_rne(), g, a, b, c), 6, q, -puma.gravity)
    close(host(puma.gravjac(qt)[0]), want0, 1e-12)
    for sp in ("2", "0"):
        monkeypatch.setenv("B2K_RNE_SPEC", sp)
        close(host(puma.gravload(qt)), want0, 1e-12)


def test_robot_pay_on_ets_panda_and_urdf_tree():
    rng = np.random.default_rng(8)
    panda = rtb.models.Panda()
    q = dev(rng.uniform(-2, 2, (1017, 7)))
    W = rng.normal(size=6)
    for frame, jac in ((0, panda.jacob0), (1, panda.jacobe)):
        want = -np.einsum("nkj,k->nj", host(jac(q)), W)
        close(host(panda.pay(W, q, frame=frame)), want, 1e-12)
    tree = rtb.Robot.URDF(os.path.join(GOLDEN, "urdf", "two_arm.urdf"))
    qt = dev(rng.uniform(-1, 1, (1017, tree.n)))
    for end in ("r_skew", "l_flange"):
        WN = rng.normal(size=(1017, 6))
        for frame, jac in ((0, tree.jacob0), (1, tree.jacobe)):
            J = host(jac(qt, end=end))
            want = -np.einsum("nkj,nk->nj", J, WN)
            close(host(tree.pay(dev(WN), qt, frame=frame, end=end)), want, 1e-12)
            close(tree.pay(WN, J=J), want, 1e-12)  # numpy in, numpy out
