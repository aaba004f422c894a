"""DHRobot.rne_regressor / regressor_gram / identify on the GPU against the float64 regressor of tests/regressor_ref.py
(14 n oracle rne calls on unit link tables), and against rne itself through Y @ dynamic_parameters() == rne.

Tolerances are relative to the largest reference entry (at least 1): fp64 1e-9, fp32 1e-3."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import regressor_ref as RR  # noqa: E402
import rne_derivs_ref as R  # noqa: E402

TOL = {np.float64: 1e-9, np.float32: 1e-3}
G_CUSTOM = np.array([1.5, -2.0, -9.81])  # a robot gravity; the kernel receives minus it


def cuda(x, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()


def rel(got, want):
    got = got.cpu().numpy() if torch.is_tensor(got) else np.asarray(got)
    return float(np.max(np.abs(got.astype(np.float64) - want)) / max(float(np.max(np.abs(want))), 1.0))


CASES = [(n, mdh, pris, dt, g) for n in range(1, 11) for mdh in (0, 1) for pris in (False, True)
         for dt in (np.float64, np.float32) for g in ("default", "custom")]


@pytest.mark.parametrize("n,mdh,pris,dt,g", CASES,
                         ids=[f"n{c[0]}-{'mdh' if c[1] else 'dh'}-{'pris' if c[2] else 'rev'}-{np.dtype(c[3]).name}-{c[4]}" for c in CASES])
def test_regressor_matches_the_reference(n, mdh, pris, dt, g):
    L = R.robot(n, mdh, pris, True, 900 + 10 * n + 4 * mdh + 2 * pris)
    rob = R.dhrobot(L, mdh)
    q, qd, qdd = RR.states(L, 45, n)
    q, qd, qdd = (x.astype(dt).astype(np.float64) for x in (q, qd, qdd))  # the reference sees what the kernel sees
    gravity = None if g == "default" else G_CUSTOM
    Y = rob.rne_regressor(cuda(q, dt), cuda(qd, dt), cuda(qdd, dt), gravity=gravity)
    assert Y.dtype == (torch.float64 if dt == np.float64 else torch.float32) and tuple(Y.shape) == (45, n, 14 * n)
    want = RR.regressor(L, mdh, rob._kernel_gravity(gravity), q, qd, qdd)
    assert rel(Y, want) <= TOL[dt], rel(Y, want)
    assert torch.all(Y[:, torch.from_numpy(RR.structural_mask(n)).cuda()] == 0)  # exact zeros


def models():
    out = []
    for name in ("Puma560", "PandaMDH", "UR10"):
        r = getattr(rtb.models, name)()
        out += [(name, r), (name + "-nofriction", r.nofriction(True, True))]
    return out


@pytest.mark.parametrize("name,rob", models(), ids=[m[0] for m in models()])
def test_regressor_times_parameters_is_rne(name, rob):
    n = rob.n
    pi = cuda(rob.dynamic_parameters())
    rng = np.random.default_rng(5)
    for N in (1, 31, 32, 33, 4097, 1 << 20):
        q = cuda(rng.uniform(-np.pi, np.pi, (N, n)))
        qd = cuda(rng.choice([-1.0, 0.0, 1.0], (N, n)) * rng.uniform(0.1, 2.0, (N, n)))
        qdd = cuda(rng.normal(size=(N, n)))
        Y = rob.rne_regressor(q, qd, qdd)
        tau = rob.rne(q, qd, qdd)
        assert rel(torch.einsum("rjk,k->rj", Y, pi), tau.cpu().numpy()) < 1e-9, (name, N)
        del Y
    # one state as (n,) arrays on the host
    y1 = rob.rne_regressor(np.zeros(n), np.ones(n), np.ones(n))
    assert isinstance(y1, np.ndarray) and y1.shape == (n, 14 * n)


def test_regressor_depends_on_kinematics_and_gear_ratios_only():
    a = rtb.models.Puma560()
    L = a._pack_rne().reshape(-1, 24).copy()
    rng = np.random.default_rng(3)
    L[:, 6] *= 2.5
    L[:, 7:10] += rng.normal(size=(6, 3)) * 0.05
    L[:, 10:19] *= 3.0
    L[:, 19] *= 0.5
    L[:, 21:24] *= -2.0
    b = R.dhrobot(L.ravel(), 0)
    q, qd, qdd = (cuda(rng.normal(size=(1000, 6))) for _ in range(3))
    assert torch.equal(a.rne_regressor(q, qd, qdd), b.rne_regressor(q, qd, qdd))


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["Puma560", "PandaMDH"])
def test_gram_matches_the_materialised_regressor(name, dt):
    rob = getattr(rtb.models, name)()
    n, p = rob.n, 14 * rob.n
    rng = np.random.default_rng(8)
    for N in (1, 4095, 4096, 4097, 8193):
        q, qd, qdd, tau = (cuda(rng.normal(size=(N, n)), dt) for _ in range(4))
        Y = rob.rne_regressor(q, qd, qdd).double()
        t = tau.double()
        for w in (None, rng.uniform(0.0, 2.0, n)):
            W = torch.ones(n, dtype=torch.float64, device="cuda") if w is None else cuda(w)
            G, b, s = rob.regressor_gram(q, qd, qdd, tau, weights=w)
            assert G.shape == (p, p) and b.shape == (p,) and G.dtype == np.float64
            Gw = torch.einsum("rjk,j,rjl->kl", Y, W, Y).cpu().numpy()
            bw = torch.einsum("rjk,j,rj->k", Y, W, t).cpu().numpy()
            sw = float(torch.einsum("rj,j,rj->", t, W, t))
            assert rel(G, Gw) < 1e-11 and rel(b, bw) < 1e-11 and abs(s - sw) <= 1e-11 * max(abs(sw), 1.0), (N, w is None)
            assert np.array_equal(G, G.T)
            G2, b2, s2 = rob.regressor_gram(q, qd, qdd, tau, weights=w)
            assert np.array_equal(G, G2) and np.array_equal(b, b2) and s == s2


def rms_floor(s, count):
    """What rms = sqrt((s - 2 pi.b + pi.G.pi) / count) resolves: the three terms are each about s, so the difference
    carries a rounding error of a few eps s, and an exact fit reads as up to sqrt(eps) times the rms of tau."""
    return np.sqrt(16 * np.finfo(np.float64).eps * s / count)


def trajectory(n, N, seed):
    rng = np.random.default_rng(seed)
    return (rng.uniform(-np.pi, np.pi, (N, n)), rng.choice([-1.0, 1.0], (N, n)) * rng.uniform(0.05, 2.0, (N, n)),
            rng.normal(size=(N, n)) * 3)


@pytest.mark.parametrize("name", ["Puma560", "PandaMDH", "UR10"])
def test_identify_recovers_the_identifiable_combinations(name):
    rob = getattr(rtb.models, name)()
    n = rob.n
    q, qd, qdd = (cuda(x) for x in trajectory(n, 20000, 11))
    tau = rob.rne(q, qd, qdd)
    res = rob.identify(q, qd, qdd, tau)
    G, b, s = rob.regressor_gram(q, qd, qdd, tau)
    assert res.rms <= rms_floor(s, tau.numel()), (res.rms, rms_floor(s, tau.numel()))
    d = res.pi - rob.dynamic_parameters()
    assert np.max(np.abs(G @ d)) <= 1e-7 * np.max(np.abs(b)), np.max(np.abs(G @ d))
    # the rank is that of the stacked regressor (checked at a small N)
    qs, qds, qdds = (x[:300] for x in (q, qd, qdd))
    Ys = rob.rne_regressor(qs, qds, qdds).cpu().numpy().reshape(-1, 14 * n)
    norms = np.linalg.norm(Ys, axis=0)
    nz = norms > 1e3 * np.finfo(np.float64).eps * norms.max()  # identify's zero columns
    sv = np.linalg.svd(Ys[:, nz] / norms[nz], compute_uv=False)  # and its scaling: unit columns
    assert rob.identify(qs, qds, qdds, rob.rne(qs, qds, qdds)).rank == int(np.sum(sv ** 2 > 1e-10 * sv[0] ** 2))


def column_residuals(G, s, d):
    """|y_k . (Y d)| / (|y_k| sqrt(s)) per nonzero column k of Y: how much of the residual Y d of a parameter error d
    each column still explains, independently of the column's scale (the armature columns are 1e4 times the inertial
    ones on Puma560)."""
    g = np.diag(G)
    nz = g > 0
    return np.abs(G @ d)[nz] / np.sqrt(g[nz] * s)


@pytest.mark.parametrize("name", ["Puma560", "PandaMDH"])
def test_identify_in_float32_keeps_every_identifiable_parameter(name):
    """In float32 the inertial columns sit 1e-4 and less below the armature columns: none of them may be taken for a
    zero column.  With an rcond above float32's rounding the rank is the float64 rank, and no column explains what the
    float32 fit leaves."""
    rob = getattr(rtb.models, name)()
    n = rob.n
    q, qd, qdd = (x.astype(np.float32).astype(np.float64) for x in trajectory(n, 20000, 13))
    q64, qd64, qdd64 = cuda(q), cuda(qd), cuda(qdd)
    tau = rob.rne(q64, qd64, qdd64)
    r64 = rob.identify(q64, qd64, qdd64, tau)
    # rcond above float32's rounding of the scaled gram (1e-10 suits float64)
    r32 = rob.identify(cuda(q, np.float32), cuda(qd, np.float32), cuda(qdd, np.float32), tau.float(), rcond=1e-5)
    G, b, s = rob.regressor_gram(q64, qd64, qdd64, tau)
    G32 = rob.regressor_gram(cuda(q, np.float32), cuda(qd, np.float32), cuda(qdd, np.float32), tau.float())[0]
    ratio = np.sqrt(np.diag(G32) / np.diag(G32).max())
    assert r32.rank == r64.rank, (r32.rank, r64.rank, np.sort(ratio[(ratio > 0) & (np.diag(G) <= 1e-24 * np.diag(G).max())]))
    true = rob.dynamic_parameters()
    assert np.max(column_residuals(G, s, r64.pi - true)) < 1e-9
    assert np.max(column_residuals(G, s, r32.pi - true)) < 1e-4, np.max(column_residuals(G, s, r32.pi - true))


def test_identify_without_friction_on_a_friction_free_robot():
    """friction=False drops all four joint columns, the armature G^2 Jm qdd among them, so the robot has none either."""
    rob = rtb.models.Puma560().nofriction(True, True)
    for link in rob.links:
        link.Jm = 0.0
    q, qd, qdd = (cuda(x) for x in trajectory(6, 5000, 12))
    tau = rob.rne(q, qd, qdd)
    w = np.linspace(0.5, 2.0, 6)
    res = rob.identify(q, qd, qdd, tau, friction=False, weights=w)
    assert res.rms <= rms_floor(rob.regressor_gram(q, qd, qdd, tau, weights=w)[2], tau.numel())
    assert np.all(res.pi.reshape(6, 14)[:, 10:] == 0)
    # with friction kept, noise on tau shows in rms
    res2 = rob.identify(q, qd, qdd, tau + 0.01 * torch.randn_like(tau))
    assert 0.005 < res2.rms < 0.02


def test_bad_input_is_rejected_before_launch_and_an_empty_batch_launches_nothing():
    rob = rtb.models.Puma560()
    n0 = rtb.launch_count()
    x = cuda(np.zeros((4, 6)))
    with pytest.raises(ValueError):
        rob.rne_regressor(x, x, cuda(np.zeros((4, 5))))
    with pytest.raises(ValueError):
        rob.regressor_gram(x, x, x, cuda(np.zeros((3, 6))))
    with pytest.raises(ValueError):
        rob.regressor_gram(x, x, x, x, weights=np.ones(5))
    with pytest.raises(ValueError, match="weights"):
        rob.regressor_gram(x, x, x, x, weights=-np.ones(6))
    with pytest.raises(ValueError, match="weights"):
        rob.regressor_gram(x, x, x, x, weights=np.full(6, np.nan))
    e = cuda(np.zeros((0, 6)))
    assert tuple(rob.rne_regressor(e, e, e).shape) == (0, 6, 84)
    G, b, s = rob.regressor_gram(e, e, e, e)
    assert not G.any() and not b.any() and s == 0.0
    torch.cuda.synchronize()
    assert rtb.launch_count() == n0
