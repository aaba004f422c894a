"""Static forces without a GPU: the float64 restatement of tests/static_ref.py against the oracle, the worked paycap case,
the host side of DHRobot (mass table, payload) and the argument checks of the Python methods and of the C entry points,
all of which run before any device is touched."""
import numpy as np
import pytest

import b2kin as rtb
import rne_wrench_ref as wref
import static_ref as ref
from oracle import chains as ch
from oracle import oracle as orc

ROBOTS = wref.robots()


def base_of(name):
    return ch.trotz(0.4) @ ch.troty(-0.9) @ ch.transl(0.1, -0.2, 0.3) if sum(map(ord, name)) % 2 else None


@pytest.mark.parametrize("name,n,mdh,L,physical", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_gravjac_restatement_matches_oracle(name, n, mdh, L, physical):
    rng = np.random.default_rng(sum(map(ord, name)))
    links = ref.links_of(n, L)
    base = base_of(name)
    tool = ch.panda_mdh_tool() if name == "panda_mdh" else None
    q = rng.uniform(-3, 3, (8, n))
    g = np.array([0.3, -0.5, -9.81])
    tau, J0 = ref.gravjac(links, mdh, q, g, base, tool)
    gb = g if base is None else base[:3, :3].T @ g
    want = orc.dyn_gravload(lambda a, b, c, gg: orc.rne(n, mdh, L, gg, a, b, c), n, q, -gb)
    if physical:
        np.testing.assert_allclose(tau, want, rtol=1e-11, atol=1e-11 * max(1.0, np.abs(want).max()))
    else:  # ne.c's quirk for MDH with a prismatic first joint bends gravload; gravjac stays physical
        assert not np.allclose(tau, want, rtol=1e-6, atol=1e-6)
    chain = orc.Chain(ch.dh_to_ets(links, mdh=bool(mdh), base=base, tool=tool))
    np.testing.assert_allclose(J0, chain.jacob0(q), rtol=1e-12, atol=1e-12)


def test_flipped_joints_follow_the_chain():
    rng = np.random.default_rng(3)
    for mdh in (0, 1):
        L = ch.pack_rne(wref.random_links(rng, 5, mdh, prismatic=True), mdh=bool(mdh))
        links = ref.links_of(5, L, flips=[1, 0, 1, 1, 0])
        q = rng.uniform(-2, 2, (6, 5))
        _, J0 = ref.gravjac(links, mdh, q, np.zeros(3))
        np.testing.assert_allclose(J0, orc.Chain(ch.dh_to_ets(links, mdh=bool(mdh))).jacob0(q), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name,n,mdh,L,physical", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_pay_frame1_is_rne_with_the_opposite_tip_wrench(name, n, mdh, L, physical):
    if not physical:
        pytest.skip("ne.c's quirk for MDH with a prismatic first joint")
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    links = ref.links_of(n, L)
    q = rng.uniform(-3, 3, (5, n))
    for W in rng.normal(size=(3, 6)):
        z = np.zeros_like(q)
        want = orc.rne(n, mdh, L, np.zeros(3), q, z, z, fext=-W)
        np.testing.assert_allclose(ref.pay(links, mdh, W, q, 1), want, rtol=1e-11, atol=1e-11 * max(1.0, np.abs(want).max()))
        # frame 0 is the same wrench expressed in the world frame
        _, _, R = ref._row(links, mdh, q[0], None, None, np.zeros(3))
        W0 = np.concatenate([R @ W[:3], R @ W[3:]])
        np.testing.assert_allclose(ref.pay(links, mdh, W0, q[:1], 0), want[:1], rtol=1e-11, atol=1e-11 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("name,n,mdh,L,physical", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_friction_is_what_rne_adds(name, n, mdh, L, physical):
    rng = np.random.default_rng(sum(map(ord, name)) + 2)
    q, qd, qdd = rng.uniform(-3, 3, (7, n)), rng.normal(size=(7, n)), rng.normal(size=(7, n))
    qd[0] = 0.0
    g = np.array([0, 0, 9.81])
    d = orc.rne(n, mdh, L, g, q, qd, qdd) - orc.rne(n, mdh, orc.nofriction_L(L), g, q, qd, qdd)
    np.testing.assert_allclose(d, -ref.friction(ref.links_of(n, L), qd), rtol=1e-12, atol=1e-12)


def test_worked_paycap_case():
    c = ref.PLANAR_2R_CASE
    links = ref.PLANAR_2R
    tauB, _ = ref.gravjac(links, 0, c["q"], c["gravity"])
    np.testing.assert_allclose(tauB[0], c["tauB"], rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(ref.pay(links, 0, c["w"], c["q"], c["frame"])[0], c["tauP"], rtol=1e-14, atol=1e-14)
    wmax, joint = ref.paycap(links, 0, c["w"], c["tauR"], c["frame"], c["q"], c["gravity"])
    np.testing.assert_allclose(wmax[0], c["wmax"], rtol=1e-13)
    assert joint[0] == c["joint"]
    # a zero row gives NaN and -1; an unloaded joint +inf
    wmax, joint = ref.paycap(links, 0, [[0] * 6, [0, 0, 1, 0, 0, 0]], c["tauR"], 0, [c["q"]] * 2, c["gravity"])
    assert np.isnan(wmax[0]).all() and joint[0] == -1
    assert np.isinf(wmax[1]).all() and joint[1] == 0


def test_mass_table_and_payload_on_the_host():
    puma = rtb.models.Puma560()
    M = puma._static_mass_table()
    for j, l in enumerate(puma.links):  # standard DH: the tail behind the joint is tz(d) tx(a) Rx(alpha)
        A = ch.transl(0, 0, l.d) @ ch.transl(l.a, 0, 0) @ ch.trotx(l.alpha)
        np.testing.assert_allclose(M[j], np.concatenate([[l.m], (A @ np.append(l.r, 1))[:3]]), rtol=0, atol=1e-15)
    assert puma._static_mass_table() is M  # cached
    I6 = puma.links[5].I.copy()
    puma.payload(2.5, [0, 0, 0.1])
    assert puma._dynchanged and puma._static_mass is None
    assert puma.links[5].m == 2.5 and np.array_equal(puma.links[5].r, [0, 0, 0.1]) and np.array_equal(puma.links[5].I, I6)
    np.testing.assert_allclose(puma._static_mass_table()[5], [2.5, 0, 0, 0.1])
    puma.payload(0)
    assert puma.links[5].m == 0 and puma._static_mass_table()[5, 0] == 0
    puma.links[1].a = 0.5  # a kinematic change drops the table too
    assert puma._static_mass is None
    assert puma._static_mass_table()[1, 1] == pytest.approx(0.5 - 0.3638)
    mdh = rtb.models.PandaMDH()  # modified DH: the joint is the link's last transform, so c_j = r_j
    Mm = mdh._static_mass_table()
    for j, l in enumerate(mdh.links):
        np.testing.assert_array_equal(Mm[j, 1:], l.r)


def test_argument_errors_come_before_any_device():
    puma = rtb.models.Puma560()
    q = np.zeros(6)
    with pytest.raises(ValueError, match="tauR"):
        puma.paycap([0, 0, -1, 0, 0, 0], np.ones((6, 3)), q=q)
    with pytest.raises(ValueError, match="tauR"):
        puma.paycap([0, 0, -1, 0, 0, 0], np.ones((2, 6)), q=q)
    with pytest.raises(ValueError, match="needs q"):
        puma.paycap([0, 0, -1, 0, 0, 0], np.ones((6, 2)))
    with pytest.raises(ValueError, match="zero"):
        puma.paycap(np.zeros(6), np.ones((6, 2)), q=q)
    with pytest.raises(ValueError, match="frame"):
        puma.paycap([0, 0, -1, 0, 0, 0], np.ones((6, 2)), frame=2, q=q)
    with pytest.raises(ValueError, match="exactly one"):
        puma.pay(np.ones(6))
    with pytest.raises(ValueError, match="exactly one"):
        puma.pay(np.ones(6), q=q, J=np.zeros((6, 6)))
    with pytest.raises(ValueError, match="frame"):
        puma.pay(np.ones(6), q=q, frame=-1)
    with pytest.raises(ValueError, match="shape"):
        puma.pay(np.ones(5), q=q)
    with pytest.raises(ValueError, match="shape"):
        puma.pay(np.ones((3, 6)), q=np.zeros((4, 6)))
    with pytest.raises(ValueError, match="J must be"):
        puma.pay(np.ones(6), J=np.zeros((5, 6)))
    with pytest.raises(ValueError, match="qd must"):
        puma.friction(np.zeros(5))


def test_entry_points_validate_before_cuda():
    """Every rejection below returns B2K_ERR_INVALID from host-side checks; N = 0 returns OK without a device."""
    L = rtb._lib.lib()
    puma = rtb.models.Puma560()
    chain = puma.ets()._chain
    mass = puma._static_mass_table()
    g = np.array([0, 0, -9.81])
    tauR = np.ones((6, 2))
    params = np.zeros((6, 4))
    dp = rtb._lib.dptr
    F64, F32 = rtb._lib.F64, rtb._lib.F32
    fake = 1 << 20  # aligned; never dereferenced on the paths below
    bad = [
        L.b2k_gravjac(None, F64, fake, 4, 6, dp(mass), dp(g), fake, fake, None),
        L.b2k_gravjac(chain, 7, fake, 4, 6, dp(mass), dp(g), fake, fake, None),
        L.b2k_gravjac(chain, F64, fake, -1, 6, dp(mass), dp(g), fake, fake, None),
        L.b2k_gravjac(chain, F64, fake, 4, 5, dp(mass), dp(g), fake, fake, None),
        L.b2k_gravjac(chain, F64, fake, 4, 6, None, dp(g), fake, fake, None),
        L.b2k_gravjac(chain, F64, fake, 4, 6, dp(mass), None, fake, fake, None),
        L.b2k_gravjac(chain, F64, fake, 4, 6, dp(mass), dp(g), None, fake, None),
        L.b2k_gravjac(chain, F64, fake + 4, 4, 6, dp(mass), dp(g), fake, fake, None),
        L.b2k_gravjac(chain, F64, fake, 4, 6, dp(mass), dp(g), fake, fake + 2, None),
        L.b2k_pay(chain, F64, fake, 4, 6, fake, 6, 2, fake, None),
        L.b2k_pay(chain, F64, fake, 4, 6, fake, 3, 1, fake, None),
        L.b2k_pay(chain, F64, fake, 4, 6, None, 0, 1, fake, None),
        L.b2k_pay(chain, F32, fake, 4, 6, fake + 2, 0, 1, fake, None),
        L.b2k_pay_jacobian(F64, 0, fake, fake, 0, 4, fake, None),
        L.b2k_pay_jacobian(F64, 11, fake, fake, 0, 4, fake, None),
        L.b2k_pay_jacobian(F64, 6, None, fake, 0, 4, fake, None),
        L.b2k_pay_jacobian(F64, 6, fake, fake, 0, 4, fake + 4, None),
        L.b2k_paycap(chain, F64, fake, 4, 6, dp(mass), dp(g), fake, 0, 1, None, fake, fake, None),
        L.b2k_paycap(chain, F64, fake, 4, 6, dp(mass), dp(g), fake, 0, 3, dp(tauR), fake, fake, None),
        L.b2k_paycap(chain, F64, fake, 4, 6, dp(mass), dp(g), fake, 0, 1, dp(tauR), fake, None, None),
        L.b2k_paycap(chain, F64, fake, 4, 6, dp(mass), dp(g), fake, 0, 1, dp(tauR), fake, fake + 2, None),
        L.b2k_friction(F64, 6, None, fake, 4, fake, None),
        L.b2k_friction(F64, 0, dp(params), fake, 4, fake, None),
        L.b2k_friction(F64, 6, dp(params), fake + 1, 4, fake, None),
    ]
    assert bad == [-1] * len(bad), bad
    nanmass = mass.copy()
    nanmass[2, 1] = np.nan
    assert L.b2k_gravjac(chain, F64, fake, 4, 6, dp(nanmass), dp(g), fake, fake, None) == -1
    assert b"not finite" in L.b2k_last_error()
    ok = [
        L.b2k_gravjac(chain, F64, None, 0, 6, dp(mass), dp(g), None, None, None),
        L.b2k_pay(chain, F32, None, 0, 6, None, 0, 0, None, None),
        L.b2k_pay_jacobian(F64, 6, None, None, 6, 0, None, None),
        L.b2k_paycap(chain, F64, None, 0, 6, dp(mass), dp(g), None, 6, 1, dp(tauR), None, None, None),
        L.b2k_friction(F32, 6, dp(params), None, 0, None, None),
    ]
    assert ok == [0] * len(ok), ok
