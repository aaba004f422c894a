"""Closed-form inverse kinematics of UR-type arms (DHRobot.ikine_ur) without a GPU: the C ABI and the public method reject
bad arguments and robots outside the UR link pattern before any CUDA call, and the numpy restatement in ikine_ur_ref.py --
the specification the kernel is checked against -- is pinned by round trips through the oracle's forward kinematics, by
branch recovery and by the configuration predicates."""
import os
import sys

import numpy as np
import pytest

import b2kin as rtb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_ur_ref as ref  # noqa: E402

lib = rtb._lib.lib()
UR10_DH = ref.dh_table(rtb.models.UR10())
h = np.pi / 2


def _call(dtype=1, dh=UR10_DH, base=None, tool=None, T=8, N=4, nconf=1, conf=(0,), q=8, ok=8):
    dh = None if dh is None else np.ascontiguousarray(dh, dtype=np.float64)
    c = None if conf is None else np.ascontiguousarray(conf, dtype=np.int32)
    rc = lib.b2k_ikine_ur(dtype, rtb._lib.dptr(dh), rtb._lib.dptr(base), rtb._lib.dptr(tool), T, N, nconf,
                          None if c is None else c.ctypes.data_as(rtb._lib.ip), q, ok, None)
    return rc, lib.b2k_last_error().decode()


def _dh(**changes):
    """the UR10 table with entries replaced: key '<name><link>' with name in d, a, alpha, off and link 1..6"""
    dh = UR10_DH.copy()
    for key, v in changes.items():
        name, link = key[:-1], int(key[-1])
        dh[link - 1, {"d": 0, "a": 1, "alpha": 2, "off": 3}[name]] = v
    return dh


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=2), "b2k_ikine_ur: bad dtype"),
    (dict(N=-1), "bad N"),
    (dict(nconf=0), "nconf must be 1..8, got 0"),
    (dict(nconf=9, conf=range(9)), "nconf must be 1..8, got 9"),
    (dict(conf=(8,)), "configuration code 8 of slot 0 is not 0..7"),
    (dict(nconf=2, conf=(0, -1)), "configuration code -1 of slot 1"),
    (dict(dh=None), "dh and conf must not be NULL"),
    (dict(conf=None), "dh and conf must not be NULL"),
    (dict(T=None), "T, q and ok must not be NULL"),
    (dict(q=None), "T, q and ok must not be NULL"),
    (dict(ok=None), "T, q and ok must not be NULL"),
    (dict(dh=_dh(d2=np.nan)), "dh[1][0] is not finite"),
    (dict(dh=_dh(off6=np.inf)), "dh[5][3] is not finite"),
    (dict(dh=_dh(alpha1=-h)), "not a UR-type arm: alpha1 must be +pi/2"),
    (dict(dh=_dh(a1=0.1)), "a1 must be 0"),
    (dict(dh=_dh(alpha2=0.3)), "alpha2 must be 0"),
    (dict(dh=_dh(a2=0.0)), "a2 must not be 0"),
    (dict(dh=_dh(alpha3=-h)), "alpha3 must be 0 (got -1.5707963267948966)"),
    (dict(dh=_dh(a3=0.0)), "a3 must not be 0"),
    (dict(dh=_dh(a3=5e-10)), "a3 must not be 0"),
    (dict(dh=_dh(alpha4=-h)), "alpha4 must be +pi/2"),
    (dict(dh=_dh(a4=0.01)), "a4 must be 0"),
    (dict(dh=_dh(alpha5=h)), "alpha5 must be -pi/2"),
    (dict(dh=_dh(a5=0.01)), "a5 must be 0"),
    (dict(dh=_dh(alpha1=h + 2e-9)), "alpha1 must be +pi/2"),
    (dict(dh=ref.dh_table(rtb.models.Puma560())), "b2k_ikine_ur: not a UR-type arm: alpha3 must be 0"),
])
def test_entry_rejects_bad_arguments_before_launching(kw, msg):
    rc, err = _call(**kw)
    assert rc == -1
    assert msg in err, err


def test_entry_accepts_what_it_documents_without_work():
    # N = 0 returns before touching the device; every argument below is valid
    assert _call(N=0)[0] == 0
    assert _call(N=0, T=None, q=None, ok=None)[0] == 0
    assert _call(N=0, nconf=8, conf=range(8))[0] == 0
    assert _call(N=0, base=np.eye(4), tool=np.eye(4))[0] == 0
    assert _call(N=0, dtype=0)[0] == 0
    # d1 .. d6, a6, alpha6, the offsets and either sign of a2 and a3 are free; each pattern entry is held to 1e-9
    assert _call(N=0, dh=_dh(d1=1, d2=0.3, d3=-0.2, d4=0, d5=-0.1, d6=0, a2=0.4, a3=-0.3, a6=0.05, alpha6=1.0, off1=0.3,
                             off5=-2, alpha1=h + 5e-10, alpha3=-5e-10))[0] == 0


def test_the_puma_entry_keeps_its_own_messages():
    rc = lib.b2k_ikine_6s(1, rtb._lib.dptr(UR10_DH), None, None, None, 0, 1, np.zeros(1, np.int32).ctypes.data_as(rtb._lib.ip),
                          None, None, None)
    assert rc == -1
    assert lib.b2k_last_error().decode() == (
        "b2k_ikine_6s: not a Puma-type arm: alpha3 must be -pi/2 (got 0); the closed form needs alpha = (pi/2, 0, -pi/2, "
        "+-pi/2, -+pi/2, any), a1 = a4 = a5 = 0, d5 = 0, a2 != 0")


def _robots():
    rng = np.random.default_rng(2025)
    return [rtb.models.UR10()] + [ref.random_robot(rtb, rng) for _ in range(16)]


def well_conditioned(c, s5, rm, ax):
    return (c > 1e-4) & (s5 > 1e-2) & (rm > 1e-4) & (ax > 1e-4)


def _q(rng, dh, n=2000):
    """random joint vectors, with rows at theta5 = 0 and pi exactly (theta6 = 0 there, the solver's choice)"""
    q = rng.uniform(-np.pi, np.pi, (n, 6))
    q[:100, 4] = np.where(np.arange(100) < 50, 0.0, np.pi) - dh[4, 3]
    q[:100, 5] = -dh[5, 3]
    return q


@pytest.mark.parametrize("k", range(17))
def test_restatement_round_trips_and_recovers_its_branch(k):
    rob = _robots()[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(300 + k)
    q = _q(rng, dh)
    T = ref.fk(rob, q)
    codes = ref.config_code(dh, q)
    wrist_singular = np.arange(len(q)) < 100
    sols, goods = [], []
    for code in range(8):
        qs, ok = ref.ikine_ur(dh, rob._base, rob._tool, T, code)
        # every row off the wrist singularity is reachable in its own configuration; the others may be out of reach.  At
        # theta5 = 0 or pi, |u| and |v| can round to more than 10 eps, and theta6 from rounding noise then moves O4.
        assert ok[(codes == code) & ~wrist_singular].all()
        assert np.isnan(qs[~ok]).all() and np.isfinite(qs[ok]).all()
        assert np.abs(ref.fk(rob, qs[ok]) - T[ok]).max() <= 1e-12, (code, np.abs(ref.fk(rob, qs[ok]) - T[ok]).max())
        good = ok & well_conditioned(*ref.margins(dh, rob._base, rob._tool, T, code))
        assert (ref.config_code(dh, qs[good]) == code).all()  # every solution has the letters asked for
        sel = good & (codes == code)
        assert sel.sum() >= 50
        assert np.abs(ref.wrap(qs[sel] - q[sel])).max() <= 1e-9  # the solution in q's own configuration is q
        sols.append(qs)
        goods.append(good)
    # the solutions of a well-conditioned row are eight distinct joint vectors
    S = np.stack(sols, 1)
    every = np.all(goods, 0)
    assert every.sum() >= 100
    for i in range(8):
        for j in range(i):
            assert (np.abs(ref.wrap(S[every, i] - S[every, j])).max(-1) > 1e-6).all(), (i, j)


def test_wrist_singular_rows_round_trip():
    rob = _robots()[3]
    dh = ref.dh_table(rob)
    q = _q(np.random.default_rng(8), dh, 100)
    T = ref.fk(rob, q)
    assert np.abs(np.sin(q[:, 4] + dh[4, 3])).max() < 1e-15
    for code in range(8):
        qs, ok = ref.ikine_ur(dh, rob._base, rob._tool, T, code)
        assert ok.sum() >= 40
        assert np.abs(ref.fk(rob, qs[ok]) - T[ok]).max() <= 1e-12


def test_only_the_sum_of_d2_d3_d4_matters():
    rng = np.random.default_rng(9)
    rob = _robots()[5]
    dh = ref.dh_table(rob)
    shift = np.array([0.0, 0.3, -0.5, 0.2, 0.0, 0.0])
    rob2 = rtb.DHRobot([rtb.RevoluteDH(d=x[0] + s, a=x[1], alpha=x[2], offset=x[3]) for x, s in zip(dh, shift)],
                       base=rob._base, tool=rob._tool)
    dh2 = ref.dh_table(rob2)
    q = rng.uniform(-np.pi, np.pi, (1000, 6))
    T = ref.fk(rob, q)
    np.testing.assert_allclose(ref.fk(rob2, q), T, atol=1e-14)  # the same arm
    for code in range(8):
        q1, ok1 = ref.ikine_ur(dh, rob._base, rob._tool, T, code)
        q2, ok2 = ref.ikine_ur(dh2, rob2._base, rob2._tool, T, code)
        good = ok1 & well_conditioned(*ref.margins(dh, rob._base, rob._tool, T, code))
        assert (ok1 == ok2)[good].all()
        assert np.abs(ref.wrap(q1[good] - q2[good])).max() <= 1e-12


def test_restatement_marks_both_kinds_of_unreachable_pose():
    u = rtb.models.UR10()
    dh = ref.dh_table(u)
    T = np.tile(ref.fk(u, u.qr)[0], (3, 1, 1))
    T[1, :3, 3] = (0.05, 0.0, 0.5)  # on the first axis: r < |D|
    T[2, :3, 3] = (2.0, 0.5, 0.5)   # beyond the stretched arm: |c3| > 1
    for code in range(8):
        q, ok = ref.ikine_ur(dh, u._base, u._tool, T, code)
        assert ok[1:].tolist() == [False, False]
        assert np.isnan(q[1:]).all()


@pytest.mark.parametrize("name,letters", [("qz", "ldn"), ("qr", "ldn")])
def test_ur10_named_configurations_round_trip_in_their_own_letters(name, letters):
    """qz and qr have a straight elbow: c3 = 1 up to rounding, inside the elbow band"""
    u = rtb.models.UR10()
    dh = ref.dh_table(u)
    qn = getattr(u, name)
    assert ref.config_of(dh, qn) == [letters]
    T = ref.fk(u, qn)
    q, ok = ref.ikine_ur(dh, u._base, u._tool, T, letters)
    assert ok.all()
    np.testing.assert_allclose(ref.fk(u, q), T, atol=1e-12)
    # theta3 = acos(c3) is sqrt-sensitive at a straight elbow: an ulp of c3 is 2e-8 of theta3
    np.testing.assert_allclose(ref.wrap(q[0] - qn), 0, atol=1e-7)
    # the other shoulder is genuinely out of reach at both poses
    assert not ref.ikine_ur(dh, u._base, u._tool, T, "r" + letters[1:])[1].any()


def _prismatic():
    L = [rtb.RevoluteDH(d=x[0], a=x[1], alpha=x[2]) for x in UR10_DH]
    L[2] = rtb.PrismaticDH(a=UR10_DH[2, 1], alpha=UR10_DH[2, 2])
    return rtb.DHRobot(L)


def _mdh():
    return rtb.DHRobot([rtb.RevoluteMDH(d=x[0], a=x[1], alpha=x[2]) for x in UR10_DH])


def _flipped():
    return rtb.DHRobot([rtb.RevoluteDH(d=x[0], a=x[1], alpha=x[2], flip=j == 4) for j, x in enumerate(UR10_DH)])


def _table(dh):
    return lambda: rtb.DHRobot([rtb.RevoluteDH(d=x[0], a=x[1], alpha=x[2], offset=x[3]) for x in dh])


@pytest.mark.parametrize("make,msg", [
    (rtb.models.Puma560, "ikine_ur: not a UR-type arm: alpha3 must be 0"),
    (rtb.models.PandaMDH, "ikine_ur: the closed form serves 6-joint arms; this robot has 7 joints"),
    (_mdh, "ikine_ur: the closed form serves standard DH; this robot uses modified DH"),
    (_prismatic, "ikine_ur: joint 3 is prismatic"),
    (_flipped, "ikine_ur: joint 5 is flipped"),
    (_table(_dh(a3=0.0)), "a3 must not be 0"),
    (_table(_dh(d4=np.nan)), "dh[3][0] is not finite"),
])
def test_robots_outside_the_pattern_raise_before_any_device_work(make, msg):
    with pytest.raises(ValueError, match=msg.replace("[", r"\[").replace("]", r"\]")):
        make().ikine_ur(np.eye(4))


@pytest.mark.parametrize("config,msg", [
    ("lr", "more than one of 'lr'"),
    ("lux", "bad config specifier 'x'"),
    ([], "ikine_ur: give 1 to 8 configurations, got 0"),
    (["lun"] * 9, "ikine_ur: give 1 to 8 configurations, got 9"),
])
def test_bad_configurations_raise_before_any_device_work(config, msg):
    with pytest.raises(ValueError, match=msg):
        rtb.models.UR10().ikine_ur(np.eye(4), config=config)


def test_ikine_a_keeps_its_messages():
    with pytest.raises(ValueError, match="^ikine_a: give 1 to 8 configurations, got 0$"):
        rtb.models.Puma560().ikine_a(np.eye(4), config=[])
    with pytest.raises(ValueError, match="^ikine_a: the closed form serves 6-joint arms; this robot has 7 joints$"):
        rtb.models.PandaMDH().ikine_a(np.eye(4))
    with pytest.raises(ValueError, match="^b2k_ikine_6s: not a Puma-type arm: alpha3 must be -pi/2"):
        rtb.models.UR10().ikine_a(np.eye(4))
