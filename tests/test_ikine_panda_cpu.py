"""Closed-form inverse kinematics of Panda-type arms at a given q7 (DHRobot.ikine_panda) without a GPU: the C ABI and the
public method reject bad arguments and robots outside the Panda link pattern before any CUDA call, and the numpy
restatement in ikine_panda_ref.py -- the specification the kernel is checked against -- is pinned by round trips
through the oracle's modified-DH forward kinematics, by branch recovery and by the configuration predicates."""
import os
import re
import sys

import numpy as np
import pytest

import b2kin as rtb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_panda_ref as ref  # noqa: E402
from oracle import chains  # noqa: E402
from oracle import oracle as orc  # noqa: E402

lib = rtb._lib.lib()
PANDA_DH = ref.dh_table(rtb.models.PandaMDH())
h = np.pi / 2


def _call(dtype=1, dh=PANDA_DH, base=None, tool=None, T=8, q7=8, N=4, nconf=1, conf=(0,), q=8, ok=8):
    dh = None if dh is None else np.ascontiguousarray(dh, dtype=np.float64)
    c = None if conf is None else np.ascontiguousarray(conf, dtype=np.int32)
    rc = lib.b2k_ikine_panda(dtype, rtb._lib.dptr(dh), rtb._lib.dptr(base), rtb._lib.dptr(tool), T, q7, N, nconf,
                             None if c is None else c.ctypes.data_as(rtb._lib.ip), q, ok, None)
    return rc, lib.b2k_last_error().decode()


def _dh(**changes):
    """the PandaMDH table with entries replaced: key '<name><link>' with name in d, a, alpha, off and link 1..7"""
    dh = PANDA_DH.copy()
    for key, v in changes.items():
        name, link = key[:-1], int(key[-1])
        dh[link - 1, {"d": 0, "a": 1, "alpha": 2, "off": 3}[name]] = v
    return dh


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=2), "b2k_ikine_panda: bad dtype"),
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
    (dict(q7=None), "b2k_ikine_panda: q7 must not be NULL"),
    (dict(q7=12), "q7 must be aligned to its element size"),
    (dict(q7=6, dtype=0), "q7 must be aligned to its element size"),
    (dict(dh=_dh(d2=np.nan)), "dh[1][0] is not finite"),
    (dict(dh=_dh(off7=np.inf)), "dh[6][3] is not finite"),
    (dict(dh=_dh(alpha2=h)), "not a Panda-type arm: alpha2 must be -pi/2 (got 1.5707963267948966)"),
    (dict(dh=_dh(a2=0.1)), "a2 must be 0"),
    (dict(dh=_dh(d2=0.1)), "d2 must be 0"),
    (dict(dh=_dh(alpha3=-h)), "alpha3 must be +pi/2"),
    (dict(dh=_dh(a3=0.01)), "a3 must be 0"),
    (dict(dh=_dh(alpha4=0.0)), "alpha4 must be +pi/2"),
    (dict(dh=_dh(d4=0.01)), "d4 must be 0"),
    (dict(dh=_dh(a4=0.0, d3=0.0)), "hypot(a4, d3) must not be 0"),
    (dict(dh=_dh(alpha5=h)), "alpha5 must be -pi/2"),
    (dict(dh=_dh(a5=5e-10, d5=0.0)), "hypot(a5, d5) must not be 0"),
    (dict(dh=_dh(alpha6=-h)), "alpha6 must be +pi/2"),
    (dict(dh=_dh(a6=0.01)), "a6 must be 0"),
    (dict(dh=_dh(d6=0.01)), "d6 must be 0"),
    (dict(dh=_dh(alpha2=-h + 2e-9)), "alpha2 must be -pi/2"),
])
def test_entry_rejects_bad_arguments_before_launching(kw, msg):
    rc, err = _call(**kw)
    assert rc == -1
    assert msg in err, err


def test_entry_states_the_pattern_it_needs():
    rc, err = _call(N=0, dh=_dh(d4=0.2))
    assert rc == -1
    assert err == ("b2k_ikine_panda: not a Panda-type arm: d4 must be 0 (got 0.20000000000000001); the closed form needs "
                   "modified DH with alpha2 .. alpha6 = (-pi/2, pi/2, pi/2, -pi/2, pi/2), a2 = a3 = a6 = 0, d2 = d4 = d6 = 0, "
                   "hypot(a4, d3) != 0, hypot(a5, d5) != 0")


def test_entry_accepts_what_it_documents_without_work():
    # N = 0 returns before touching the device; every argument below is valid
    assert _call(N=0)[0] == 0
    assert _call(N=0, T=None, q7=None, q=None, ok=None)[0] == 0
    assert _call(N=0, nconf=8, conf=range(8))[0] == 0
    assert _call(N=0, base=np.eye(4), tool=np.eye(4))[0] == 0
    assert _call(N=0, dtype=0, q7=4)[0] == 0
    # a1, alpha1, d1, d3, a4, a5, d5, a7, alpha7, d7 and the offsets are free; each pattern entry is held to 1e-9
    assert _call(N=0, dh=_dh(a1=0.2, alpha1=1.0, d1=-0.3, d3=-0.2, a4=0.0, a5=0.3, d5=0.0, a7=-0.1, alpha7=-2.0, d7=0.0,
                             off1=0.3, off7=-2, alpha2=-h + 5e-10, d6=-5e-10))[0] == 0


def test_the_other_entries_keep_their_own_messages():
    conf = np.zeros(1, np.int32).ctypes.data_as(rtb._lib.ip)
    for fn in ("b2k_ikine_6s", "b2k_ikine_ur"):
        assert getattr(lib, fn)(1, rtb._lib.dptr(PANDA_DH[:6].copy()), None, None, None, 0, 1, conf, None, None, None) == -1
        assert lib.b2k_last_error().decode().startswith(f"{fn}: not a ")
    with pytest.raises(ValueError, match="^ikine_a: the closed form serves 6-joint arms; this robot has 7 joints$"):
        rtb.models.PandaMDH().ikine_a(np.eye(4))
    with pytest.raises(ValueError, match="^ikine_ur: the closed form serves standard DH; this robot uses modified DH$"):
        rtb.DHRobot([rtb.RevoluteMDH(d=0.1 * j) for j in range(6)]).ikine_ur(np.eye(4))


def _robots():
    rng = np.random.default_rng(2026)
    return [rtb.models.PandaMDH()] + [ref.random_robot(rtb, rng) for _ in range(16)]


def well_conditioned(el, wr, sh, hh):
    return (el > 1e-4) & (wr > 1e-4) & (sh > 1e-3) & (hh > 1e-3)


@pytest.mark.parametrize("k", range(17))
def test_restatement_round_trips_and_recovers_its_branch(k):
    rob = _robots()[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(400 + k)
    q = rng.uniform(-np.pi, np.pi, (400, 7))
    T = ref.fk_mdh(rob, q)
    np.testing.assert_allclose(ref.fk(rob, q), T, atol=1e-14)  # the oracle's ETS chain and its MDH link transform agree
    codes = ref.config_code(dh, q)
    sols, goods = [], []
    for code in range(8):
        qs, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q[:, 6], code)
        assert ok[codes == code].all()  # every row is reachable in its own configuration
        assert np.isnan(qs[~ok]).all() and np.isfinite(qs[ok]).all()
        assert (qs[ok, 6] == q[ok, 6]).all()  # q7 as given
        err = np.abs(ref.fk_mdh(rob, qs[ok]) - T[ok]).max()
        assert err <= 1e-12, (code, err)
        good = ok & well_conditioned(*ref.margins(dh, rob._base, rob._tool, T, q[:, 6], code))
        assert (ref.config_code(dh, qs[good]) == code).all()  # every solution has the letters asked for
        sel = good & (codes == code)
        assert sel.sum() >= 10
        assert np.abs(ref.wrap(qs[sel] - q[sel])).max() <= 1e-9  # the solution in q's own configuration is q
        sols.append(qs)
        goods.append(good)
    # the solutions of a well-conditioned row are distinct joint vectors
    S = np.stack(sols, 1)
    every = np.all(goods, 0)
    assert every.sum() >= 20
    for i in range(8):
        for j in range(i):
            assert (np.abs(ref.wrap(S[every, i] - S[every, j])).max(-1) > 1e-6).all(), (i, j)


def test_panda_solutions_round_trip_through_the_ets_model():
    """PandaMDH and the ETS Panda (oracle.chains.panda_ets) have the same kinematics"""
    rob = rtb.models.PandaMDH()
    dh = ref.dh_table(rob)
    C = orc.Chain(chains.panda_ets())
    q = np.random.default_rng(12).uniform(-np.pi, np.pi, (500, 7))
    T = C.fkine(q)
    for code in range(8):
        qs, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q[:, 6], code)
        assert ok.sum() >= 200
        assert np.abs(C.fkine(qs[ok]) - T[ok]).max() <= 1e-12


def test_named_configurations():
    rob = rtb.models.PandaMDH()
    dh = ref.dh_table(rob)
    assert ref.config_of(dh, rob.qr) == ["lun"]
    for name in ("qr", "qz"):
        qn = getattr(rob, name)
        T = ref.fk_mdh(rob, qn)
        letters = ref.config_of(dh, qn)[0]
        for code in range(8):
            q, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, qn[6], code)
            if ok.all():
                np.testing.assert_allclose(ref.fk_mdh(rob, q), T, atol=1e-12)
        q, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, qn[6], letters)
        assert ok.all()
        if name == "qr":
            np.testing.assert_allclose(ref.wrap(q[0] - qn), 0, atol=1e-12)
    # qz has sin(theta2) = 0: axes 1 and 3 coincide.  Its elbow-down solutions keep theta2 = 0: theta1 = 0 by the tr2eul
    # rule, and both shoulder codes give theta2 within rounding of 0, so both read as "r"
    T = ref.fk_mdh(rob, rob.qz)
    singular = 0
    for code in range(8):
        q, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, 0.0, code)
        assert ok.all()
        if abs(np.sin(q[0, 1])) < 1e-12:
            singular += 1
            assert q[0, 0] == 0 and 0 <= q[0, 1] < 1e-12
            assert ref.config_code(dh, q)[0] & 1 == 1
    assert singular == 4


def test_singular_shoulder_and_degenerate_wrist_rows_round_trip():
    rng = np.random.default_rng(13)
    for rob in _robots()[:6]:
        dh = ref.dh_table(rob)
        q = rng.uniform(-np.pi, np.pi, (300, 7))
        q[:100, 1] = rng.choice([0.0, np.pi], 100) - dh[1, 3]  # sin(theta2) = 0
        q[100:200, 4] = rng.choice([h, -h], 100) - dh[4, 3]     # theta5 = +-pi/2: on the wrist boundary
        q[200:, 3] = np.arctan2(dh[3, 1] * dh[4, 0] - dh[2, 0] * dh[4, 1], -dh[3, 1] * dh[4, 1] - dh[2, 0] * dh[4, 0]) \
            + rng.choice([0.0, np.pi], 100) - dh[3, 3]          # theta4 = phi or phi + pi: on the elbow boundary
        T = ref.fk_mdh(rob, q)
        codes = ref.config_code(dh, q)
        reached = np.zeros(len(q), bool)
        for code in range(8):
            qs, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q[:, 6], code)
            if ok.any():
                assert np.abs(ref.fk_mdh(rob, qs[ok]) - T[ok]).max() <= 1e-12
            reached |= ok & (codes % 4 == code % 4)
        assert reached[:100].all() and reached[200:].all() and reached[100:200].mean() >= 0.95


def _theta4_on_axis(dh, joint, sign):
    """theta4 (before the offset) that puts O2 on joint 6's axis (with theta5 = +-pi/2: p = 0) or on joint 5's axis
    (r = 0); with H = hypot(a4, d3), gamma = atan2(d3, a4): p = 0 at H sin(theta4 - gamma) = d5, r = 0 at
    H cos(theta4 - gamma) = -a5"""
    d3, a4, a5, d5 = dh[2, 0], dh[3, 1], dh[4, 1], dh[4, 0]
    H, g = np.hypot(a4, d3), np.arctan2(d3, a4)
    if joint == 6:
        return g + (np.arcsin(d5 / H) if sign > 0 else np.pi - np.arcsin(d5 / H)) - dh[3, 3]
    return g + sign * np.arccos(-a5 / H) - dh[3, 3]


@pytest.mark.parametrize("joint", [5, 6])
def test_degenerate_wrist_rows_round_trip(joint):
    """O2 on joint 6's axis (h = 0: theta6 is free, the solver takes psi = 0 and reads the wrist equation as p = 0), and
    O2 on joint 5's axis (theta5 is free, the solver takes theta5 = 0 where both of its arguments are at rounding)"""
    rng = np.random.default_rng(14 + joint)
    # joint 6's case needs |d5| < hypot(a4, d3), which PandaMDH does not have
    rob = _table(_dh(d5=0.2) if joint == 6 else PANDA_DH)()
    rob.base, rob.tool = ref.random_se3(rng), ref.random_se3(rng, 0.1)
    dh = ref.dh_table(rob)
    q = rng.uniform(-np.pi, np.pi, (200, 7))
    sign = rng.choice([-1, 1], 200)
    q[:, 3] = [_theta4_on_axis(dh, joint, s) for s in sign]
    if joint == 6:
        q[:, 4] = rng.choice([h, -h], 200) - dh[4, 3]
    T = ref.fk_mdh(rob, q)
    codes = ref.config_code(dh, q)
    if joint == 6:
        assert ref.margins(dh, rob._base, rob._tool, T, q[:, 6], 0)[3].max() <= 1e-14  # h at rounding
    reached = np.zeros(len(q), bool)
    for code in range(8):
        qs, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q[:, 6], code)
        if ok.any():
            assert np.abs(ref.fk_mdh(rob, qs[ok]) - T[ok]).max() <= 1e-12
        reached |= ok & (codes & 2 == code & 2)
    assert reached.all()


def test_restatement_marks_unreachable_poses_and_bad_q7():
    rob = rtb.models.PandaMDH()
    dh = ref.dh_table(rob)
    T = np.tile(ref.fk_mdh(rob, rob.qr)[0], (4, 1, 1))
    T[1, :3, 3] = (2.0, 0.5, 0.5)  # beyond the stretched arm: |C / rho| > 1
    q7 = np.array([0.3, 0.3, np.nan, np.inf])
    for code in range(8):
        q, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q7, code)
        assert ok[1:].tolist() == [False, False, False]
        assert np.isnan(q[1:]).all()


def _prismatic():
    L = [rtb.RevoluteMDH(d=x[0], a=x[1], alpha=x[2]) for x in PANDA_DH]
    L[2] = rtb.PrismaticMDH(a=PANDA_DH[2, 1], alpha=PANDA_DH[2, 2])
    return rtb.DHRobot(L)


def _sdh():
    return rtb.DHRobot([rtb.RevoluteDH(d=x[0], a=x[1], alpha=x[2]) for x in PANDA_DH])


def _flipped():
    return rtb.DHRobot([rtb.RevoluteMDH(d=x[0], a=x[1], alpha=x[2], flip=j == 5) for j, x in enumerate(PANDA_DH)])


def _table(dh):
    return lambda: rtb.DHRobot([rtb.RevoluteMDH(d=x[0], a=x[1], alpha=x[2], offset=x[3]) for x in dh])


@pytest.mark.parametrize("make,msg", [
    (rtb.models.UR10, "ikine_panda: the closed form serves 7-joint arms; this robot has 6 joints"),
    (_sdh, "ikine_panda: the closed form serves modified DH; this robot uses standard DH"),
    (_prismatic, "ikine_panda: joint 3 is prismatic"),
    (_flipped, "ikine_panda: joint 6 is flipped"),
    (_table(_dh(alpha4=-h)), "b2k_ikine_panda: not a Panda-type arm: alpha4 must be +pi/2"),
    (_table(_dh(a4=0.0, d3=0.0)), "hypot(a4, d3) must not be 0"),
    (_table(_dh(d5=np.nan)), "dh[4][0] is not finite"),
])
def test_robots_outside_the_pattern_raise_before_any_device_work(make, msg):
    with pytest.raises(ValueError, match=re.escape(msg)):
        make().ikine_panda(np.eye(4), 0.0)


@pytest.mark.parametrize("config,msg", [
    ("lr", "more than one of 'lr'"),
    ("lux", "bad config specifier 'x'"),
    ([], "ikine_panda: give 1 to 8 configurations, got 0"),
    (["lun"] * 9, "ikine_panda: give 1 to 8 configurations, got 9"),
])
def test_bad_configurations_raise_before_any_device_work(config, msg):
    with pytest.raises(ValueError, match=msg):
        rtb.models.PandaMDH().ikine_panda(np.eye(4), 0.0, config=config)
