"""Closed-form inverse kinematics (DHRobot.ikine_a) without a GPU: the C ABI rejects bad arguments and robots outside the
Puma link pattern before any CUDA call, config_validate follows the reference's rules, and the numpy restatement in
ikine_a_ref.py -- the specification the kernel is checked against -- is pinned by round trips through the oracle's
forward kinematics and by the configuration predicates."""
import os
import sys

import numpy as np
import pytest

import b2kin as rtb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_a_ref as ref  # noqa: E402

lib = rtb._lib.lib()
PUMA_DH = ref.dh_table(rtb.models.Puma560())


def _call(dtype=1, dh=PUMA_DH, base=None, tool=None, T=8, N=4, nconf=1, conf=(0,), q=8, ok=8):
    dh = None if dh is None else np.ascontiguousarray(dh, dtype=np.float64)
    c = None if conf is None else np.ascontiguousarray(conf, dtype=np.int32)
    rc = lib.b2k_ikine_6s(dtype, rtb._lib.dptr(dh), rtb._lib.dptr(base), rtb._lib.dptr(tool), T, N, nconf,
                          None if c is None else c.ctypes.data_as(rtb._lib.ip), q, ok, None)
    return rc, lib.b2k_last_error().decode()


def _dh(**changes):
    """the Puma560 table with entries replaced: key '<name><link>' with name in d, a, alpha, off and link 1..6"""
    dh = PUMA_DH.copy()
    for key, v in changes.items():
        name, link = key[:-1], int(key[-1])
        dh[link - 1, {"d": 0, "a": 1, "alpha": 2, "off": 3}[name]] = v
    return dh


h = np.pi / 2


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=2), "bad dtype"),
    (dict(N=-1), "bad N"),
    (dict(nconf=0), "nconf must be 1..8"),
    (dict(nconf=9, conf=range(9)), "nconf must be 1..8"),
    (dict(conf=(8,)), "configuration code 8"),
    (dict(nconf=2, conf=(0, -1)), "configuration code -1 of slot 1"),
    (dict(dh=None), "dh and conf must not be NULL"),
    (dict(conf=None), "dh and conf must not be NULL"),
    (dict(T=None), "T, q and ok must not be NULL"),
    (dict(q=None), "T, q and ok must not be NULL"),
    (dict(ok=None), "T, q and ok must not be NULL"),
    (dict(dh=_dh(d2=np.nan)), "dh[1][0] is not finite"),
    (dict(dh=_dh(alpha1=-h)), "alpha1 must be +pi/2"),
    (dict(dh=_dh(a1=0.1)), "a1 must be 0"),
    (dict(dh=_dh(alpha2=0.3)), "alpha2 must be 0"),
    (dict(dh=_dh(a2=0.0)), "a2 must not be 0"),
    (dict(dh=_dh(alpha3=h)), "alpha3 must be -pi/2"),
    (dict(dh=_dh(alpha4=0.5)), "alpha4 must be +pi/2 or -pi/2"),
    (dict(dh=_dh(a4=0.01)), "a4 must be 0"),
    (dict(dh=_dh(alpha5=h)), "alpha5 must be -alpha4"),
    (dict(dh=_dh(a5=0.01)), "a5 must be 0"),
    (dict(dh=_dh(d5=0.01)), "d5 must be 0"),
    (dict(dh=_dh(alpha1=h + 2e-9)), "alpha1 must be +pi/2"),
    # the first six links of PandaMDH read as a standard-DH table
    (dict(dh=ref.dh_table(rtb.models.PandaMDH())[:6]), "alpha1 must be +pi/2"),
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
    assert _call(N=0, dh=_dh(alpha4=-h, alpha5=h, alpha1=h + 5e-10, d1=1, d2=0.3, a3=-0.2, d6=0.1, a6=0.05, alpha6=1.0,
                             off1=0.3, off5=-2))[0] == 0


def test_config_validate():
    cv = rtb.DHRobot.config_validate
    L = ("lr", "ud", "nf")
    assert cv("", L) == "lun"
    assert cv("r", L) == "run"
    assert cv("fd", L) == "ldf"
    assert cv("rdf", L) == "rdf"
    assert rtb.models.Puma560().config_validate("u", L) == "lun"
    for bad in ("lr", "lud", "nfu", "x", "lux", "L"):
        with pytest.raises(ValueError):
            cv(bad, L)


def _robots():
    rng = np.random.default_rng(2024)
    return [rtb.models.Puma560()] + [ref.random_robot(rtb, rng, s) for s in (1, -1) * 10]


@pytest.mark.parametrize("k", range(21))
def test_restatement_round_trips_and_keeps_its_letters(k):
    rob = _robots()[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(100 + k)
    q = rng.uniform(-np.pi, np.pi, (2000, 6))
    T = ref.fk(rob, q)
    for code in range(8):
        qs, ok = ref.ikine_a(dh, rob._base, rob._tool, T, code)
        assert ok.all()
        assert np.abs(ref.fk(rob, qs) - T).max() <= 1e-12, (code, np.abs(ref.fk(rob, qs) - T).max())
        assert set(ref.config_of(dh, qs)) == {ref.letters_of(code)}
    # the solution of the configuration q* has is q* itself, away from the wrist singularity
    letters = np.array(ref.config_of(dh, q))
    keep = np.abs(np.sin(q[:, 4] + dh[4, 3])) > 1e-3
    for code in range(8):
        sel = (letters == ref.letters_of(code)) & keep
        if sel.any():
            qs, ok = ref.ikine_a(dh, rob._base, rob._tool, T[sel], code)
            assert np.abs(ref.wrap(qs - q[sel])).max() <= 1e-9


def test_reference_literal_qn_lun():
    """the reference's own ikine_a test: fkine(ikine_a(fkine(qn), "lun").q) == fkine(qn)"""
    p = rtb.models.Puma560()
    dh = ref.dh_table(p)
    T = ref.fk(p, p.qn)
    q, ok = ref.ikine_a(dh, p._base, p._tool, T, "lun")
    assert ok.all()
    np.testing.assert_allclose(ref.fk(p, q), T, atol=1e-12)
    assert ref.config_of(dh, p.qn) == ["ruf"]


def test_restatement_marks_both_kinds_of_unreachable_pose():
    p = rtb.models.Puma560()
    dh = ref.dh_table(p)
    T = np.tile(np.eye(4), (3, 1, 1))
    T[0, :3, 3] = (0.5, 0.2, 0.3)   # reachable
    T[1, :3, 3] = (0.05, 0.0, 0.67)  # on the shoulder axis: r < |D|
    T[2, :3, 3] = (2.0, 0.0, 0.67)   # beyond the stretched arm: |c| > 1
    for code in range(8):
        q, ok = ref.ikine_a(dh, p._base, p._tool, T, code)
        assert ok.tolist() == [True, False, False]
        assert np.isfinite(q[0]).all() and np.isnan(q[1:]).all()


def _prismatic():
    L = [rtb.RevoluteDH(d=x[0], a=x[1], alpha=x[2]) for x in PUMA_DH]
    L[2] = rtb.PrismaticDH(a=PUMA_DH[2, 1], alpha=PUMA_DH[2, 2])
    return rtb.DHRobot(L)


def _mdh():
    return rtb.DHRobot([rtb.RevoluteMDH(d=x[0], a=x[1], alpha=x[2]) for x in PUMA_DH])


def _alpha3_plus():
    return rtb.DHRobot([rtb.RevoluteDH(d=x[0], a=x[1], alpha=(h if j == 2 else x[2])) for j, x in enumerate(PUMA_DH)])


@pytest.mark.parametrize("make,msg", [
    (rtb.models.UR10, "alpha3 must be -pi/2"),
    (rtb.models.PandaMDH, "7 joints"),
    (_mdh, "modified DH"),
    (_prismatic, "joint 3 is prismatic"),
    (_alpha3_plus, "alpha3 must be -pi/2"),
])
def test_robots_outside_the_pattern_raise_before_any_device_work(make, msg):
    rob = make()
    with pytest.raises(ValueError, match=msg):
        rob.ikine_a(np.eye(4))
    with pytest.raises(ValueError):
        rtb.models.Puma560().ikine_a(np.eye(4), config="lr")
