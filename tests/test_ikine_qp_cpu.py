"""Quadratic-programming IK step (ikine_QP) without a GPU: the exact QP of the restatement in ikine_qp_ref.py -- the
specification the kernel is checked against -- is pinned to scipy's bounded least squares and to the KKT conditions,
reduces to the oracle's Wampler LM step without bounds or manipulability term, and the C ABI and the Python layer
reject bad arguments before any CUDA call."""
import os
import sys

import numpy as np
import pytest
from scipy.optimize import lsq_linear

import b2kin as rtb
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_qp_ref as ref  # noqa: E402

lib = rtb._lib.lib()
PANDA = rtb.models.Panda().ets()
MDH = rtb.models.PandaMDH().ets()  # real joint limits
UR10 = rtb.models.UR10().ets()
PUMA = rtb.models.Puma560().ets()
CM = orc.Chain(MDH.describe())
SHORT = rtb.ETS([rtb.ET.Rz(jindex=0), rtb.ET.tx(0.5), rtb.ET.Rz(jindex=1), rtb.ET.tx(0.3)])  # kept alive: its chain handle


def kkt_residual(H, r, sgn, bnd, x):
    """largest violation of primal feasibility, dual feasibility, stationarity and complementarity, relative to the
    size of the terms"""
    g = H @ x - r
    mu = np.where(sgn != 0, -sgn * g, 0.0)
    act = (sgn != 0) & np.isclose(sgn * x, bnd, rtol=0, atol=1e-12 * (1 + np.abs(bnd)))
    scale = 1.0 + np.abs(r).max() + np.abs(H).max() * np.abs(x).max()
    primal = np.max(np.where(sgn != 0, sgn * x - bnd, 0.0), initial=0.0)
    dual = max(0.0, -np.min(np.where(act, mu, 0.0), initial=0.0))
    stat = np.abs(np.where(act, 0.0, g)).max()  # a free coordinate has zero gradient
    return max(primal, dual, stat / scale)


def lsq(H, r, J, e, w, kj, c, sgn, bnd):
    n = len(r)
    A = np.vstack([np.sqrt(kj) * np.eye(n), np.sqrt(w) * J])
    y = np.concatenate([-c / np.sqrt(kj), np.sqrt(w) * e])
    lb = np.where(sgn < 0, -bnd, -np.inf)
    ub = np.where(sgn > 0, bnd, np.inf)
    return lsq_linear(A, y, bounds=(lb, ub), method="bvls", tol=1e-15, lsmr_tol=None).x


def _instances(count, seed):
    """QP instances of the PandaMDH step from q near the limits: (J, e, q, kj, ks, kq, km, ps, pi)"""
    rng = np.random.default_rng(seed)
    ql, qh = CM.qlim_l, CM.qlim_h
    for _ in range(count):
        side = rng.integers(0, 3, 7)
        q = np.where(side == 0, ql + rng.uniform(0, 0.3, 7), np.where(side == 1, qh - rng.uniform(0, 0.3, 7),
                                                                       rng.uniform(ql, qh)))
        T = CM.fkine(rng.uniform(ql, qh))[0]
        e = orc.angle_axis(CM.fkine(q)[0], T)
        J = CM.jacob0(q)[0]
        kj, ks = rng.uniform(0.2, 3.0, 2)
        kq = rng.choice([0.0, 0.5, 1.0, 4.0])
        km = rng.choice([0.0, 0.5, 2.0])
        yield J, e, q, kj, ks, kq, km, 0.05, np.full(7, 0.3)


def test_qp_step_is_bounded_least_squares_and_meets_kkt():
    active = 0
    for J, e, q, kj, ks, kq, km, ps, pi in _instances(300, 1):
        H, r, sgn, bnd, w = ref.qp_problem(J, e, q, CM.qlim_l, CM.qlim_h, kj, ks, kq, km, ps, pi)
        c = -ref.jacobm_term(J) / km if km > 0 else np.zeros(7)
        x = ref.qp_bounded(H, r, sgn, bnd)
        want = lsq(H, r, J, e, w, kj, c, sgn, bnd)
        np.testing.assert_allclose(x, want, rtol=0, atol=1e-10)
        assert kkt_residual(H, r, sgn, bnd, x) < 1e-12
        active += int(((sgn != 0) & np.isclose(sgn * x, bnd, rtol=0, atol=1e-14)).sum())
    assert active > 50, active  # the instances exercise active bounds, not only the unconstrained solve


def test_qp_solver_on_random_bounded_problems():
    rng = np.random.default_rng(7)
    active = 0
    for _ in range(500):
        n = int(rng.integers(1, 11))
        J = rng.normal(size=(6, n))
        e = rng.normal(size=6) * 0.1
        kj, w = rng.uniform(0.1, 2.0), rng.uniform(0.5, 50.0)
        c = rng.normal(size=n) * rng.choice([0.0, 0.1])
        H = kj * np.eye(n) + w * J.T @ J
        r = w * J.T @ e - c
        sgn = rng.choice([-1.0, 0.0, 1.0], n)
        bnd = rng.uniform(-0.05, 0.1, n) * (sgn != 0)
        x = ref.qp_bounded(H, r, sgn, bnd)
        np.testing.assert_allclose(x, lsq(H, r, J, e, w, kj, c, sgn, bnd), rtol=0, atol=1e-10)
        assert kkt_residual(H, r, sgn, bnd, x) < 1e-12
        active += int(((sgn != 0) & np.isclose(sgn * x, bnd, rtol=0, atol=1e-14)).sum())
    assert active > 200, active


def test_damper_rows_and_the_both_limits_case():
    ql, qh = np.array([-1.0, -1.0, -1.0, -0.1]), np.array([1.0, 1.0, 1.0, 0.15])
    pi = np.full(4, 0.2)
    sgn, bnd = ref.damper(np.array([-0.95, 0.0, 0.9, 0.0]), ql, qh, 2.0, 0.05, pi)
    np.testing.assert_array_equal(sgn, [-1.0, 0.0, 1.0, 1.0])  # joint 3 is within pi of both limits: the upper row wins
    np.testing.assert_allclose(bnd[[0, 2, 3]], [(0.05 - 0.05) / 0.15 / 2, (0.1 - 0.05) / 0.15 / 2,
                                                (0.15 - 0.05) / 0.15 / 2], rtol=1e-12, atol=1e-15)
    assert ref.damper(np.zeros(4), ql, qh, 0.0, 0.05, pi)[0].tolist() == [0.0] * 4  # kq = 0: no rows
    # the both-limits case through the exact QP: an upper bound is active, the lower limit imposes nothing
    H, r = np.eye(1) * 2.0, np.array([1.0])
    x = ref.qp_bounded(H, r, np.array([1.0]), np.array([0.1]))
    assert x[0] == 0.1
    x = ref.qp_bounded(H, -r, np.array([1.0]), np.array([0.1]))
    assert x[0] == -0.5


def test_without_bounds_or_manipulability_one_step_is_wamplers_lm_step():
    rng = np.random.default_rng(3)
    ql, qh = CM.qlim_l, CM.qlim_h
    for row in range(40):
        q0 = rng.uniform(ql, qh)
        T = CM.fkine(rng.uniform(ql, qh))[0]
        kj, ks = rng.uniform(0.2, 3.0, 2)
        e = orc.angle_axis(CM.fkine(q0)[0], T)
        lam = kj * np.abs(e).sum() / ks
        want = CM.ik_lm(T, q0, 1, 1, 1e-300, False, None, lam, "wampler", seed=0, semantics=1, rng_per_row=False)[0][0]
        got = ref.solve_row(CM, T, q0, 1, 1, 1e-300, False, None, 0, 0, kj=kj, ks=ks)[0]
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def test_zero_error_takes_a_zero_step_and_finishes():
    q0 = np.random.default_rng(4).uniform(CM.qlim_l, CM.qlim_h)
    T = CM.fkine(q0)[0]
    q, s, it, sr, E = ref.solve_row(CM, T, q0, 30, 1, 1e-6, True, None, 0, 0, kq=1.0, km=1.0)
    assert E < 1e-20 and s == 1 and it == 1 and sr == 1
    np.testing.assert_allclose(q, q0, rtol=0, atol=1e-12)


def _qp_call(chain=None, dtype=1, N=4, kj=1.0, ks=1.0, kq=1.0, km=0.0, ps=0.0, pi=None, ilimit=30, slimit=1, Tep=8,
             q_out=8, succ=8, its=8, srch=8, res=8, n=7):
    chain = MDH._chain if chain is None else chain
    if pi is None:
        pi = np.full(n, 0.3)
    pi = None if isinstance(pi, str) else np.ascontiguousarray(pi, dtype=np.float64)
    rc = lib.b2k_ikine_qp(chain, dtype, Tep, N, None, ilimit, slimit, 1e-6, 1, None, 0, 0, kj, ks, kq, km, ps,
                          rtb._lib.dptr(pi), q_out, succ, its, srch, res, None)
    return rc, lib.b2k_last_error().decode()


def _pi_with(i, v):
    p = np.full(7, 0.3)
    p[i] = v
    return p


@pytest.mark.parametrize("kw,msg", [
    (dict(chain=0), "chain handle is NULL"),
    (dict(dtype=2), "dtype must be"),
    (dict(N=-1), "N is negative"),
    (dict(ilimit=0), "ilimit and slimit"),
    (dict(slimit=0), "ilimit and slimit"),
    (dict(kj=0.0), "kj and ks must be > 0"),
    (dict(ks=-1.0), "kj and ks must be > 0"),
    (dict(kj=np.nan), "must be finite"),
    (dict(ks=np.inf), "must be finite"),
    (dict(kq=np.nan), "must be finite"),
    (dict(km=-np.inf), "must be finite"),
    (dict(ps=np.nan), "must be finite"),
    (dict(pi="null"), "pi is NULL"),
    (dict(pi=_pi_with(3, np.inf)), "pi[3] is not finite"),
    (dict(ps=0.3), "ps == pi[0]"),
    (dict(ps=0.1, pi=_pi_with(6, 0.1)), "ps == pi[6]"),
    (dict(chain=PUMA._chain, km=1.0, kq=0.0, n=6, N=0, Tep=None), None),  # n = 6 is enough for the term
    (dict(chain=SHORT._chain, km=1.0, kq=0.0, n=2), "km > 0 needs"),
    (dict(Tep=None), "Tep is NULL"),
    (dict(q_out=None), "q_out is NULL"),
    (dict(res=None), "residual is NULL"),
])
def test_entry_rejects_bad_arguments_before_launching(kw, msg):
    rc, err = _qp_call(**kw)
    if msg is None:
        assert rc == 0, err
        return
    assert rc == -1
    assert msg in err, err


def test_entry_accepts_what_it_documents_without_work():
    assert _qp_call(N=0)[0] == 0
    assert _qp_call(N=0, kq=0.0, ps=0.3)[0] == 0           # ps == pi is harmless without the damper
    assert _qp_call(N=0, kq=0.0, pi="null")[0] == 0        # pi is read only with the damper
    assert _qp_call(N=0, kq=-1.0, km=-1.0)[0] == 0         # gains <= 0 switch the terms off
    assert _qp_call(N=0, Tep=None, q_out=None, succ=None, its=None, srch=None, res=None)[0] == 0


@pytest.mark.parametrize("call", ["ets", "solver", "robot", "dhrobot"])
def test_python_layer_rejects_bad_arguments(call):
    T = np.eye(4)

    def go(**kw):
        if call == "ets":
            return MDH.ikine_QP(T, **kw)
        if call == "solver":
            return rtb.IK_QP(**kw).solve(MDH, T)
        if call == "robot":
            return rtb.models.Panda().ikine_QP(T, **kw)
        return rtb.models.PandaMDH().ikine_QP(T, **kw)

    for kw, msg in ((dict(kj=0.0), "kj and ks must be > 0"), (dict(ks=-2.0), "kj and ks must be > 0"),
                    (dict(kq=np.nan), "must be finite"), (dict(pi=np.inf), "must be finite"),
                    (dict(kq=1.0, ps=0.3, pi=0.3), "ps == pi"), (dict(pi=np.full(8, 0.3)), "pi must be a scalar"),
                    (dict(km=np.inf), "must be finite")):
        with pytest.raises(ValueError, match=msg):
            go(**kw)


def test_python_layer_rejects_manipulability_on_short_chains():
    with pytest.raises(ValueError, match="km > 0 needs at least 6 joints"):
        SHORT.ikine_QP(np.eye(4), km=1.0)
    assert PUMA._qp_args(1.0, 1.0, 0.0, 1.0, 0.0, 0.3)[3] == 1.0  # n = 6 passes


def test_python_layer_normalises_arguments():
    kj, ks, kq, km, ps, pi = MDH._qp_args(2, 3, 0, 0, 0, 0.25)
    assert (kj, ks, kq, km, ps) == (2.0, 3.0, 0.0, 0.0, 0.0) and pi.shape == (7,) and (pi == 0.25).all()
    assert (MDH._qp_args(1.0, 1.0, 1.0, 0.0, 0.0, np.arange(1.0, 8.0))[5] == np.arange(1.0, 8.0)).all()
    s = rtb.IK_QP(kj=0.5, ks=2.0)
    assert s.name == "QP (kj=0.5, ks=2.0)"
    assert hasattr(rtb.DHRobot, "ikine_NR") and hasattr(rtb.DHRobot, "ikine_GN") and hasattr(rtb.DHRobot, "ikine_QP")
