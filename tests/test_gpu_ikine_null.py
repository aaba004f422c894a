"""Null-space terms of the Python IK solvers on the device (b2k_ikine_null): one step pins the term itself, full loops
and the two-phase restart kernels report what the sequential restatement in ikine_null_ref.py reports, the terms do
what they are for, and every path without them is unchanged."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import oracle as orc  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_null_ref as ref  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")
PARITY = 0.97  # the bar of the existing IK parity tests (test_gpu_parity.IK_COUNTER_PARITY)
SEM = rtb._lib.SEM_PYTHON


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def run(e, Tep, q0, ilimit, slimit, k, method, seed, kq=0.0, km=0.0, ps=0.0, pi=0.3, jl=False, rng_per_row=True,
        dt=np.float64):
    """per-row (q, success, iterations, searches, residual) of the device solver, on the host"""
    r = e._ik(dev(Tep, dt), None if q0 is None else dev(q0, dt), ilimit, slimit, 1e-6, None, jl, k, method, seed, SEM,
              rng_per_row, None, null=e._null_args(kq, km, ps, pi))
    return tuple(x.cpu().numpy() for x in r[:5])


PANDA = rtb.models.Panda().ets()
CP = orc.Chain(PANDA.describe())
MDH = rtb.models.PandaMDH().ets()  # real joint limits
CM = orc.Chain(MDH.describe())
STEPS = [("chan", 1.0), ("wampler", 1.0), ("sugihara", 1.0), (rtb._lib.IK_NR, 0.0), (rtb._lib.IK_GN, 0.0)]
TERMS = [(1.0, 0.0), (0.0, 1.0), (2.0, 0.5)]


@pytest.mark.parametrize("method,k", STEPS)
def test_one_step_adds_the_restated_qnull(method, k):
    rng = np.random.default_rng(11)
    N = 64
    ql, qh = CM.qlim_l, CM.qlim_h
    q0 = rng.uniform(ql, qh, (N, 7))  # many joints inside the 0.3 rad band of a limit
    Tep = CM.fkine(rng.uniform(ql, qh, (N, 7)))
    base = run(MDH, Tep, q0, 1, 1, k, method, 1)
    for kq, km in TERMS:
        got = run(MDH, Tep, q0, 1, 1, k, method, 1, kq=kq, km=km, ps=0.05, pi=0.3)
        assert (got[2] == base[2]).all()
        d = got[0] - base[0]
        for r in range(N):
            J = CM.jacob0(q0[r])[0]
            want = ref.qnull(J, q0[r], ql, qh, kq, km, 0.05, np.full(7, 0.3))
            np.testing.assert_allclose(d[r], want, rtol=0, atol=1e-9)
            assert np.linalg.norm(J @ d[r]) <= 1e-9 * max(1.0, np.linalg.norm(d[r]))


@pytest.mark.parametrize("N", [1, 33, 1000, 100001])
def test_full_loop_matches_the_restatement(N):
    rng = np.random.default_rng(N)
    ql, qh = CM.qlim_l, CM.qlim_h
    qs = rng.uniform(ql, qh, (N, 7))
    Tep = CM.fkine(qs)
    q0 = np.clip(qs + rng.normal(0, 0.4, (N, 7)), ql, qh)
    rows = np.arange(N) if N <= 1000 else np.sort(rng.choice(N, 300, replace=False))
    if N == 1000:
        rows = rows[::4]
    for method, k, kq, km in (("chan", 1.0, 2.0, 0.5), (rtb._lib.IK_NR, 0.0, 1.0, 0.0)):
        q, s, it, sr, E = run(MDH, Tep, q0, 30, 1, k, method, 3, kq=kq, km=km, ps=0.0, pi=0.3, jl=True)
        want = ref.solve(CM, Tep[rows], q0[rows], 30, 1, 1e-6, True, None, k, method, 3, kq=kq, km=km, ps=0.0, pi=0.3)
        same = (s[rows] == want[1]) & (it[rows] == want[2]) & (sr[rows] == want[3])
        assert same.mean() >= PARITY, (method, N, same.mean())
        ok = same & (want[1] == 1)
        np.testing.assert_allclose(q[rows][ok], want[0][ok], rtol=0, atol=1e-6)


@pytest.mark.parametrize("slimit,ilimit", [(3, 10), (20, 15)])
def test_two_phase_restarts_report_the_sequential_counters(slimit, ilimit):
    z = np.load(os.path.join(G, "panda_ik.npz"))
    Tep = np.tile(z["Tep"], (8, 1, 1))  # 1536 targets: N >= 1024 with restarts runs the two-phase kernels
    q, s, it, sr, E = run(PANDA, Tep, None, ilimit, slimit, 1.0, "chan", 21, kq=2.0, km=0.5, jl=True)
    hard = np.flatnonzero((sr > 1) | (s == 0))
    assert hard.size > 20
    easy = np.setdiff1d(np.arange(len(Tep)), hard)
    rows = np.union1d(hard[:250], np.random.default_rng(0).choice(easy, 100, replace=False))
    want = ref.solve(CP, Tep, None, ilimit, slimit, 1e-6, True, None, 1.0, "chan", 21, rows=rows, kq=2.0, km=0.5, ps=0.0,
                     pi=0.3)
    same = (s[rows] == want[1]) & (it[rows] == want[2]) & (sr[rows] == want[3])
    assert same.mean() >= PARITY, same.mean()
    assert same[np.isin(rows, hard)].mean() >= PARITY


def _purpose_run(kq, km):
    rng = np.random.default_rng(5)
    N = 4000
    ql, qh = CM.qlim_l, CM.qlim_h
    Tep = CM.fkine(rng.uniform(ql, qh, (N, 7)))
    side = rng.integers(0, 2, (N, 7))
    q0 = np.where(side == 0, ql + 0.05 * (qh - ql), qh - 0.05 * (qh - ql))  # every joint starts near a limit
    q, s, it, sr, E = run(MDH, Tep, q0, 30, 5, 1.0, "chan", 3, kq=kq, km=km, ps=0.0, pi=0.3, jl=True)
    ok = s == 1
    assert ok.mean() > 0.6
    err = np.abs(CM.fkine(q[ok]) - Tep[ok]).max(axis=(1, 2))
    # E < tol was tested BEFORE the last step (IK.py); the returned q is one step later, and a null-space step is only
    # null to first order, so a few rows move off the pose by more: the bar is on the 99th percentile
    assert np.percentile(err, 99) < 5e-3, np.percentile(err, 99)
    return q[ok]


def test_joint_limit_term_keeps_solutions_away_from_the_limits():
    ql, qh = CM.qlim_l, CM.qlim_h
    dist = [np.median(np.minimum(q - ql, qh - q)) for q in (_purpose_run(0.0, 0.0), _purpose_run(2.0, 0.0))]
    assert dist[1] > dist[0], dist


def test_manipulability_term_raises_manipulability():
    man = [np.mean([orc.yoshikawa(CM.jacob0(x)[0]) for x in q]) for q in (_purpose_run(0.0, 0.0), _purpose_run(0.0, 0.2))]
    assert man[1] > man[0], man


def test_fp32_outcomes():
    rng = np.random.default_rng(2)
    Tep = CP.fkine(rng.uniform(-np.pi, np.pi, (20000, 7)))
    q, s, it, sr, E = run(PANDA, Tep, None, 30, 100, 1.0, "chan", 5, kq=2.0, km=0.5, jl=True, rng_per_row=False,
                          dt=np.float32)
    assert s.mean() > 0.99, s.mean()
    ok = s == 1
    err = np.abs(CP.fkine(q[ok].astype(np.float64)) - Tep[ok]).max(axis=(1, 2))
    assert np.percentile(err, 99) < 5e-3, np.percentile(err, 99)


def test_paths_without_the_terms_are_unchanged():
    rng = np.random.default_rng(9)
    Tep = CP.fkine(rng.uniform(-2.5, 2.5, (1500, 7)))
    base = PANDA.ikine_LM(Tep, seed=4)
    for kq, km in ((0.0, 0.0), (-1.0, 0.0), (0.0, -2.0), (-1.0, -1.0)):
        sol = PANDA.ikine_LM(Tep, seed=4, kq=kq, km=km, ps=0.1, pi=0.2)
        assert np.array_equal(sol.q, base.q) and sol.iterations == base.iterations and sol.searches == base.searches
    for robot in (rtb.models.UR10(), rtb.models.Puma560()):
        e = robot.ets()
        T6 = e.eval(rng.uniform(-2, 2, (300, 6)))
        base = e.ikine_LM(T6, seed=4)
        for meth in ("ikine_LM", "ikine_NR", "ikine_GN"):
            b = getattr(e, meth)(T6, seed=4)
            sol = getattr(e, meth)(T6, seed=4, kq=1.0, km=1.0)
            assert np.array_equal(sol.q, b.q) and sol.iterations == b.iterations
        assert np.array_equal(e.ikine_LM(T6, seed=4, kq=1.0, km=1.0).q, base.q)


def test_entry_points_run_with_the_terms():
    rng = np.random.default_rng(3)
    qs = rng.uniform(CM.qlim_l, CM.qlim_h, (200, 7))
    Tep = CM.fkine(qs)
    for solver in (rtb.IK_LM(kq=2.0, km=0.5, seed=1), rtb.IK_NR(kq=2.0, seed=1), rtb.IK_GN(km=0.5, seed=1)):
        sol = solver.solve(MDH, Tep)
        assert isinstance(sol, rtb.IKSolution) and sol.q.shape == (200, 7)
        sol = solver.solve(MDH, Tep[0])
        assert isinstance(sol, rtb.IKSolution) and sol.q.shape == (7,)
    sol = rtb.models.PandaMDH().ikine_LM(Tep[:50], kq=2.0, km=0.5, seed=2)
    assert isinstance(sol, rtb.IKSolution) and sol.q.shape == (50, 7)
    panda = rtb.models.Panda()  # a Robot: ikine_LM over the chain it extracts
    sol = panda.ikine_LM(CP.fkine(qs[:50]), kq=2.0, km=0.5, seed=2)
    assert isinstance(sol, rtb.IKSolution) and sol.q.shape == (50, 7)
