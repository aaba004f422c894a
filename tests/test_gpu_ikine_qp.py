"""Quadratic-programming IK on the device (b2k_ikine_qp): one step is the exact QP of the restatement in ikine_qp_ref.py
and keeps every damper row, full loops and the two-phase restart kernels report what the sequential restatement
reports, fp32 solves what fp64 solves, and every entry point serves one pose and a batch on host and device."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import oracle as orc  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_qp_ref as ref  # noqa: E402

G = os.path.join(os.path.dirname(__file__), "golden")
PARITY = 0.97  # the bar of the existing IK parity tests (test_gpu_parity.IK_COUNTER_PARITY)
SEM = rtb._lib.SEM_PYTHON


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def run(e, Tep, q0, ilimit, slimit, seed, kj=1.0, ks=1.0, kq=0.0, km=0.0, ps=0.0, pi=0.3, jl=False, tol=1e-6,
        rng_per_row=False, dt=np.float64):
    """per-row (q, success, iterations, searches, residual) of the device solver, on the host"""
    r = e._ik(dev(Tep, dt), None if q0 is None else dev(q0, dt), ilimit, slimit, tol, None, jl, 0.0, 0, seed, SEM,
              rng_per_row, None, qp=e._qp_args(kj, ks, kq, km, ps, pi))
    return tuple(x.cpu().numpy() for x in r[:5])


PANDA = rtb.models.Panda().ets()
CP = orc.Chain(PANDA.describe())
MDH = rtb.models.PandaMDH().ets()  # real joint limits
CM = orc.Chain(MDH.describe())
GAINS = [dict(kq=0.0, km=0.0), dict(kq=1.0, km=0.0), dict(kq=0.0, km=0.5), dict(kq=2.0, km=0.5, kj=0.5, ks=2.0)]


def _near_limits(rng, ql, qh, N):
    n = len(ql)
    side = rng.integers(0, 3, (N, n))
    return np.where(side == 0, ql + rng.uniform(0, 0.3, (N, n)),
                    np.where(side == 1, qh - rng.uniform(0, 0.3, (N, n)), rng.uniform(ql, qh, (N, n))))


def _check_one_step(e, C, q0, Tep, gains, ps=0.05, pi=0.3):
    got = run(e, Tep, q0, 1, 1, 1, ps=ps, pi=pi, tol=1e-300, **gains)
    assert (got[2] == 1).all()
    n = C.n
    kw = dict(kj=1.0, ks=1.0, kq=0.0, km=0.0)
    kw.update(gains)
    active = 0
    for r in range(len(q0)):
        ev = orc.angle_axis(C.fkine(q0[r])[0], Tep[r])
        J = C.jacob0(q0[r])[0]
        want = ref.step(J, ev, q0[r], C.qlim_l, C.qlim_h, kw["kj"], kw["ks"], kw["kq"], kw["km"], ps, np.full(n, pi))
        d = got[0][r] - q0[r]
        np.testing.assert_allclose(d, want, rtol=0, atol=1e-9)
        sgn, bnd = ref.damper(q0[r], C.qlim_l, C.qlim_h, kw["kq"], ps, np.full(n, pi))
        assert (sgn * d - bnd <= 1e-12).all(), (r, sgn * d - bnd)
        active += int(((sgn != 0) & (np.abs(sgn * d - bnd) < 1e-12)).sum())
    return active


@pytest.mark.parametrize("gi", range(len(GAINS)))
def test_one_step_is_the_restated_qp(gi):
    rng = np.random.default_rng(11 + gi)
    N = 128
    q0 = _near_limits(rng, CM.qlim_l, CM.qlim_h, N)
    Tep = CM.fkine(rng.uniform(CM.qlim_l, CM.qlim_h, (N, 7)))
    active = _check_one_step(MDH, CM, q0, Tep, GAINS[gi])
    if GAINS[gi]["kq"] > 0:
        assert active > 10, active  # bounds are active on some rows, so the active-set rounds ran


def _random_chain(n, rng):
    ets = []
    for j in range(n):
        if j % 4 == 3:
            ets.append(rtb.ET.tz(jindex=j, qlim=np.array([-0.4, 0.5])))
        else:
            a = rng.uniform(1.0, 2.8)
            ets.append([rtb.ET.Rz, rtb.ET.Ry, rtb.ET.Rx][j % 3](jindex=j, qlim=np.array([-a, a * rng.uniform(0.6, 1.0)])))
        ets.append(rtb.ET.tx(rng.uniform(0.1, 0.4)))
        ets.append(rtb.ET.tz(rng.uniform(0.05, 0.3)))
    return rtb.ETS(ets)


@pytest.mark.parametrize("n", range(1, 11))
def test_one_step_at_every_joint_count(n):
    rng = np.random.default_rng(100 + n)
    e = _random_chain(n, rng)
    C = orc.Chain(e.describe())
    N = 48
    q0 = _near_limits(rng, C.qlim_l, C.qlim_h, N)
    Tep = C.fkine(rng.uniform(C.qlim_l, C.qlim_h, (N, n)))
    _check_one_step(e, C, q0, Tep, dict(kq=1.0, km=0.0))
    if n >= 6:
        _check_one_step(e, C, q0, Tep, dict(kq=1.0, km=0.5, kj=0.7))


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
    for gains in (dict(kq=1.0, km=0.0), dict(kq=2.0, km=0.5)):
        q, s, it, sr, E = run(MDH, Tep, q0, 30, 1, 3, ps=0.0, pi=0.3, jl=True, **gains)
        want = ref.solve(CM, Tep[rows], q0[rows], 30, 1, 1e-6, True, None, 3, ps=0.0, pi=0.3, **gains)
        same = (s[rows] == want[1]) & (it[rows] == want[2]) & (sr[rows] == want[3])
        assert same.mean() >= PARITY, (gains, N, same.mean())
        ok = same & (want[1] == 1)
        np.testing.assert_allclose(q[rows][ok], want[0][ok], rtol=0, atol=1e-6)


@pytest.mark.parametrize("slimit,ilimit", [(3, 30), (20, 30)])
def test_two_phase_restarts_report_the_sequential_counters(slimit, ilimit):
    z = np.load(os.path.join(G, "panda_ik.npz"))
    Tep = np.tile(z["Tep"], (8, 1, 1))  # 1536 targets: N >= 1024 with restarts runs the two-phase kernels
    q, s, it, sr, E = run(PANDA, Tep, None, ilimit, slimit, 21, kq=1.0, km=0.5, jl=True, rng_per_row=True)
    hard = np.flatnonzero((sr > 1) | (s == 0))
    assert hard.size > 20
    easy = np.setdiff1d(np.arange(len(Tep)), hard)
    rows = np.union1d(hard[:150], np.random.default_rng(0).choice(easy, min(100, easy.size), replace=False))
    want = ref.solve(CP, Tep, None, ilimit, slimit, 1e-6, True, None, 21, rng_per_row=True, rows=rows, kq=1.0, km=0.5,
                     ps=0.0, pi=0.3)
    same = (s[rows] == want[1]) & (it[rows] == want[2]) & (sr[rows] == want[3])
    assert same.mean() >= PARITY, same.mean()
    assert same[np.isin(rows, hard)].mean() >= PARITY


def test_fp32_outcomes():
    rng = np.random.default_rng(2)
    Tep = CP.fkine(rng.uniform(-np.pi, np.pi, (20000, 7)))  # config 4's targets
    # with 30 iterations per search the QP step itself leaves about 1 % (no terms) and 25 % (both terms) of these
    # targets unsolved in fp64 too (its damping kj sum|e| / ks is heavy far from a target): fp32 is held to fp64's rate
    for gains, floor in ((dict(), 0.95), (dict(kq=1.0, km=0.5), 0.7)):
        q, s, it, sr, E = run(PANDA, Tep, None, 30, 100, 5, jl=True, dt=np.float32, **gains)
        s64 = run(PANDA, Tep, None, 30, 100, 5, jl=True, **gains)[1]
        assert s.mean() > floor and abs(s.mean() - s64.mean()) < 0.01, (gains, s.mean(), s64.mean())
        ok = s == 1
        err = np.abs(CP.fkine(q[ok].astype(np.float64)) - Tep[ok]).max(axis=(1, 2))
        assert np.percentile(err, 99) < 5e-3, np.percentile(err, 99)


def test_every_entry_point_takes_one_pose_and_a_batch_on_host_and_device():
    rng = np.random.default_rng(3)
    qs = rng.uniform(CM.qlim_l, CM.qlim_h, (64, 7))
    Tep = CM.fkine(qs)
    panda, pmdh = rtb.models.Panda(), rtb.models.PandaMDH()
    calls = [
        ("ets", lambda T, **k: MDH.ikine_QP(T, **k)),
        ("robot", lambda T, **k: panda.ikine_QP(T, **k)),
        ("robot_end", lambda T, **k: panda.ikine_QP(T, end=panda.ee_links[0], start=panda.base_link, **k)),
        ("dhrobot", lambda T, **k: pmdh.ikine_QP(T, **k)),
        ("solver", lambda T, **k: rtb.IK_QP(kq=1.0, km=0.5, **k).solve(MDH, T)),
    ]
    for name, f in calls:
        T = Tep if name not in ("robot", "robot_end") else CP.fkine(qs)
        for host in (True, False):
            Tb = T if host else dev(T)
            sol = f(Tb, seed=1)
            assert isinstance(sol, rtb.IKSolution) and np.asarray(sol.q).shape == (64, 7), name
            assert sol.searches >= 64 and sol.iterations >= 64
            one = f(Tb[0], seed=1)
            assert isinstance(one, rtb.IKSolution) and np.asarray(one.q).shape == (7,), name
            assert one.success in (True, False)
    # DHRobot gains ikine_NR / ikine_GN delegations alongside ikine_QP
    assert pmdh.ikine_NR(Tep[:8], seed=1).q.shape == (8, 7)
    assert pmdh.ikine_GN(Tep[:8], seed=1).q.shape == (8, 7)
