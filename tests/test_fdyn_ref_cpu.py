"""The reference side of the forward-dynamics sweep (tests/fdyn_ref.py), checked without a GPU: it is oracle.fdyn
step for step, its solver counters are right on an ODE with a closed-form solution, and its output grid is
np.arange's."""
import os
import sys

import numpy as np
import pytest

from oracle import chains as ch
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fdyn_ref  # noqa: E402


def puma_accel():
    links = ch.puma560_links()
    for l in links:
        l.update(Tc=[0.0, 0.0])
    L = ch.pack_rne(links)
    rne = lambda q, qd, qdd, g: orc.rne(6, 0, L, -np.asarray(g, dtype=float), q, qd, qdd)  # noqa: E731
    return rne, lambda q, qd, tau: orc.dyn_accel(rne, 6, q, qd, tau, np.array([0, 0, -9.81]))[0]  # noqa: E731


@pytest.mark.parametrize("kw", [dict(), dict(solver_args=dict(rtol=1e-6, atol=1e-9), dt=0.01),
                                dict(solver_args=dict(max_step=0.01, first_step=1e-3), qd0=[0.3, -0.2, 0.1, 0, 0.5, 0])])
def test_helper_equals_oracle_fdyn_bit_for_bit(kw):
    _, acc = puma_accel()
    q0 = np.array([0, np.pi / 4, np.pi, 0, np.pi / 4, 0])
    tau = np.array([5.0, -20.0, 3.0, 0.5, 0.2, 0.1])
    torque = lambda t, q, qd: tau - 2.0 * qd  # noqa: E731
    r = fdyn_ref.fdyn(acc, 6, 0.2, q0, torque=torque, **kw)
    t, q, qd = orc.fdyn(acc, 6, 0.2, q0, torque_fn=torque, **kw)
    for a, b in ((r.t, t), (r.q, q), (r.qd, qd)):
        assert a.shape == b.shape and np.array_equal(a, b)
    if "dt" not in kw:
        assert r.accepted == len(t) - 1 == len(r.steps)
        np.testing.assert_allclose(np.cumsum(r.steps), t[1:], rtol=1e-14, atol=1e-15)


def test_counters_on_a_scalar_linear_ode():
    """y' = -k y, y = exp(-k t): every right-hand-side call is counted here as well, so nfev, accepted and rejected
    are checked against an independent count; a first step the size of the interval must be rejected."""
    k = 40.0
    calls = []

    def rhs(t, y):
        calls.append(t)
        return -k * y

    for sa, want_rejected in ((dict(), False), (dict(first_step=1.0), True), (dict(max_step=0.01), False),
                              (dict(rtol=1e-10, atol=1e-12), False)):  # the others may reject a step too
        calls.clear()
        t, y, nfev, acc, rej, steps = fdyn_ref.rk45(rhs, [1.0], 1.0, sa)
        assert nfev == len(calls) == (1 if "first_step" in sa else 2) + 6 * (acc + rej)
        assert acc == len(steps) == len(t) - 1 and t[-1] == 1.0
        assert rej > 0 or not want_rejected, (sa, rej)
        np.testing.assert_allclose(np.cumsum(steps), t[1:], rtol=1e-14)
        if "max_step" in sa:
            assert steps.max() <= sa["max_step"] * (1 + 1e-12) and acc >= 1.0 / sa["max_step"]  # t - t_old rounds
        tol = sa.get("rtol", 1e-3)
        assert np.abs(y[:, 0] - np.exp(-k * t)).max() < 50 * tol, sa
    # a rejection without first_step: a large initial slope change after the automatic first step
    calls.clear()
    t, y, nfev, acc, rej, _ = fdyn_ref.rk45(lambda t, y: (calls.append(t), -k * y * (1 + 1e3 * (t > 0.05)))[1], [1.0], 0.3)
    assert rej > 0 and nfev == len(calls) == 2 + 6 * (acc + rej)


@pytest.mark.parametrize("T,dt,M", [(0.3, 0.1, 3), (2.1, 0.3, 8), (0.25, 0.02, 13), (0.2, 0.2, 1), (0.2, 0.5, 1)])
def test_grid_follows_arange(T, dt, M):
    r = fdyn_ref.rk45(lambda t, y: -y, [1.0, 2.0], T, dt=dt)
    assert r[0].shape == (M,) and np.array_equal(r[0], np.arange(0, T, dt))
    assert r[0][-1] <= T and r[1].shape == (M, 2)
    ts, ys = fdyn_ref.rk45(lambda t, y: -y, [1.0, 2.0], T)[:2]
    for c in range(2):  # linear interpolation between RK45's accepted steps
        np.testing.assert_allclose(r[1][:, c], np.interp(r[0], ts, ys[:, c]), rtol=1e-14, atol=1e-15)
    assert r[1][0, 1] == 2.0


def test_velocity_sign_helper():
    qd = np.array([[0.5, -1.0], [0.1, -0.2], [0.3, -3.0]])
    assert fdyn_ref.keeps_velocity_signs(qd)
    assert not fdyn_ref.keeps_velocity_signs(np.r_[qd, [[-0.1, -1.0]]])
    assert not fdyn_ref.keeps_velocity_signs(np.r_[[[0.0, -1.0]], qd])
