"""Pins the one-step IK reference of tests/ik_lm_ref.py (no GPU needed): the mpmath steps against numpy's fp64 solvers,
and against one step of the compiled oracle's own solver loop (ilimit = slimit = 1, Python semantics, which returns
exactly q0 + dq), at n = 1..10 on DH-like, generic and random chains with prismatic joints.  The masked Gauss-Newton
rows at n = 4 and 5 (fewer weighted rows than joints) check that the oracle's truncated SVD takes the minimum-norm step."""
import numpy as np
import pytest

from oracle import chains as ch
from oracle import oracle as orc

import fkj_ref as FR
import ik_lm_ref as R

WEIGHTS = {"unit": np.ones(6), "mask": np.array([1, 1, 1, 0, 0, 0.0]), "wts": np.array([1, 1, 1, 0.3, 0.3, 0.3])}
LAMBDA = {"chan": 1.0, "wampler": 0.05, "sugihara": 0.05, "nr": 0.1, "nr0": 0.0, "gn": 0.0}


def chains(n, seed):
    """(name, description) of a DH-like, a generic and a random chain (prismatic joints, flips) of n joints."""
    rng = np.random.default_rng(seed)
    kinds = list(rng.permutation(FR.ALL_KINDS))
    return [("dh", FR.dh_family(n, rng)), ("gen", FR.generic_family(n, rng, kinds)),
            ("rand", ch.random_chain(rng, n_joints=n))]


def problems(C, rows, rng, spread=0.3):
    """(q0, Tep): targets from random in-limit configurations, starts a random distance away from them."""
    lo, hi = C.qlim_l, C.qlim_h
    qt = lo + (hi - lo) * rng.uniform(0.1, 0.9, (rows, C.n))
    q0 = qt + rng.normal(0.0, spread, qt.shape) * (hi - lo) / 4
    return q0, C.fkine(qt)


def meth(tag):
    return "nr" if tag == "nr0" else tag


@pytest.mark.parametrize("n", range(1, 11))
def test_lm_step_matches_fp64_solve(n):
    rng = np.random.default_rng(100 + n)
    checked = 0
    for name, desc in chains(n, n):
        C = orc.Chain(desc)
        q0, Tep = problems(C, 3, rng)
        for wname, we in WEIGHTS.items():
            for m in ("chan", "wampler", "sugihara"):
                lam = LAMBDA[m]
                for q, T in zip(q0, Tep):
                    e, E, dq = R.step(C, q, T, m, lam, we)
                    J = C.jacob0(q[None])[0]
                    wn = {"chan": lam * E, "wampler": lam, "sugihara": E + lam}[m]
                    if not R.cond(J, E, m, lam, we) < 1e6:
                        continue
                    A = J.T @ (we[:, None] * J) + wn * np.eye(n)
                    ref = np.linalg.solve(A, J.T @ (we * e))
                    checked += 1
                    np.testing.assert_allclose(dq, ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max(),
                                               err_msg=f"{name} n={n} {m} {wname}")
                    assert E == pytest.approx(0.5 * float(e @ (we * e)), rel=1e-15)
    assert checked >= 0.9 * 3 * 3 * 3 * 3, checked


@pytest.mark.parametrize("n", range(1, 11))
def test_pinv_steps_match_numpy_pinv(n):
    rng = np.random.default_rng(200 + n)
    for name, desc in chains(n, 50 + n):
        C = orc.Chain(desc)
        q0, Tep = problems(C, 2, rng)
        for wname, we in WEIGHTS.items():
            for tag in ("nr", "nr0", "gn"):
                m, d = meth(tag), LAMBDA[tag]
                for q, T in zip(q0, Tep):
                    e, E, dq = R.step(C, q, T, m, d, we)
                    J = C.jacob0(q[None])[0]
                    if m == "gn":
                        ws = np.sqrt(we)
                        ref = np.linalg.pinv(ws[:, None] * J, rcond=R.EPS * max(6, n)) @ (ws * e)
                    elif d > 0:
                        U, s, Vt = np.linalg.svd(J, full_matrices=False)
                        ref = Vt.T @ ((s / (s * s + d * d)) * (U.T @ e))
                    else:
                        ref = np.linalg.pinv(J, rcond=0.0) @ e
                    c = R.cond(J, E, m, d, we)
                    if c < 1e8:
                        np.testing.assert_allclose(dq, ref, rtol=0, atol=max(1.0, np.abs(ref).max()) * 1e-16 * c * 10,
                                                   err_msg=f"{name} n={n} {tag} {wname} cond {c:.1e}")


def _oracle_one_step(C, q0, Tep, tag, we):
    """One step of the oracle's own loop: Python semantics with ilimit = slimit = 1 returns q0 + dq (q0 where the
    step is refused)."""
    q, s, it, sr, E = C.ik_lm(Tep, q0=q0, ilimit=1, slimit=1, tol=1e-300, joint_limits=False, mask=we,
                              k=LAMBDA[tag], method=meth(tag), seed=0, semantics=1, rng_per_row=True)
    assert (it == 1).all() and (sr == 1).all()
    return q - q0, E, s == 0  # a row met at q0 (E = 0 under a mask) is wrapped, not stepped


@pytest.mark.parametrize("n", range(1, 11))
def test_every_rule_matches_one_oracle_step(n):
    rng = np.random.default_rng(300 + n)
    for name, desc in chains(n, 80 + n):
        C = orc.Chain(desc)
        q0, Tep = problems(C, 3, rng)
        for wname, we in WEIGHTS.items():
            for tag in LAMBDA:
                m, lam = meth(tag), LAMBDA[tag]
                got, Eo, stepped = _oracle_one_step(C, q0, Tep, tag, we)
                for r in range(len(q0)):
                    e, E, dq = R.step(C, q0[r], Tep[r], m, lam, we)
                    assert Eo[r] == pytest.approx(E, rel=1e-14, abs=1e-300)
                    if not stepped[r]:
                        continue
                    c = R.cond(C.jacob0(q0[r][None])[0], E, m, lam, we)
                    if c < 1e8:
                        np.testing.assert_allclose(got[r], dq, rtol=0, atol=1e-10 * max(1.0, np.abs(dq).max()),
                                                   err_msg=f"{name} n={n} {tag} {wname} row {r} cond {c:.1e}")


@pytest.mark.parametrize("n", [4, 5])
def test_masked_gn_below_six_joints_is_the_minimum_norm_step(n):
    """A position-only mask leaves three weighted rows: J_w^T J_w is singular for n = 4, 5, and the step must be the
    minimum-norm least-squares solution (the oracle's truncated SVD, the reference's BDCSVD solve)."""
    rng = np.random.default_rng(400 + n)
    we = WEIGHTS["mask"]
    checked = 0
    for name, desc in chains(n, 90 + n):
        C = orc.Chain(desc)
        q0, Tep = problems(C, 8, rng)
        got, _, stepped = _oracle_one_step(C, q0, Tep, "gn", we)
        assert stepped.all()
        for r in range(len(q0)):
            e, E, dq = R.step(C, q0[r], Tep[r], "gn", 0.0, we)
            J = C.jacob0(q0[r][None])[0]
            c = R.cond(J, E, "gn", 0.0, we)
            if not c < 1e8:  # dependent position rows (a joint that cannot move the tip, say): rank < 3
                continue
            checked += 1
            # minimum norm: the least-squares solution of the three weighted rows with no null-space component
            np.testing.assert_allclose(dq, np.linalg.pinv(J[:3], rcond=R.EPS * 6) @ e[:3], rtol=0,
                                       atol=1e-14 * c * max(1.0, np.abs(dq).max()))
            np.testing.assert_allclose(got[r], dq, rtol=0, atol=1e-10 * max(1.0, np.abs(dq).max()),
                                       err_msg=f"{name} n={n} row {r}")
    assert checked >= 12, checked


def test_rand_q_restates_the_oracle_draw():
    """rand_q gives the start the oracle's loop draws for search 0 when no q0 is given (ilimit = 1, Python semantics:
    q_out = draw + dq, and the draw is what a refused step leaves; here checked through the step reference)."""
    rng = np.random.default_rng(7)
    for name, desc in chains(5, 3):
        C = orc.Chain(desc)
        _, Tep = problems(C, 8, rng)
        q, s, it, sr, E = C.ik_lm(Tep, q0=None, ilimit=1, slimit=1, tol=1e-300, joint_limits=False, k=0.05,
                                  method="wampler", seed=1234, semantics=1, rng_per_row=True)
        for r in range(len(Tep)):
            qs = R.rand_q(C.qlim_l, C.qlim_h, 1234, r, 0)
            assert ((qs >= C.qlim_l) & (qs <= C.qlim_h)).all()
            _, Er, dq = R.step(C, qs, Tep[r], "wampler", 0.05)
            assert E[r] == pytest.approx(Er, rel=1e-14)
            np.testing.assert_allclose(q[r], qs + dq, atol=1e-10)
