"""Null-space terms of the Python IK solvers (kq, km) without a GPU: the numpy restatement in ikine_null_ref.py -- the
specification the kernel is checked against -- is pinned against the oracle's solver loop and by the identities the
terms must satisfy, and the C ABI and the Python layer reject bad arguments before any CUDA call."""
import os
import sys

import numpy as np
import pytest

import b2kin as rtb
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_null_ref as ref  # noqa: E402

lib = rtb._lib.lib()
PANDA = rtb.models.Panda().ets()
UR10 = rtb.models.UR10().ets()  # kept alive: the tests below pass its chain handle
C = orc.Chain(PANDA.describe())


def _targets(N, seed):
    return C.fkine(np.random.default_rng(seed).uniform(-2.5, 2.5, (N, 7)))


@pytest.mark.parametrize("method", ["chan", "wampler", "sugihara", "nr"])
def test_restatement_without_terms_is_the_oracle_loop(method):
    Tep = _targets(24, 1)
    k = 0.1 if method == "nr" else 1.0  # damped NR: an undamped pseudo-inverse step from a random start is chaotic
    want = C.ik_lm(Tep, None, 30, 4, 1e-6, True, None, k, method, seed=5, semantics=1, rng_per_row=True)
    got = ref.solve(C, Tep, None, 30, 4, 1e-6, True, None, k, method, seed=5)
    for g, w in zip(got[1:4], want[1:4]):
        np.testing.assert_array_equal(g, w)
    # 1e-10, not 1e-12: near convergence the chan matrix J^T J + k E I of a 7-joint arm is within k E of singular, and
    # numpy's LAPACK solve and the oracle's LU round its last step differently
    np.testing.assert_allclose(got[0], want[0], rtol=0, atol=1e-10)


def test_qnull_lies_in_the_null_space():
    rng = np.random.default_rng(3)
    for _ in range(50):
        q = rng.uniform(-2.8, 2.8, 7)
        J = C.jacob0(q)[0]
        for kq, km in ((1.0, 0.0), (0.0, 1.0), (0.5, 2.0)):
            qn = ref.qnull(J, q, C.qlim_l, C.qlim_h, kq, km, 0.0, np.full(7, 0.3))
            assert np.linalg.norm(J @ qn) <= 1e-12 * max(1.0, np.linalg.norm(qn)) * np.linalg.norm(J)


def test_sigma_pushes_away_from_each_limit_inside_its_band():
    ql, qh = np.full(3, -1.0), np.full(3, 1.0)
    ps, pi = 0.05, np.full(3, 0.2)
    s = ref.sigma(np.array([-0.95, 0.0, 0.9]), ql, qh, ps, pi)
    assert s[0] > 0 and s[1] == 0 and s[2] < 0
    # magnitude: ((distance - pi) / (ps - pi))^2, i.e. 1 at distance ps and 0 at the edge of the band
    np.testing.assert_allclose(ref.sigma(np.array([-1 + ps, 0.0, 1 - ps]), ql, qh, ps, pi), [1.0, 0.0, -1.0])
    np.testing.assert_allclose(ref.sigma(np.array([-0.8, 0.8, 0.0]), ql, qh, ps, pi), [0.0, 0.0, 0.0], atol=1e-30)
    # a joint within pi of both limits takes the upper-limit value, as in the reference
    s = ref.sigma(np.array([0.0]), np.array([-0.1]), np.array([0.15]), 0.0, np.array([0.2]))
    assert s[0] == -((0.15 - 0.2) ** 2) / 0.2 ** 2


def test_jacobm_term_is_the_gradient_of_yoshikawa():
    rng = np.random.default_rng(8)
    h = 1e-6
    for _ in range(10):
        q = rng.uniform(-2.5, 2.5, 7)
        g = ref.jacobm_term(C.jacob0(q)[0])
        num = np.array([(orc.yoshikawa(C.jacob0(q + h * d)[0]) - orc.yoshikawa(C.jacob0(q - h * d)[0])) / (2 * h)
                        for d in np.eye(7)])
        np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-9)


def test_restated_step_adds_qnull_to_the_solver_step():
    Tep = _targets(1, 4)[0]
    q0 = np.random.default_rng(4).uniform(-2.5, 2.5, 7)
    base = ref.solve_row(C, Tep, q0, 1, 1, 1e-6, False, None, 1.0, "chan", 0, 0)
    with_terms = ref.solve_row(C, Tep, q0, 1, 1, 1e-6, False, None, 1.0, "chan", 0, 0, kq=1.0, km=1.0, ps=0.0, pi=0.3)
    J = C.jacob0(q0)[0]
    np.testing.assert_allclose(with_terms[0] - base[0],
                               ref.qnull(J, q0, C.qlim_l, C.qlim_h, 1.0, 1.0, 0.0, np.full(7, 0.3)), atol=1e-12)


def _null_call(chain=None, dtype=1, N=4, method=0, kq=1.0, km=0.0, ps=0.0, pi=None, lam=1.0, ilimit=30, slimit=1,
               Tep=8, q_out=8, succ=8, its=8, srch=8, res=8):
    chain = PANDA._chain if chain is None else chain
    if pi is None:
        pi = np.full(7, 0.3)
    pi = None if isinstance(pi, str) else np.ascontiguousarray(pi, dtype=np.float64)
    rc = lib.b2k_ikine_null(chain, dtype, Tep, N, None, ilimit, slimit, 1e-6, 1, None, lam, method, 0, 1, kq, km, ps,
                            rtb._lib.dptr(pi), q_out, succ, its, srch, res, None)
    return rc, lib.b2k_last_error().decode()


def _pi_with(i, v):
    p = np.full(7, 0.3)
    p[i] = v
    return p


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=2), "dtype must be"),
    (dict(N=-1), "N is negative"),
    (dict(chain=UR10._chain), "7..10 joints (n = 6)"),
    (dict(ilimit=0), "ilimit and slimit"),
    (dict(slimit=0), "ilimit and slimit"),
    (dict(method=5), "bad method"),
    (dict(method=3, lam=-1.0), "pinv_damping is negative"),
    (dict(kq=np.nan), "kq and km must be finite"),
    (dict(km=np.inf), "kq and km must be finite"),
    (dict(kq=0.0, km=0.0), "at least one of kq and km"),
    (dict(kq=-1.0, km=-2.0), "at least one of kq and km"),
    (dict(ps=np.nan), "ps must be finite"),
    (dict(pi="null"), "pi is NULL"),
    (dict(pi=_pi_with(3, np.inf)), "pi[3] is not finite"),
    (dict(ps=0.3), "ps == pi[0]"),
    (dict(ps=0.1, pi=_pi_with(6, 0.1)), "ps == pi[6]"),
    (dict(Tep=None), "Tep is NULL"),
    (dict(q_out=None), "q_out is NULL"),
    (dict(res=None), "residual is NULL"),
])
def test_entry_rejects_bad_arguments_before_launching(kw, msg):
    rc, err = _null_call(**kw)
    assert rc == -1
    assert msg in err, err


def test_entry_accepts_what_it_documents_without_work():
    assert _null_call(N=0)[0] == 0
    assert _null_call(N=0, kq=0.0, km=1.0, ps=0.3)[0] == 0  # ps == pi is harmless without the joint-limit term
    assert _null_call(N=0, method=4, kq=2.0, km=-1.0)[0] == 0
    assert _null_call(N=0, Tep=None, q_out=None, succ=None, its=None, srch=None, res=None)[0] == 0


@pytest.mark.parametrize("robot", [rtb.models.Panda, rtb.models.UR10])
def test_python_layer_rejects_bad_null_space_arguments(robot):
    e = robot().ets()
    T = np.eye(4)
    with pytest.raises(ValueError, match="pi must be a scalar or have"):
        e.ikine_LM(T, kq=1.0, pi=np.full(e.n + 1, 0.3))
    with pytest.raises(ValueError, match="pi must be a scalar or have"):
        e.ikine_NR(T, km=1.0, pi=np.zeros((2, e.n)))
    with pytest.raises(ValueError, match="ps == pi"):
        e.ikine_GN(T, kq=1.0, ps=0.3, pi=0.3)
    with pytest.raises(ValueError, match="ps == pi"):
        rtb.IK_LM(kq=0.5, ps=0.2, pi=np.full(e.n, 0.2)).solve(e, T)
    with pytest.raises(ValueError, match="must be finite"):
        e.ikine_LM(T, km=1.0, ps=np.nan)


def test_python_layer_normalises_pi_and_switches_terms_by_sign():
    assert PANDA._null_args(0.0, 0.0, 0.0, 0.3) is None
    assert PANDA._null_args(-1.0, -0.5, 0.0, [1, 2]) is None  # terms off: pi is not used
    kq, km, ps, pi = PANDA._null_args(2.0, 0.0, 0.1, 0.3)
    assert (kq, km, ps) == (2.0, 0.0, 0.1) and pi.shape == (7,) and (pi == 0.3).all()
    assert (PANDA._null_args(0.0, 1.0, 0.0, np.arange(7.0))[3] == np.arange(7.0)).all()
    assert UR10._null_args(1.0, 1.0, 0.0, 0.3) is None  # n <= 6: no null space
