"""Functions of the Jacobian without a GPU: the batched restatement in jacfun_ref.py -- the specification
test_gpu_jacfun.py checks the kernels against -- is pinned row by row against the oracle's loops at every joint count,
and the six C entry points that take a batch of Jacobians reject every bad argument before any CUDA call."""
import os
import sys

import numpy as np
import pytest

import b2kin as rtb
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jacfun_ref as ref  # noqa: E402

# all six axes, translational, rotational, single rows, interleaved, five of six
MASKS = (63, 7, 56, 1, 32, 5, 42, 21, 51, 62, 31)


def _close_rows(got, want, rows, rel):
    """each selected row within `rel` (scalar or per row) of that row's largest |want| (a row of exact zeros must
    match exactly)"""
    scale = np.abs(want).reshape(len(want), -1).max(axis=1)
    err = np.abs(got - want).reshape(len(want), -1).max(axis=1)
    return bool((err <= rel * scale)[rows].all())


@pytest.mark.parametrize("n", range(1, 11))
def test_restatement_matches_the_oracle_row_by_row(n):
    rng = np.random.default_rng(100 + n)
    J = rng.normal(size=(24, 6, n))
    qd = rng.normal(size=(24, n))
    H = ref.hessian_batch(J)
    Jd = ref.jacob_dot(J, qd)
    for k in range(len(J)):
        np.testing.assert_array_equal(H[k], orc.hessian(J[k]))
    assert _close_rows(Jd, np.stack([orc.jacob_dot(orc.hessian(Jk), q) for Jk, q in zip(J, qd)]), slice(None), 1e-14)
    for mask in MASKS:
        ax = ref.axes(mask)
        s = ref.singular_values(J, mask)
        good = s[:, -1] > 1e-3 * s[:, 0]  # well-conditioned rows: cond(Ja) < 1e3
        assert good.sum() >= len(J) // 2, (n, mask)
        m = ref.yoshikawa(J, mask)
        want = np.array([orc.yoshikawa(Jk, ax) for Jk in J])
        np.testing.assert_allclose(m[good], want[good], rtol=1e-14, atol=0, err_msg=f"n={n} mask={mask}")
        for kind, fn in (("minsingular", ref.minsingular), ("invcondition", ref.invcondition)):
            np.testing.assert_allclose(fn(J, mask)[good], orc.manip_svd(J, ax, kind)[good], rtol=1e-14, atol=0,
                                       err_msg=f"n={n} mask={mask} {kind}")
        if ax.sum() <= n:  # more selected rows than joints: the Gram matrix is singular and jacobm undefined
            Jm = ref.jacobm(J, mask)
            want = np.stack([orc.jacobm(Jk, Hk, ax)[:, 0] for Jk, Hk in zip(J, H)])
            # both invert the Gram matrix Ja Ja^T (condition number cond(Ja)^2) and sum in different orders: a few ulp
            # per term of the (6 + n)-long contractions, amplified by the inverse
            cond = s[:, 0] / s[:, -1]
            assert _close_rows(Jm, want, good, 4 * (6 + n) * np.finfo(float).eps * cond ** 2), (n, mask)


def test_restatement_edges():
    """invcondition of an all-zero Ja is 0 (as the oracle's s[0] > 0 test); integer input stays exact."""
    Z = np.zeros((2, 6, 4))
    assert (ref.invcondition(Z) == 0).all() and (ref.minsingular(Z) == 0).all() and (ref.yoshikawa(Z) == 0).all()
    Ji = np.random.default_rng(0).integers(-8, 9, size=(5, 6, 10))
    qi = np.random.default_rng(1).integers(-8, 9, size=(5, 10))
    Jd = ref.jacob_dot(Ji, qi)
    assert Jd.dtype == np.int64
    np.testing.assert_array_equal(Jd, ref.jacob_dot(Ji.astype(np.float64), qi.astype(np.float64)))


ENTRY_POINTS = ("b2k_hessian", "b2k_manipulability", "b2k_manipulability_svd", "b2k_jacob_dot", "b2k_jacobm")


@pytest.mark.parametrize("fn", ENTRY_POINTS)
@pytest.mark.parametrize("n", [-1, 0, 11])
def test_entry_points_reject_a_bad_joint_count_before_any_cuda_call(fn, n):
    """Every other argument is valid; the host buffer stands in for a (never dereferenced) device pointer.  Without a
    device, an entry point that reached the CUDA runtime first would report a CUDA error instead."""
    lib = rtb._lib.lib()
    buf = np.zeros(64)
    p = buf.ctypes.data
    args = {"b2k_hessian": (1, n, p, 4, p, None),
            "b2k_manipulability": (1, n, p, 4, 63, p, None),
            "b2k_manipulability_svd": (1, n, p, 4, 63, 0, p, None),
            "b2k_jacob_dot": (1, n, p, p, 4, p, None),
            "b2k_jacobm": (1, n, p, 4, 63, p, None)}[fn]
    n0 = lib.b2k_launch_count()
    assert getattr(lib, fn)(*args) == -1
    assert b"joint count" in lib.b2k_last_error(), lib.b2k_last_error()
    assert lib.b2k_launch_count() == n0



# ---- the six entry points on one table of bad arguments.  Each call has valid arguments except the ones a case names; a
# host buffer stands in for the (never dereferenced) device arrays.  Without a device, a call that reached the CUDA
# runtime would report a CUDA error instead.
JACFUN_OUT = {"b2k_hessian": "H", "b2k_manipulability": "m", "b2k_manipulability_svd": "m", "b2k_jacob_dot": "Jd",
              "b2k_jacobm": "Jm", "b2k_partial_fkine": "D"}
MASKED = ("b2k_manipulability", "b2k_manipulability_svd", "b2k_jacobm")
_BUF = np.zeros(64)
_P = _BUF.ctypes.data  # 16-byte aligned


def _jacfun_call(fn, dtype=1, n=4, J=_P, qd=_P, out=_P, N=4, mask=63, kind=0, order=3):
    lib = rtb._lib.lib()
    args = {"b2k_hessian": (dtype, n, J, N, out),
            "b2k_manipulability": (dtype, n, J, N, mask, out),
            "b2k_manipulability_svd": (dtype, n, J, N, mask, kind, out),
            "b2k_jacob_dot": (dtype, n, J, qd, N, out),
            "b2k_jacobm": (dtype, n, J, N, mask, out),
            "b2k_partial_fkine": (dtype, n, order, J, N, out)}[fn]
    n0 = lib.b2k_launch_count()
    rc = getattr(lib, fn)(*args, None)
    assert lib.b2k_launch_count() == n0, fn
    return rc, lib.b2k_last_error().decode()


# (case, the entry points that take the argument (None: all six), the arguments, what the message says ({out}: the
# output's name); None: the call is accepted)
JACFUN_CASES = [
    ("dtype 2", None, dict(dtype=2), "dtype"),
    ("n -1", None, dict(n=-1), "joint count"),
    ("n 0", None, dict(n=0), "joint count"),
    ("n 11", None, dict(n=11), "joint count"),
    ("N -1", None, dict(N=-1), "N is negative"),
    ("J NULL", None, dict(J=None), "J is NULL"),
    ("out NULL", None, dict(out=None), "{out} is NULL"),
    ("qd NULL", ("b2k_jacob_dot",), dict(qd=None), "qd is NULL"),
    ("mask 0", MASKED, dict(mask=0), "axis"),
    ("mask 64", MASKED, dict(mask=64), "axis"),  # no bit of the six Cartesian rows
    ("kind 2", ("b2k_manipulability_svd",), dict(kind=2), "kind"),
    ("order 2", ("b2k_partial_fkine",), dict(order=2), "order"),
    ("order 6", ("b2k_partial_fkine",), dict(order=6), "order"),
    *[(f"{a} {name} +{off}", ("b2k_jacob_dot",) if a == "qd" else None, {"dtype": dt, a: _P + off},
       ("{out}" if a == "out" else a) + " is not aligned")
      for a in ("J", "qd", "out") for dt, name, off in ((0, "fp32", 2), (1, "fp64", 4))],
    ("N 0, J misaligned", None, dict(N=0, J=_P + 4), "J is not aligned"),
    ("N 0, every array NULL", None, dict(N=0, J=None, qd=None, out=None), None),
    ("N 0, fp32", None, dict(N=0, dtype=0), None),
]


@pytest.mark.parametrize("fn, case", [(fn, c) for c in JACFUN_CASES for fn in JACFUN_OUT if c[1] is None or fn in c[1]],
                         ids=lambda x: x[0] if isinstance(x, tuple) else x)
def test_entry_points_reject_bad_arguments_before_any_cuda_call(fn, case):
    _, _, kw, want = case
    rc, msg = _jacfun_call(fn, **kw)
    if want is None:
        assert rc == 0, msg
    else:
        assert rc == -1 and msg.startswith(fn + ":") and want.format(out=JACFUN_OUT[fn]) in msg, msg


@pytest.mark.parametrize("fn", JACFUN_OUT)
def test_entry_points_check_in_one_order(fn):
    """dtype, joint count, N, kind / order, axes, NULL arrays, alignment: with every defect present the first one is
    reported, and repairing it reports the next."""
    args = dict(dtype=2, n=0, N=-1, kind=2, order=6, mask=0, J=None, qd=None, out=None)
    steps = [({}, "dtype", None), (dict(dtype=1), "joint count", None), (dict(n=4), "N is negative", None),
             (dict(N=4), "kind", ("b2k_manipulability_svd",)), ({}, "order", ("b2k_partial_fkine",)),
             (dict(kind=0, order=3), "axis", MASKED), (dict(mask=63), "J is NULL", None),
             (dict(J=_P + 4), "qd is NULL", ("b2k_jacob_dot",)), (dict(qd=_P + 4), "{out} is NULL", None),
             (dict(out=_P + 4), "J is not aligned", None), (dict(J=_P), "qd is not aligned", ("b2k_jacob_dot",)),
             (dict(qd=_P), "{out} is not aligned", None)]
    for fix, want, fns in steps:
        args.update(fix)
        if fns is None or fn in fns:
            rc, msg = _jacfun_call(fn, **args)
            assert rc == -1 and want.format(out=JACFUN_OUT[fn]) in msg, (want, msg)
