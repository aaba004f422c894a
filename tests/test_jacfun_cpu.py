"""Functions of the Jacobian without a GPU: the batched restatement in jacfun_ref.py -- the specification
test_gpu_jacfun.py checks the kernels against -- is pinned row by row against the oracle's loops at every joint count,
and the five C entry points reject an unsupported joint count before any CUDA call."""
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
