"""Vectorised float64 restatement of the functions of the Jacobian (b2k_extra.cu) over a whole (N, 6, n) batch.

The per-row loops of the oracle (oracle.hessian / yoshikawa / jacobm / jacob_dot / manip_svd) restated with stacked
numpy linear algebra, so that the kernels can be checked at batch sizes where a Python loop per row would dominate the
test.  tests/test_jacfun_cpu.py pins every function here against the oracle row by row.  `mask` is an axes mask as the
C ABI takes it: bit k selects row k of J (63 = all, 7 = translational, 56 = rotational).
"""
import numpy as np


def axes(mask):
    """axes mask -> the 6-element bool selection of Cartesian rows"""
    return np.array([(mask >> k) & 1 for k in range(6)], dtype=bool)


def hessian_batch(J):
    """methods.cpp:16-32 over a batch: J (N,6,n) -> H (N,n,6,n); the oracle's loop (oracle.hessian) vectorised over rows.
    Integer input stays integer (int64), so that products of small integers are exact."""
    J = np.asarray(J)
    J = J.astype(np.int64 if J.dtype.kind in "iu" else np.float64)
    N, _, n = J.shape
    H = np.zeros((N, n, 6, n), dtype=J.dtype)
    for a in range(n):
        for b in range(a, n):
            H[:, a, :3, b] = np.cross(J[:, 3:, a], J[:, :3, b])
            H[:, a, 3:, b] = np.cross(J[:, 3:, a], J[:, 3:, b])
            if b != a:
                H[:, b, :3, a] = H[:, a, :3, b]
    return H


def _selected(J, mask):
    return np.asarray(J, dtype=np.float64)[:, axes(mask), :]


def yoshikawa(J, mask=63):
    """ETS.py:1780-1787: |det Ja| when Ja is square, sqrt|det(Ja Ja^T)| otherwise.  (N,)"""
    Ja = _selected(J, mask)
    if Ja.shape[1] == Ja.shape[2]:
        return np.abs(np.linalg.det(Ja))
    return np.sqrt(np.abs(np.linalg.det(Ja @ Ja.transpose(0, 2, 1))))


def singular_values(J, mask=63):
    """the min(rows, n) singular values of each Ja, descending.  (N, min(rows, n))"""
    return np.linalg.svd(_selected(J, mask), compute_uv=False)


def minsingular(J, mask=63):
    """ETS.py:1789-1796, method "minsingular": the smallest singular value of Ja.  (N,)"""
    return singular_values(J, mask)[:, -1]


def invcondition(J, mask=63):
    """ETS.py:1789-1796, method "invcondition": s_min / s_max, 0 where s_max = 0.  (N,)"""
    s = singular_values(J, mask)
    smax = s[:, 0]
    return np.where(smax > 0, s[:, -1] / np.where(smax > 0, smax, 1.0), 0.0)


def jacobm(J, mask=63, H=None):
    """ETS.jacobm ETS.py:1672-1685 / Robot.jacobm Robot.py:1215-1232 over a batch:
    Jm[i] = m * sum_{a,b} (Ja Ha_i^T)[a,b] inv(Ja Ja^T)[a,b].  (N,n)  Only defined where Ja Ja^T is invertible, i.e.
    at most n rows selected and Ja of full rank.  H: hessian_batch(J), if the caller has it."""
    J = np.asarray(J, dtype=np.float64)
    ax = axes(mask)
    Ja, Ha = J[:, ax, :], (hessian_batch(J) if H is None else H)[:, :, ax, :]
    inv = np.linalg.inv(Ja @ Ja.transpose(0, 2, 1))
    return yoshikawa(J, mask)[:, None] * np.einsum("nak,nibk,nab->ni", Ja, Ha, inv, optimize=True)


def jacob_dot(J, qd):
    """Robot.jacob0_dot Robot.py:1099 (np.tensordot(H, qd, (0, 0))) per row: Jd (N,6,n) from J (N,6,n), qd (N,n).
    Integer J and qd give an exact int64 result."""
    H = hessian_batch(J)
    qd = np.asarray(qd)
    return np.einsum("nirb,ni->nrb", H, qd.astype(H.dtype))
