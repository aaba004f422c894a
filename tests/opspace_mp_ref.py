"""High-precision reference of the b2k_opspace / b2k_opspace_xdd epilogue (csrc/b2k_opspace.cu), and the synthetic operands
test_opspace_mp_ref_cpu.py and test_gpu_opspace_sweep.py feed it.

The operands are given as exact float64 values (an fp32 kernel's inputs are rounded to fp32 first, so the reference sees
what the kernel sees).  Per row, in mpmath at DPS digits:
  Ji   B2K_OPS_INV: LU with partial pivoting; an exactly zero pivot makes the row NaN, as the kernel does.
       B2K_OPS_PINV: mp.svd_r, keeping s_k > 1e-15 s_max (numpy.linalg.pinv's default rcond, the kernel's cut).
Ji is then carried in long double (its mpmath value to 2 x 53 bits, then rounded to 64), and the products
  Mx = Ji^T M Ji,  Cx = Ji^T C Ji - Mx Jd Ji,  Gx = Ji^T G,  qd = Ji xd,  tau = Ja^T w,  xdd = Ja qdd + Jd qd
are taken in long double: their rounding (u = 2^-64, sums of at most 10 terms) is 2^11 times below the unit roundoff of
fp64 and so three orders below the smallest fp64 bar.  The products are exact polynomials of Ji and the operands, so
nothing is gained by evaluating them at 40 digits, and mpmath would cost ~30 ms more per row.

Every output comes with a per-row error bar  BAR_C * u * max(1, kappa) * scale:
  u      the unit roundoff of the kernel's dtype (2^-53 or 2^-24);
  kappa  the 2-norm condition number of Ja over the singular values kept (1 for tau and xdd, which invert nothing);
  scale  the largest entry of the output's expression evaluated on absolute values, e.g. max |Ji|^T |M| |Ji| for Mx and
         max (|Ji|^T |C| |Ji| + |Ji|^T |M| |Ji| |Jd| |Ji|) for Cx.
BAR_C = 64 for the whole module.  The inverse's normwise relative error is bounded by kappa times its backward error:
Gauss-Jordan on a 6x6 is a few u times its growth factor (at most 2^5, in practice ~2); one-sided Jacobi keeps a backward
error of a few u per sweep (about 6 sweeps at these sizes) and stops at a relative orthogonality of 1e-15 ~ 9u (fp64) or
1e-6 ~ 17u (fp32).  The products add at most three dot products of <= 10 terms, gamma_10 ~ 10u each, bounded by scale.
Either part stays below ~30u, so 64u leaves a factor of two; a factor of four more, as an error that is off by a whole
rank-one term of a kept small singular value, or by one unconverged rotation, is caught (test_opspace_mp_ref_cpu.py
shows six such defects each exceeding the bar).

The cut holds in fp32 too, where a singular value that is exactly zero but rounding makes ~1e-8 s_max is kept, so such a
row has no well-defined fp32 pseudo-inverse.  The kernel's Jacobi rotations keep only one kind of zero singular value
exactly: an all-zero column of the matrix it iterates on (a zero column of Ja when n <= 6, a zero row of Ja when n >= 7).
`exact_in_fp32` tells which rows are rank-deficient in no other way; an fp32 comparison is meaningful only there.
"""
import mpmath as mp
import numpy as np

DPS = 40
RCOND = 1e-15
BAR_C = 64.0
LD = np.longdouble
UNIT = {np.float64: 2.0 ** -53, np.float32: 2.0 ** -24}
assert np.finfo(LD).eps <= 2.0 ** -63, "the products need an 80-bit long double"

SPECTRA = ("well", "graded", "dup", "zcol", "zrow")  # the Ja kinds of `synthetic`
GRADE = {np.float64: 1e-8, np.float32: 1e-3}  # s_min / s_max of the graded spectrum


# ------------------------------------------------------------------ the inverse, per row in mpmath

def _to_ld(x):
    hi = float(x)
    return LD(hi) + LD(float(x - hi))


def _mp_inv(a):
    """inv(a) of a 6x6 by Gauss-Jordan with partial pivoting in mpmath, or None on an exactly zero pivot"""
    n = len(a)
    A = [[mp.mpf(v) for v in row] + [mp.mpf(int(i == j)) for j in range(n)] for i, row in enumerate(a)]
    for c in range(n):
        p = max(range(c, n), key=lambda r: abs(A[r][c]))
        if A[p][c] == 0:
            return None
        A[c], A[p] = A[p], A[c]
        ip = 1 / A[c][c]
        A[c] = [v * ip for v in A[c]]
        for r in range(n):
            if r != c and A[r][c] != 0:
                f = A[r][c]
                A[r] = [x - f * y for x, y in zip(A[r], A[c])]
    return [row[n:] for row in A]


def _mp_pinv(a):
    """(pinv(a) as lists, singular values kept) of a 6 x n in mpmath: svd_r and numpy's rule s_k > RCOND s_max"""
    U, S, V = mp.svd_r(mp.matrix(a))
    s = [S[k] for k in range(len(S))]
    keep = [k for k in range(len(s)) if s[k] > RCOND * max(s)]
    m, n = len(a), len(a[0])
    X = [[mp.fsum(V[k, i] * U[j, k] / s[k] for k in keep) for j in range(m)] for i in range(n)]
    return X, [s[k] for k in keep]


def inverse(Ja, pinv):
    """(Ji (N, n, 6) long double, kappa (N,), rank (N,)) of float64 Ja (N, 6, n).  An INV row with an exactly zero pivot
    is NaN with kappa = inf."""
    Ja = np.asarray(Ja, dtype=np.float64)
    N, _, n = Ja.shape
    Ji, kappa, rank = np.full((N, n, 6), np.nan, dtype=LD), np.full(N, np.inf), np.zeros(N, dtype=int)
    with mp.workdps(DPS):
        for r in range(N):
            a = Ja[r].tolist()
            if pinv:
                X, s = _mp_pinv(a)
            else:
                X = _mp_inv(a)
                sv = mp.svd_r(mp.matrix(a), compute_uv=False)
                s = [sv[k] for k in range(6) if sv[k] > 0]
            rank[r] = len(s)
            if X is None:
                continue
            Ji[r] = [[_to_ld(v) for v in row] for row in X]
            kappa[r] = float(max(s) / min(s)) if s else 1.0
    return Ji, kappa, rank


# ------------------------------------------------------------------ products and their bars

def _bar(dt, kappa, scale):
    return BAR_C * UNIT[dt] * np.maximum(1.0, kappa) * scale.reshape(len(scale), -1).max(1)


def _T(x):
    return np.swapaxes(x, -1, -2)


def opspace(Ja, pinv, dt, M=None, C=None, Jd=None, G=None, xd=None, w=None, inv=None):
    """{name: (value (N, ...) long double, bar (N,))} for Ji and every output whose operands are given.
    inv: a precomputed `inverse(Ja, pinv)`."""
    Ji, kappa, _ = inverse(Ja, pinv) if inv is None else inv
    L = lambda x: np.asarray(x, dtype=np.float64).astype(LD)  # noqa: E731
    A = lambda x: np.abs(np.asarray(x, dtype=np.float64))  # noqa: E731
    aJi = np.abs(Ji.astype(np.float64))
    out = {"Ji": (Ji, _bar(dt, kappa, aJi))}
    if M is not None:
        out["Mx"] = (_T(Ji) @ L(M) @ Ji, _bar(dt, kappa, _T(aJi) @ A(M) @ aJi))
    if C is not None:
        Mx = _T(Ji) @ L(M) @ Ji
        aMx = _T(aJi) @ A(M) @ aJi
        out["Cx"] = (_T(Ji) @ L(C) @ Ji - Mx @ L(Jd) @ Ji, _bar(dt, kappa, _T(aJi) @ A(C) @ aJi + aMx @ A(Jd) @ aJi))
    if G is not None:
        out["Gx"] = (np.einsum("kia,ki->ka", Ji, L(G)), _bar(dt, kappa, np.einsum("kia,ki->ka", aJi, A(G))))
    if xd is not None:
        out["qd"] = (np.einsum("kij,kj->ki", Ji, L(xd)), _bar(dt, kappa, np.einsum("kij,kj->ki", aJi, A(xd))))
    if w is not None:
        out["tau"] = (np.einsum("kri,kr->ki", L(Ja), L(w)), _bar(dt, np.ones(len(Ji)), np.einsum("kri,kr->ki", A(Ja), A(w))))
    return out


def xdd(Ja, qdd, Jd, qd, dt):
    """(xdd = Ja qdd + Jd qd long double, bar) of b2k_opspace_xdd"""
    L = lambda x: np.asarray(x, dtype=np.float64).astype(LD)  # noqa: E731
    A = lambda x: np.abs(np.asarray(x, dtype=np.float64))  # noqa: E731
    v = np.einsum("kri,ki->kr", L(Ja), L(qdd)) + np.einsum("kri,ki->kr", L(Jd), L(qd))
    s = np.einsum("kri,ki->kr", A(Ja), A(qdd)) + np.einsum("kri,ki->kr", A(Jd), A(qd))
    return v, _bar(dt, np.ones(len(v)), s)


def ratio(got, want, bar):
    """per-row max |got - want| / bar (0 where both are exactly zero); NaN where either side is not finite"""
    d = np.abs(np.asarray(got, dtype=np.float64).astype(LD) - want).astype(np.float64)
    d = d.reshape(len(d), -1).max(1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(d == 0, 0.0, d / bar)


# ------------------------------------------------------------------ synthetic operands

def exact_in_fp32(Ja, rank):
    """Rows whose rank deficiency (min(6, n) - rank) is no more than the all-zero columns of the matrix the kernel's
    Jacobi iterates on -- Ja's zero columns when n <= 6, its zero rows when n >= 7 -- so that every dropped singular
    value stays exactly zero in fp32 as well."""
    Ja = np.asarray(Ja)
    n = Ja.shape[2]
    zero = (Ja == 0).all(1 if n <= 6 else 2).sum(1)
    return min(6, n) - np.asarray(rank) <= zero


def compared(Ja, names, pinv, dt, inv):
    """Rows whose every output has a finite, well-defined value to compare with: not an INV row with a zero pivot (NaN),
    not an INV row with a duplicated column (singular, but no elimination pivot of it is exactly zero in floating
    point), and in fp32 only rows that `exact_in_fp32` admits."""
    use = np.isfinite(inv[1])
    if not pinv:
        use &= np.asarray(names) != "dup"
    if dt == np.float32:
        use &= exact_in_fp32(Ja, inv[2])
    return use


def _orth(rng, k):
    q, r = np.linalg.qr(rng.normal(size=(k, k)))
    return q * np.sign(np.diag(r))


def synthetic(n, N, dt, rng, spectra=SPECTRA):
    """(Ja (N, 6, n) float64 holding dtype values, spectrum name per row): row k has spectrum spectra[k % len], built as
    U diag(s) V^T from random orthogonal factors times 10^U(-1, 1), rounded to dt.
      well    s in [0.5, 2]            graded  s from 1 down to GRADE[dt], log-spaced
      dup     well, one column copied over another (n >= 2)
      zcol    well, one column zeroed   zrow    well, one row zeroed"""
    k = min(6, n)
    Ja = np.empty((N, 6, n))
    names = [spectra[r % len(spectra)] for r in range(N)]
    for r, name in enumerate(names):
        s = np.geomspace(1.0, GRADE[dt], k) if name == "graded" else rng.uniform(0.5, 2.0, k)
        a = (_orth(rng, 6)[:, :k] * s) @ _orth(rng, n)[:, :k].T * 10.0 ** rng.uniform(-1, 1)
        if name == "dup" and n >= 2:
            i, j = rng.choice(n, 2, replace=False)
            a[:, i] = a[:, j]
        elif name == "zcol":
            a[:, rng.integers(n)] = 0
        elif name == "zrow":
            a[rng.integers(6), :] = 0
        Ja[r] = a
    return Ja.astype(dt).astype(np.float64), names


def operands(n, N, dt, rng):
    """{M (symmetric positive definite), C, Jd, G, xd, w, qdd, qd}, float64 arrays holding dtype values"""
    B = rng.normal(size=(N, n, n))
    o = {"M": B @ _T(B) / n + np.eye(n), "C": rng.normal(size=(N, n, n)), "Jd": rng.normal(size=(N, 6, n)),
         "G": rng.normal(size=(N, n)) * 10, "xd": rng.normal(size=(N, 6)), "w": rng.normal(size=(N, 6)) * 5,
         "qdd": rng.normal(size=(N, n)), "qd": rng.normal(size=(N, n))}
    o["M"] = (o["M"] + _T(o["M"])) / 2
    return {k: v.astype(dt).astype(np.float64) for k, v in o.items()}


def sample(N, rng, k=48):
    """at most k row indices: 0, 31, 32, N - 1 and random others"""
    fixed = sorted({i for i in (0, 31, 32, N - 1) if 0 <= i < N})
    rest = np.setdiff1d(np.arange(N), fixed)
    pick = rng.choice(rest, min(len(rest), k - len(fixed)), replace=False) if len(rest) else []
    return np.array(sorted(set(fixed) | {int(i) for i in pick}))
