"""The operational-space mpmath reference (tests/opspace_mp_ref.py) without a GPU: it agrees with numpy's inv / pinv on
well-conditioned rows, it satisfies the four Penrose conditions at exact rank deficiency, a numpy port of the kernel's
inverse stays inside its error bars at every joint count and spectrum, and plausible defects of that port each leave
them -- so the bars test_gpu_opspace_sweep.py holds the kernel to are neither loose nor vacuous."""
import functools
import zlib

import numpy as np
import pytest

import opspace_mp_ref as R

KINDS = [(n, True) for n in range(1, 11)] + [(6, False)]


# ------------------------------------------------------------------ numpy port of the kernel's inverse

def port_inv6(a, dt):
    """ops_inv6 (csrc/b2k_opspace.cu, lines 47-89) over rows (N, 6, 6) in dtype: Gauss-Jordan with partial pivoting on
    the first row of largest magnitude; rows with an exactly zero pivot are NaN."""
    A = a.astype(dt).copy()
    N = len(A)
    X = np.broadcast_to(np.eye(6, dtype=dt), (N, 6, 6)).copy()
    ok = np.ones(N, bool)
    rows = np.arange(N)
    for c in range(6):
        p = c + np.argmax(np.abs(A[:, c:, c]), axis=1)
        ok &= A[rows, p, c] != 0
        for M in (A, X):
            top, piv = M[rows, c].copy(), M[rows, p].copy()
            M[rows, c], M[rows, p] = piv, top
        with np.errstate(divide="ignore", invalid="ignore"):
            ip = dt(1) / A[:, c, c]
            A[:, c, c + 1:] *= ip[:, None]
            X[:, c] *= ip[:, None]
            for r in range(6):
                if r != c:
                    f = A[:, r, c].copy()
                    A[:, r, c + 1:] -= f[:, None] * A[:, c, c + 1:]
                    X[:, r] -= f[:, None] * X[:, c]
    X[~ok] = np.nan
    return X


def port_pinv(a, dt, defect=None):
    """ops_pinv (lines 91-164) over rows (N, 6, n) in dtype: one-sided Jacobi on W = Ja (n <= 6) or Ja^T (n >= 7), the
    pair order, convergence test and rotation of the kernel, then sum over kept k of x_k y_k^T / s_k^2.
    defect: "s2" cuts on s^2 instead of s, "nocut" keeps every nonzero singular value, "one_sweep" stops after one
    sweep, "loose" stops fp64 at fp32's orthogonality 1e-6, "swap" takes the other orientation (wide at n = 6, tall at
    n = 7)."""
    a = a.astype(dt)
    N, _, n = a.shape
    tall = (n <= 6) != (defect == "swap")
    W = a.copy() if tall else np.swapaxes(a, 1, 2).copy()
    P, D = W.shape[1:]
    V = np.broadcast_to(np.eye(D, dtype=dt), (N, D, D)).copy()
    eps = dt(1e-15 if dt == np.float64 and defect != "loose" else 1e-6)
    with np.errstate(all="ignore"):
        for _ in range(1 if defect == "one_sweep" else 30):
            rotated = np.zeros(N, bool)
            for p in range(D - 1):
                for q in range(p + 1, D):
                    al, be, ga = (np.zeros(N, dt) for _ in range(3))
                    for r in range(P):
                        x, y = W[:, r, p], W[:, r, q]
                        al, be, ga = al + x * x, be + y * y, ga + x * y
                    skip = (np.abs(ga) <= eps * np.sqrt(al * be)) | (ga == 0)
                    rotated |= ~skip
                    zeta = (be - al) / (dt(2) * np.where(skip, dt(1), ga))
                    t = np.where(zeta >= 0, dt(1), dt(-1)) / (np.abs(zeta) + np.sqrt(dt(1) + zeta * zeta))
                    c0 = dt(1) / np.sqrt(dt(1) + t * t)
                    cs, sn = np.where(skip, dt(1), c0)[:, None], np.where(skip, dt(0), c0 * t)[:, None]
                    for M in (W, V):
                        x, y = M[:, :, p].copy(), M[:, :, q].copy()
                        M[:, :, p], M[:, :, q] = cs * x - sn * y, sn * x + cs * y
            if not rotated.any():
                break
        nn = np.zeros((N, D), dt)
        for r in range(P):
            nn = nn + W[:, r] * W[:, r]
        cut = dt(1e-15) * np.sqrt(nn.max(1, keepdims=True))
        keep = {"s2": nn > cut, "nocut": nn > 0}.get(defect, np.sqrt(nn) > cut)
        inv2 = np.where(keep, dt(1) / nn, dt(0))
    x, y = (V, W) if tall else (W, V)
    return np.einsum("nik,nk,njk->nij", x, inv2, y)


def port(Ja, pinv, dt, ops, defect=None):
    """every output of one b2k_opspace launch, in dtype, from the ported inverse (defect "transposed" uses Ji^T as Ji,
    "cx_sign" adds the Mx Jd Ji term of Cx)"""
    Ji = port_pinv(Ja, dt, defect) if pinv else port_inv6(Ja, dt)
    if defect == "transposed":
        Ji = np.swapaxes(Ji, 1, 2).copy()
    f = lambda k: ops[k].astype(dt)  # noqa: E731
    JiT = np.swapaxes(Ji, 1, 2)
    Mx = JiT @ f("M") @ Ji
    sign = 1 if defect == "cx_sign" else -1
    return {"Ji": Ji, "Mx": Mx, "Cx": JiT @ f("C") @ Ji + sign * (Mx @ (f("Jd") @ Ji)),
            "Gx": np.einsum("kia,ki->ka", Ji, f("G")), "qd": np.einsum("kij,kj->ki", Ji, f("xd")),
            "tau": np.einsum("kri,kr->ki", Ja.astype(dt), f("w"))}


# ------------------------------------------------------------------ cases

@functools.lru_cache(maxsize=None)
def case(dt, n, pinv, N=15):
    """synthetic Ja of every spectrum (three rows each) with operands, and the reference of every output on them"""
    rng = np.random.default_rng(zlib.crc32(f"cpu{np.dtype(dt).name}{n}{pinv}".encode()))
    Ja, names = R.synthetic(n, N, dt, rng)
    ops = R.operands(n, N, dt, rng)
    inv = R.inverse(Ja, pinv)
    ref = R.opspace(Ja, pinv, dt, M=ops["M"], C=ops["C"], Jd=ops["Jd"], G=ops["G"], xd=ops["xd"], w=ops["w"], inv=inv)
    return Ja, names, ops, ref, R.compared(Ja, names, pinv, dt, inv)


def worst(dt, n, pinv, defect=None):
    """{output: largest error / bar over the compared rows} of the port"""
    Ja, _, ops, ref, use = case(dt, n, pinv)
    got = port(Ja, pinv, dt, ops, defect)
    out = {}
    for k, (v, b) in ref.items():
        r = R.ratio(got[k][use], v[use], b[use])
        out[k] = float(r.max()) if np.isfinite(r).all() else np.inf  # a NaN or Inf where the reference is finite fails
    return out


# ------------------------------------------------------------------ tests

@pytest.mark.parametrize("n,pinv", KINDS)
def test_reference_inverse_matches_numpy_on_well_conditioned_rows(n, pinv):
    rng = np.random.default_rng(100 + n)
    Ja, _ = R.synthetic(n, 6, np.float64, rng, spectra=("well",))
    Ji, kappa, rank = R.inverse(Ja, pinv)
    want = np.linalg.pinv(Ja) if pinv else np.linalg.inv(Ja)
    assert (rank == min(6, n)).all() and (kappa < 5).all()
    assert np.abs(Ji.astype(np.float64) - want).max() <= 1e-13 * np.abs(want).max()


@pytest.mark.parametrize("n,structure", [(2, "dup"), (6, "dup"), (3, "zcol"), (6, "zcol"), (6, "zrow"), (7, "zrow"),
                                         (10, "zrow")])
def test_reference_pinv_satisfies_the_penrose_conditions_at_exact_rank_deficiency(n, structure):
    rng = np.random.default_rng(200 + n)
    Ja, _ = R.synthetic(n, 4, np.float64, rng, spectra=(structure,))
    Ji, _, rank = R.inverse(Ja, True)
    assert (rank == min(6, n) - 1).all()
    A, X = Ja.astype(R.LD), Ji
    AX, XA = A @ X, X @ A
    for got, want in ((AX @ A, A), (XA @ X, X), (np.swapaxes(AX, 1, 2), AX), (np.swapaxes(XA, 1, 2), XA)):
        assert np.abs(got - want).max() <= 1e-17 * max(1.0, float(np.abs(want).max()))


def test_reference_inv_is_nan_exactly_at_a_zero_pivot():
    rng = np.random.default_rng(300)
    Ja, names = R.synthetic(6, 10, np.float64, rng)
    Ji, kappa, _ = R.inverse(Ja, False)
    singular = np.isin(names, ("zcol", "zrow", "dup"))
    assert np.isnan(Ji[singular].astype(np.float64)).all() and np.isinf(kappa[singular]).all()
    assert np.isfinite(Ji[~singular].astype(np.float64)).all()


def test_fp32_keeps_only_exactly_dropped_singular_values():
    """A zero column (n <= 6) or zero row (n >= 7) is kept; a duplicated column of a tall Ja, or a zero row of a square
    one, leaves a singular value that only exact arithmetic keeps at zero."""
    rng = np.random.default_rng(400)
    for n, spectrum, keep in ((4, "zcol", True), (6, "zcol", True), (6, "dup", False), (6, "zrow", False), (3, "zrow", True),
                              (8, "zrow", True), (8, "zcol", True), (8, "dup", True)):
        Ja, _ = R.synthetic(n, 3, np.float32, rng, spectra=(spectrum,))
        assert (R.exact_in_fp32(Ja, R.inverse(Ja, True)[2]) == keep).all(), (n, spectrum)


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("n,pinv", KINDS)
def test_the_kernel_port_stays_inside_the_bars(n, pinv, dt):
    assert case(dt, n, pinv)[4].sum() >= 6
    w = worst(dt, n, pinv)
    assert max(w.values()) <= 1.0, w


@pytest.mark.parametrize("dt", [np.float64, np.float32], ids=["f64", "f32"])
def test_either_orientation_of_the_jacobi_svd_is_inside_the_bars(dt):
    """The tall / wide choice at n = 6 / 7 is a matter of cost (D = min(6, n) columns to orthogonalise), not of the
    result: the other orientation meets the same bars, including at the exact structures fp32 admits."""
    for n in (6, 7):
        assert max(worst(dt, n, True, "swap").values()) <= 1.0


def test_the_port_leaves_a_zero_pivot_row_nan():
    Ja, names, ops, ref, _ = case(np.float64, 6, False)
    got = port(Ja, False, np.float64, ops)
    singular = np.isin(names, ("zcol", "zrow"))  # the kernel's elimination meets an exactly zero pivot here
    assert np.isnan(ref["Ji"][0][singular].astype(np.float64)).all()
    for k in ("Ji", "Mx", "Cx", "Gx", "qd"):
        assert np.isnan(got[k][singular]).all(), k
    assert np.isfinite(got["tau"]).all()


# (defect, the cases it must fail on, the output it shows in)
DEFECTS = [
    ("s2", [(np.float64, 6, True), (np.float64, 9, True)], "Ji"),
    ("nocut", [(np.float64, 4, True), (np.float64, 6, True)], "Ji"),
    ("one_sweep", [(np.float64, 5, True), (np.float64, 8, True)], "Ji"),
    ("transposed", [(np.float64, 6, True), (np.float64, 6, False), (np.float32, 6, False)], "Ji"),
    ("cx_sign", [(np.float64, n, p) for n, p in KINDS] + [(np.float32, 6, False)], "Cx"),
    ("loose", [(np.float64, 3, True), (np.float64, 7, True)], "Ji"),
]


@pytest.mark.parametrize("defect,cases,output", DEFECTS, ids=[d[0] for d in DEFECTS])
def test_each_plausible_defect_exceeds_a_bar(defect, cases, output):
    for dt, n, pinv in cases:
        assert max(worst(dt, n, pinv).values()) <= 1.0
        w = worst(dt, n, pinv, defect)
        assert w[output] > 1.0, (defect, np.dtype(dt).name, n, pinv, w)
