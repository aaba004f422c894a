"""The kernels of b2k_extra.cu that consume a Jacobian -- Yoshikawa manipulability, the singular-value measures,
jacobm and jacob0_dot -- at every joint count, axis selection and dtype, so that every kernel jacfun_launch selects is
reached (the Hessian has its own exhaustive test in test_gpu_widened_r2.py).

Most checks call the C ABI directly and compare with the batched float64 restatement in jacfun_ref.py; fp32 runs
are compared with the restatement evaluated on the fp32-rounded J, so that the rounding of the input is not counted as
kernel error.  Every output lands in a NaN-filled buffer with guard elements on both sides that must stay NaN.

Error bars come from the error model of each method (eps = the unit roundoff of the kernel's dtype, r = selected
Cartesian rows, n = joints, cond = s_max / s_min of the selected block Ja):
  * one-sided Jacobi SVD (k_singular_all / k_singular): absolute, 16 max(r, n) eps s_max -- every plane rotation moves
    the two columns it touches by a few ulp, a column takes part in min(r, n) - 1 rotations per sweep over a handful
    of sweeps, and its norm is a max(r, n)-long sum;
  * Yoshikawa through the Gram matrix Ja Ja^T (k_yoshikawa_all, k_yoshikawa when Ja is not square): relative,
    r (r + n) eps cond^2 -- forming the Gram matrix and factorising it are backward stable to (r + n) eps, the Gram
    matrix has condition number cond^2, and a determinant sums the relative errors of its r pivots;
  * |det Ja| by elimination on Ja itself (k_yoshikawa, square Ja): relative, 4 r^2 eps cond;
  * jacobm: (8 + r^2 (r + n)) eps cond^2 relative to m max|inv(Ja Ja^T)| sum |Ja| |Ha|', where |Ha|' is the size of
    the two products each Hessian entry is the difference of (an entry can cancel to far below its rounding error) --
    the error of the inverse Gram matrix propagated through the contraction, plus the fixed chain of operations that
    forms m, the Hessian terms and the product.
"""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import chains as ch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jacfun_ref as ref  # noqa: E402

B = rtb._buffers
DTYPES = (np.float64, np.float32)
EPS = {np.float64: np.finfo(np.float64).eps, np.float32: np.finfo(np.float32).eps}
# around the 32-row warp tiles and the 64- / 128-thread blocks of the kernels
N_EDGES = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129)
GUARD = 5  # odd: the outputs are only element-aligned
RATIOS = {}  # test_known_singular_values: largest observed error / bar per quantity and dtype


def n_large(n):
    """many waves of blocks at the shipped arm sizes, a ragged last tile everywhere (as the Hessian test)"""
    return 150_003 if n in (6, 7) else 9001


def popcount(mask):
    return bin(mask).count("1")


def run(what, J, n, mask=63, qd=None):
    """One call of a C entry point on the numpy batch J (its dtype is the kernel's).  Returns the output as numpy
    after checking that the guards around it are untouched."""
    N = J.shape[0]
    Jd = torch.from_numpy(np.ascontiguousarray(J)).cuda()
    width = {"jacobm": n, "jacob_dot": 6 * n}.get(what, 1)
    buf = torch.full((N * width + 2 * GUARD,), float("nan"), dtype=Jd.dtype, device="cuda")
    out = buf[GUARD:GUARD + N * width]
    lib, code, st = rtb._lib.lib(), B.code(J.dtype), B.stream_ptr(Jd)
    if what == "yoshikawa":
        rc = lib.b2k_manipulability(code, n, B.ptr(Jd), N, mask, B.ptr(out), st)
    elif what in ("minsingular", "invcondition"):
        rc = lib.b2k_manipulability_svd(code, n, B.ptr(Jd), N, mask, int(what == "invcondition"), B.ptr(out), st)
    elif what == "jacobm":
        rc = lib.b2k_jacobm(code, n, B.ptr(Jd), N, mask, B.ptr(out), st)
    else:
        qdd = torch.from_numpy(np.ascontiguousarray(qd, dtype=J.dtype)).cuda()
        rc = lib.b2k_jacob_dot(code, n, B.ptr(Jd), B.ptr(qdd), N, B.ptr(out), st)
    rtb._lib.check(rc)
    b = buf.cpu().numpy()
    assert np.isnan(b[:GUARD]).all() and np.isnan(b[-GUARD:]).all(), f"{what} n={n} N={N}: a guard was overwritten"
    return b[GUARD:GUARD + N * width].reshape({"jacobm": (N, n), "jacob_dot": (N, 6, n)}.get(what, (N,)))


def known_block(rng, N, n, mask, conds):
    """J (N,6,n) whose selected rows are Ja = U diag(s) V^T with random orthogonal U, V and prescribed singular values
    s (N, min(r, n)), descending: s_max in [0.5, 2], s_min = s_max / cond with cond = conds[row % len(conds)] (1 where
    Ja has a single singular value), the others log-uniform in between.  The rows that are not selected are random.
    Returns J, s, cond."""
    ax = ref.axes(mask)
    r = int(ax.sum())
    k = min(r, n)
    cond = np.asarray(conds, dtype=float)[np.arange(N) % len(conds)] if k > 1 else np.ones(N)
    t = np.sort(rng.uniform(0, 1, (N, k)), axis=1)
    t[:, 0], t[:, -1] = 0.0, 1.0
    s = rng.uniform(0.5, 2.0, (N, 1)) * cond[:, None] ** -t
    U = np.linalg.qr(rng.normal(size=(N, r, r)))[0]
    V = np.linalg.qr(rng.normal(size=(N, n, n)))[0]
    J = rng.normal(size=(N, 6, n))
    J[:, ax, :] = (U[:, :, :k] * s[:, None, :]) @ V[:, :, :k].transpose(0, 2, 1)
    return J, s, cond


def bar_svd(dt, r, n, smax):
    return 16 * max(r, n) * EPS[dt] * smax


def bar_yoshikawa(dt, r, n, cond):
    return 4 * r * r * EPS[dt] * cond if r == n else r * (r + n) * EPS[dt] * cond ** 2


def bar_jacobm(dt, r, n, cond):
    return (8 + r * r * (r + n)) * EPS[dt] * cond ** 2


def hessian_abs(J):
    """(N,n,6,n): |u1 w2| + |u2 w1| for every Hessian entry u1 w2 - u2 w1 (ref.hessian_batch's layout) -- the size
    of the two products an entry is the difference of, i.e. the scale of its rounding error under cancellation"""
    N, _, n = J.shape
    A = np.abs(J)

    def cross_abs(u, w):  # (N,3,n,n) indexed [row, c, a, b]: u from joint a, w from joint b
        u1, u2 = np.roll(u, -1, axis=1)[:, :, :, None], np.roll(u, -2, axis=1)[:, :, :, None]
        w1, w2 = np.roll(w, -1, axis=1)[:, :, None, :], np.roll(w, -2, axis=1)[:, :, None, :]
        return u1 * w2 + u2 * w1

    upper = np.triu(np.ones((n, n), dtype=bool))  # [a, b]: b >= a
    tr = cross_abs(A[:, 3:], A[:, :3])
    tr = np.where(upper, tr, tr.transpose(0, 1, 3, 2))  # below the diagonal: mirrored
    rot = np.where(upper, cross_abs(A[:, 3:], A[:, 3:]), 0.0)  # below the diagonal: zero
    return np.concatenate([tr, rot], axis=1).transpose(0, 2, 1, 3)


def jacobm_scale(J, mask):
    """per row: m max|inv(Ja Ja^T)| max_i sum_{a,b,k} |Ja[a,k]| hessian_abs_i[b,k]"""
    ax = ref.axes(mask)
    Ja = J[:, ax, :]
    inv = np.linalg.inv(Ja @ Ja.transpose(0, 2, 1))
    terms = np.einsum("nak,nibk->ni", np.abs(Ja), hessian_abs(J)[:, :, ax, :], optimize=True).max(axis=1)
    return ref.yoshikawa(J, mask) * np.abs(inv).max(axis=(1, 2)) * terms


def check_measures(Jk, n, mask, cond, tag, rows=slice(None), jacobm=True):
    """yoshikawa, minsingular, invcondition and (r <= n) jacobm of the batch Jk against the restatement on the same
    (rounded) values; rows = the part of the batch to launch"""
    dt = Jk.dtype.type
    Jk, cond = Jk[rows], cond[rows]
    Jr = Jk.astype(np.float64)
    r = popcount(mask)
    sv = ref.singular_values(Jr, mask)
    smax = sv[:, 0]
    bs = bar_svd(dt, r, n, smax)
    err = np.abs(run("minsingular", Jk, n, mask) - sv[:, -1])
    assert (err <= bs).all(), (tag, "minsingular", (err / bs).max())
    err = np.abs(run("invcondition", Jk, n, mask) - ref.invcondition(Jr, mask))
    assert (err <= 2 * bs / smax).all(), (tag, "invcondition", (err * smax / bs / 2).max())
    m = run("yoshikawa", Jk, n, mask)
    if r <= n:
        want = ref.yoshikawa(Jr, mask)
        err = np.abs(m - want) / want
        assert (err <= bar_yoshikawa(dt, r, n, cond)).all(), (tag, "yoshikawa", (err / bar_yoshikawa(dt, r, n, cond)).max())
    else:
        # Ja has rank n < r: det(Ja Ja^T) = 0 up to the rounding of the Gram matrix, |dA| <= r (r + n) eps s_max^2,
        # times the other r - 1 eigenvalues (<= s_max^2 each)
        assert (m <= np.sqrt(r * r * (r + n) * EPS[dt]) * smax ** r).all(), (tag, "yoshikawa of a rank-deficient Ja")
    if jacobm and r <= n:
        Jm = run("jacobm", Jk, n, mask)
        err = np.abs(Jm - ref.jacobm(Jr, mask)).max(axis=1)
        bar = bar_jacobm(dt, r, n, cond)
        # rows where the model leaves no significant digit (fp32, cond 1e3: the Gram matrix is within rounding of
        # singular, and its factorisation may break down into inf / nan) are not checked
        sig = bar < 1
        bar = bar * jacobm_scale(Jr, mask)
        assert (err <= bar)[sig].all(), (tag, "jacobm", (err / bar)[sig].max())


# ------------------------------------------------------------------ 1. jacob0_dot exactly
@pytest.mark.parametrize("n", range(1, 11))
def test_jacob_dot_is_exact_on_small_integers(n):
    """k_jacob_dot_lane: with integer J, qd in -8..8 every product and partial sum is an integer below 2^24 (a term is
    at most 8 * 2 * 64, a sum at most 10 terms), so fp64 and fp32 must equal the int64 reference bit for bit -- at
    every tile edge of the 64-thread blocks and with a ragged last tile after many waves."""
    rng = np.random.default_rng(10 + n)
    Nl = n_large(n)
    J = rng.integers(-8, 9, size=(Nl, 6, n))
    qd = rng.integers(-8, 9, size=(Nl, n))
    want = ref.jacob_dot(J, qd)
    assert np.abs(want).max() < 2 ** 24
    for dt in DTYPES:
        for N in N_EDGES + (Nl,):
            np.testing.assert_array_equal(run("jacob_dot", J[:N].astype(dt), n, qd=qd[:N]), want[:N],
                                          err_msg=f"n={n} N={N} {dt.__name__}")


# ------------------------------------------------------------------ 2. known singular values
KNOWN_MASKS = (63, 7, 56, 53, 33)  # all six axes, translational, rotational, four rows, two rows


def _note(key, ratio):
    RATIOS[key] = max(RATIOS.get(key, 0.0), float(np.max(ratio)))
    assert np.max(ratio) <= 1, (key, float(np.max(ratio)))


def test_known_singular_values():
    """Ja = U diag(s) V^T with prescribed s: minsingular = s_min, invcondition = s_min / s_max and, with no more
    selected rows than joints, yoshikawa = prod s -- across condition-number bands up to 1e6 (fp64) / 1e2 (fp32),
    for the all-axes kernels at every n (tall n < 6, square n = 6, wide n > 6) and for subsets."""
    rng = np.random.default_rng(2)
    for dt in DTYPES:
        conds = (1.0, 1e2, 1e4, 1e6) if dt == np.float64 else (1.0, 1e2)
        for n in range(1, 11):
            for mask in KNOWN_MASKS:
                r = popcount(mask)
                J, s, cond = known_block(rng, 256, n, mask, conds)
                Jk = J.astype(dt)
                if dt == np.float64:
                    smin, smax, m = s[:, -1], s[:, 0], s.prod(axis=1)
                else:  # on the rounded input, where the prescribed values no longer hold to fp32 precision
                    sv = ref.singular_values(Jk.astype(np.float64), mask)
                    smin, smax, m = sv[:, -1], sv[:, 0], ref.yoshikawa(Jk.astype(np.float64), mask)
                key = dt.__name__
                bs = bar_svd(dt, r, n, smax)
                _note(("minsingular", key), np.abs(run("minsingular", Jk, n, mask) - smin) / bs)
                _note(("invcondition", key), np.abs(run("invcondition", Jk, n, mask) - smin / smax) / (2 * bs / smax))
                if r <= n:
                    rel = np.abs(run("yoshikawa", Jk, n, mask) / m - 1)
                    _note(("yoshikawa square" if r == n else "yoshikawa gram", key), rel / bar_yoshikawa(dt, r, n, cond))
    print("\nlargest error / bar:", {" ".join(k): round(v, 4) for k, v in sorted(RATIOS.items())})


# ------------------------------------------------------------------ 3. every mask at every joint count
def test_every_mask_at_every_joint_count():
    """All 63 non-empty axis masks at n = 1..10, both dtypes, N = 97 (a partial 128-thread block): square and
    non-square k_yoshikawa, k_yoshikawa_all, k_singular / k_singular_all, k_jacobm / k_jacobm_all (n = 6: square J).
    jacobm where it is defined: no more selected rows than joints; every row has cond(Ja) <= 1e3."""
    rng = np.random.default_rng(3)
    for n in range(1, 11):
        for mask in range(1, 64):
            J, s, cond = known_block(rng, 97, n, mask, (1.0, 10.0, 1e2, 1e3))
            for dt in DTYPES:
                check_measures(J.astype(dt), n, mask, cond, f"n={n} mask={mask} {dt.__name__}")


# ------------------------------------------------------------------ 4. ragged tiles of the staged / all-axes kernels
@pytest.mark.parametrize("dt", DTYPES)
def test_all_axes_kernels_at_every_tile_edge(dt):
    """k_yoshikawa_all (n >= 7), k_jacobm_all (n >= 6) and k_singular_all (every n) at every tile edge and after many
    waves, both dtypes.  (k_jacob_dot_lane: test_jacob_dot_is_exact_on_small_integers.)"""
    rng = np.random.default_rng(4)
    for n in range(1, 11):
        Nl = n_large(n)
        J, s, cond = known_block(rng, Nl, n, 63, (1.0, 10.0, 1e2))
        Jk = J.astype(dt)
        for N in N_EDGES + (Nl,):
            check_measures(Jk, n, 63, cond, f"n={n} N={N} {dt.__name__}", rows=slice(0, N))


# ------------------------------------------------------------------ 5. row isolation
def _special_row(kind, n, rng):
    j = rng.normal(size=(6, n))
    if kind == "zero":
        j[:] = 0
    elif kind in ("nan", "+inf", "-inf"):
        j[rng.integers(0, 6), rng.integers(0, n)] = {"nan": np.nan, "+inf": np.inf, "-inf": -np.inf}[kind]
    else:  # two equal columns
        j[:, n - 1] = j[:, 0]
    return j


def test_special_rows_stay_in_their_row():
    """All-zero, NaN, +-Inf and rank-deficient (two equal columns) rows at the edges of the warp tiles and blocks:
    every other row must be bit for bit what it is when those rows are ordinary.  An all-zero row has a documented
    result: yoshikawa = minsingular = invcondition = 0 exactly (every mask), jacob_dot = 0, jacobm non-finite."""
    rng = np.random.default_rng(5)
    N = 129
    special = np.array([0, 31, 32, 63, 64, N - 1])
    others = np.setdiff1d(np.arange(N), special)
    for n in range(1, 11):
        J = rng.normal(size=(N, 6, n))
        qd = rng.normal(size=(N, n))
        for dt in DTYPES:
            Jk = J.astype(dt)
            for kind in ("zero", "nan", "+inf", "-inf", "dupcol"):
                if kind == "dupcol" and n == 1:
                    continue
                J2 = Jk.copy()
                for i in special:
                    J2[i] = _special_row(kind, n, rng)
                tag = f"n={n} {dt.__name__} {kind}"
                masks = range(1, 64) if kind == "zero" else (63, 7, 56, 21)
                for mask in masks:
                    for what in ("yoshikawa", "minsingular", "invcondition"):
                        got = run(what, J2, n, mask)
                        np.testing.assert_array_equal(got[others], run(what, Jk, n, mask)[others], err_msg=f"{tag} {what} {mask}")
                        if kind == "zero":
                            assert (got[special] == 0).all(), (tag, what, mask, got[special])
                    if popcount(mask) <= n:
                        got = run("jacobm", J2, n, mask)
                        np.testing.assert_array_equal(got[others], run("jacobm", Jk, n, mask)[others], err_msg=f"{tag} jacobm {mask}")
                        if kind == "zero":
                            assert not np.isfinite(got[special]).any(), (tag, "jacobm", mask, got[special])
                got = run("jacob_dot", J2, n, qd=qd)
                np.testing.assert_array_equal(got[others], run("jacob_dot", Jk, n, qd=qd)[others], err_msg=f"{tag} jacob_dot")
                if kind == "zero":
                    assert (got[special] == 0).all(), (tag, "jacob_dot")


# ------------------------------------------------------------------ 6. identities on real chains
AX = ["Rx", "Ry", "Rz", "tx", "ty", "tz"]


def revolute_chain(rng, n):
    """a random all-revolute chain (Rx / Ry / Rz joints, flips, constant translations and rotations between them):
    the Hessian-from-J formula of the kernels, like the reference's, holds for revolute joints only"""
    b = ch.Builder()
    for _ in range(n):
        for _ in range(int(rng.integers(1, 3))):
            b.const(int(rng.integers(0, 6)), float(rng.uniform(-1.0, 1.0)))
        b.joint(int(rng.integers(0, 3)), flip=bool(rng.random() < 0.3))
    b.const(int(rng.integers(3, 6)), float(rng.uniform(0.2, 1.0)))  # the end point off the last axis
    d = b.desc()
    return rtb.ETS([rtb.ET(AX[int(d["axis"][i])], flip=bool(d["flip"][i]), jindex=int(d["jindex"][i])) if d["isjoint"][i]
                    else rtb.ET.SE3(d["T"][i]) for i in range(len(d["isjoint"]))])


def test_derivative_identities_on_revolute_chains():
    """Independent of any restatement, through the device FK / Jacobian kernels in fp64:
    jacob0_dot(q, qd) = d/dt jacob0(q + t qd) and jacobm(q) = d manipulability / dq, by central differences.
    h = 1e-5: the truncation error h^2 f''' / 6 and the rounding error eps f / h are both ~1e-10 of the row's scale
    for these unit-sized chains, so a bar of 1e-6 of the row's largest |.| leaves four orders of margin and still
    catches any wrong term.  jacobm only on rows whose selected block has s_min > 0.1, where m is smooth."""
    rng = np.random.default_rng(6)
    h, bar = 1e-5, 1e-6
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()  # noqa: E731
    host = lambda t: t.cpu().numpy()  # noqa: E731
    for n in range(1, 11):
        e = revolute_chain(rng, n)
        Q = rng.uniform(-np.pi, np.pi, (64, n))
        qd = rng.normal(size=(64, n))
        got = host(e.jacob0_dot(dev(Q), dev(qd)))
        num = (host(e.jacob0(dev(Q + h * qd))) - host(e.jacob0(dev(Q - h * qd)))) / (2 * h)
        scale = np.abs(num).max(axis=(1, 2))
        assert (np.abs(got - num).max(axis=(1, 2)) <= bar * scale).all(), (n, "jacob0_dot")
        # all six axes, or (n < 6) square selections and the translational / rotational triple; a random chain can make
        # some of them singular everywhere (Rx joints only: the x row of the translational block is zero)
        masks = [63] if n >= 6 else [m for m in range(1, 64) if popcount(m) == n]
        masks += [7, 56] if n > 3 else []
        tested = 0
        for mask in masks:
            axes = [bool(a) for a in ref.axes(mask)]
            ok = host(e.manipulability(dev(Q), method="minsingular", axes=axes)) > 0.1
            if ok.sum() < 8 or tested == 4:
                continue
            tested += 1
            Jm = host(e.jacobm(dev(Q), axes=axes))
            num = np.stack([(host(e.manipulability(dev(Q + h * d), axes=axes)) - host(e.manipulability(dev(Q - h * d), axes=axes)))
                            / (2 * h) for d in np.eye(n)], axis=1)
            scale = np.abs(num).max(axis=1)
            assert (np.abs(Jm - num).max(axis=1) <= bar * scale)[ok].all(), (n, mask, "jacobm")
        assert tested, f"n={n}: every selection is singular on this chain"


# ------------------------------------------------------------------ 7. the wrapper checks the shape of J
def test_manipulability_rejects_a_jacobian_of_the_wrong_width():
    """ETS / Robot / DHRobot.manipulability(J=...) with J of n - 1 or n + 1 columns: a ValueError before any launch
    (with more columns the kernel would read rows at the wrong stride, with fewer past the end of the buffer)."""
    rng = np.random.default_rng(7)
    for robot in (rtb.models.Panda(), rtb.models.Puma560()):
        n = robot.n
        for m in (n - 1, n + 1):
            for J in (rng.normal(size=(6, m)), rng.normal(size=(5, 6, m)),
                      torch.from_numpy(rng.normal(size=(5, 6, m))).cuda()):
                for method in ("yoshikawa", "minsingular", "invcondition"):
                    for fn in (robot.manipulability, robot.ets().manipulability):
                        n0 = rtb.launch_count()
                        with pytest.raises(ValueError, match="Jacobian must be"):
                            fn(J=J, method=method)
                        assert rtb.launch_count() == n0, (robot.name, m, method)
        J = rng.normal(size=(5, 6, n))
        for method in ("yoshikawa", "minsingular", "invcondition"):
            got = robot.manipulability(J=J, method=method)
            assert got.shape == (5,) and isinstance(robot.manipulability(J=J[0], method=method), float)
            np.testing.assert_allclose(got, getattr(ref, method)(J), rtol=1e-10)
