"""The pose-representation kernels at the rotations where such code goes wrong -- near identity and near a half turn,
in the gimbal bands of rpy and ZYZ, on either side of every branch threshold, through every quaternion branch of
ctraj's host side -- against the mpmath restatement in pose_ref.py, both dtypes.

The C entry points are called directly on constructed inputs (no FK): every rotation is built in mpmath from an axis
and an angle (or from rpy / Euler angles) and then rounded, and the reference is evaluated on exactly the rounded
numbers.  Outputs land in NaN-filled buffers with guard elements, so an unwritten row or a stray write fails.

Bars: fp64 rtol 1e-10 / atol 1e-12, fp32 1e-4 / 1e-5, per row, relative to the row's largest |entry|.  Near the
singularity of rpy and ZYZ the bar of jacob0_analytical is multiplied by kappa = max(1, 1/|cos pitch|) (rpy) or
max(1, 1/|sin theta|) (eul): A^-1 has entries ~ kappa, and the kernel's pitch / theta carries an absolute rounding
error ~ eps, so A^-1 is known only to ~ eps kappa relative.  Rows with kappa above 1e6 (fp64) / 1e3 (fp32) leave no
significant digit at the bar and are skipped -- their count is asserted, and their translational rows must still pass
J through.  exp needs no factor: A^-1 is bounded for theta <= pi.  p_servo's edge rows take Te = I, so that Re^T Rep has
no rounding and the error angles come from exact inputs: no factor there either.
"""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pose_ref as ref  # noqa: E402

B = rtb._buffers
M = ref.M
DTYPES = (np.float64, np.float32)
TOL = {np.float64: (1e-10, 1e-12), np.float32: (1e-4, 1e-5)}
KMAX = {np.float64: 1e6, np.float32: 1e3}
N_EDGES = (1, 31, 32, 33, 63, 64, 65, 4099)  # around the 32-row warp tiles and 64-thread blocks of k_janalytical
N_BIG = 200_003  # several waves, a ragged last tile
GUARD = 4  # keeps 16-byte alignment of the output in both dtypes
WORST = {}  # largest error / row scale seen per (kernel, representation, dtype)


def dev(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def nan_buffer(n, dt):
    return torch.full((n + 2 * GUARD,), float("nan"), dtype=B.tdtype(np.dtype(dt)), device="cuda")


def unguard(buf, n, tag):
    b = buf.cpu().numpy()
    assert np.isnan(b[:GUARD]).all() and np.isnan(b[GUARD + n:]).all(), f"{tag}: a guard element was overwritten"
    return b[GUARD:GUARD + n]


def row_errors(got, want, wrap=None):
    """per row: max |got - want| and the row's largest |want|.  wrap (per column, or None): compare those columns
    modulo that period (angles at an exact +-pi may come out on either side)"""
    N = len(want)
    d = got.reshape(N, -1) - want.reshape(N, -1)
    if wrap is not None:
        w = np.broadcast_to(np.asarray(wrap, dtype=np.float64), d.shape[1:])
        m = w > 0
        d[:, m] = d[:, m] - w[m] * np.round(d[:, m] / w[m])
    return np.abs(d).max(axis=1), np.abs(want).reshape(N, -1).max(axis=1)


def check_rows(got, want, dt, key, kap=1.0, wrap=None, rows=None):
    rtol, atol = TOL[dt]
    err, scale = row_errors(got, want, wrap)
    bar = (rtol * scale + atol) * kap
    sel = np.ones(len(err), dtype=bool) if rows is None else rows
    assert np.isfinite(got.reshape(len(err), -1)[sel]).all(), (key, "non-finite output", np.flatnonzero(~np.isfinite(got.reshape(len(err), -1)).all(axis=1) & sel)[:10])
    bad = sel & ~(err <= bar)
    WORST[key] = max(WORST.get(key, 0.0), float((err / np.maximum(scale, 1e-300))[sel].max(initial=0.0)))
    assert not bad.any(), (key, f"{bad.sum()} rows over the bar, worst error / bar {float((err / bar)[bad].max()):.3g}",
                           np.flatnonzero(bad)[:10])


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    print("\nworst |error| / row scale:", {" ".join(k): f"{v:.2e}" for k, v in sorted(WORST.items())})


# ------------------------------------------------------------------ rotation sets (mpmath, exact)
AXES = ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1), (0.3, -0.5, 0.8))  # the last one generic


def sweep_angles():
    """theta = 0, log-spaced 1e-12..1e-1 and denser over 1e-4..1e-2 (times 1.37, off the powers of ten so that no row
    sits on a kappa cut), generic angles, pi - 10^-k for k = 1..12, pi"""
    a = [M.mpf(0)] + [M.mpf(float(x)) * M.mpf("1.37") for x in np.r_[np.logspace(-12, -1, 23), np.logspace(-4, -2, 21)]]
    a += [M.mpf(x) for x in ("0.3", "1", "2", "2.9")]
    a += [M.pi - M.mpf(10) ** -k for k in range(1, 13)] + [M.pi]
    return a


def edge_rotations(rep, rng):
    """the sweep about five axes, the representation's own singular band, and random rotations"""
    Rs = [ref.rot(k, a) for a in sweep_angles() for k in AXES]
    if rep.startswith("rpy"):
        for dt in DTYPES:  # pitch = +-(pi/2 - delta), delta straddling 10 eps of each dtype, 0 and a few above
            d0 = M.sqrt(20 * ref.EPS[dt])
            for delta in (0, d0 * M.mpf("0.99"), d0 * M.mpf("1.01"), M.mpf("1.3e-3"), M.mpf("5e-3"), M.mpf("0.03")):
                for s in (1, -1):
                    for roll, yaw in ((M.mpf("0.3"), M.mpf("-1.1")), (M.mpf(-2), M.mpf("2.5")), (M.pi, M.mpf("0.5"))):
                        Rs.append(ref.rpy2r(roll, s * (M.pi / 2 - delta), yaw, rep[4:]))
    elif rep == "eul":
        for dt in DTYPES:  # theta at 0 and pi, and 10 eps (1 -+ 1e-2) from them: |R02|, |R12| ~ sin(theta)
            d0 = 10 * M.mpf(ref.EPS[dt])
            for theta in (0, M.pi, d0 * M.mpf("0.99"), d0 * M.mpf("1.01"), M.pi - d0 * M.mpf("0.99"),
                          M.pi - d0 * M.mpf("1.01"), M.mpf("1.3e-3"), M.pi - M.mpf("5e-3")):
                for phi, psi in ((0, M.mpf("0.4")), (M.mpf("0.7"), M.mpf(-2)), (M.mpf(-3), M.mpf(1))):
                    Rs.append(ref.eul2r(phi, theta, psi))
    Rs += [ref.rot(rng.normal(size=3), rng.uniform(0, float(M.pi))) for _ in range(64)]
    return Rs


def exact_kappa(R, rep):
    return ref.kappa(ref.r2x(R, rep), rep)


# ------------------------------------------------------------------ 1. b2k_jacob0_analytical
def run_janalytical(T, J, rep_code, n, N, t_offset=0):
    """Ja of the first N rows (NaN-filled output with guards); T may start t_offset elements past its allocation"""
    dt = T.dtype.type
    Tb = torch.zeros(N * 16 + t_offset, dtype=B.tdtype(T.dtype), device="cuda")
    Tb[t_offset:].copy_(dev(T[:N], dt).reshape(-1))
    Jd = dev(J[:N], dt)
    out = nan_buffer(N * 6 * n, dt)
    Tp = Tb[t_offset:]
    rc = rtb._lib.lib().b2k_jacob0_analytical(B.code(T.dtype), n, B.ptr(Tp), B.ptr(Jd), N, rep_code,
                                               B.ptr(out[GUARD:]), B.stream_ptr(Jd))
    rtb._lib.check(rc)
    return unguard(out, N * 6 * n, f"n={n} N={N}").reshape(N, 6, n)


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("rep", ref.REPS)
def test_jacob0_analytical_edges(rep, dt):
    rng = np.random.default_rng(ref.REPS.index(rep))
    code = ref.REPS.index(rep)
    Rs = edge_rotations(rep, rng)
    E = len(Rs)
    tag = f"{rep} {np.dtype(dt).name}"
    base = np.stack([ref.pose(R, rng.normal(size=3), dt) for R in Rs])
    idx = np.arange(N_BIG) % E
    T = base[idx]  # the edge rows first, then over and over to the ragged last tile
    A, kap = ref.rotvel_inverse_rows(base, rep, dt)
    skip_base = kap > KMAX[dt]
    # the rows left out are those whose exact rotation is past the cut: no row is skipped for rounding
    kex = np.array([exact_kappa(R, rep) for R in Rs])
    assert skip_base.sum() == (kex > KMAX[dt]).sum(), (tag, skip_base.sum(), (kex > KMAX[dt]).sum())
    if rep == "exp":
        assert not skip_base.any()
    else:
        assert skip_base.any() and (~skip_base).sum() >= 150, (tag, skip_base.sum())
    for n in range(1, 11):
        J = rng.normal(size=(N_BIG, 6, n)).astype(dt)
        Ja = run_janalytical(T, J, code, n, N_BIG)
        want = ref.apply_rows(A[idx], J)
        np.testing.assert_array_equal(Ja[:, :3], J[:, :3], err_msg=f"{tag} n={n}: translational rows")
        check_rows(Ja, want, dt, ("jacob0_analytical", rep, np.dtype(dt).name), kap=np.maximum(kap[idx], 1.0),
                   rows=~skip_base[idx])
        # T one element past a 16-byte boundary: the scalar-load path does the same arithmetic
        np.testing.assert_array_equal(run_janalytical(T, J, code, n, N_BIG, t_offset=1), Ja, err_msg=f"{tag} n={n}: unaligned T")
        for N in N_EDGES:
            np.testing.assert_array_equal(run_janalytical(T, J, code, n, N), Ja[:N], err_msg=f"{tag} n={n} N={N}")


# ------------------------------------------------------------------ 2. b2k_p_servo_rpy, b2k_angle_axis / b2k_p_servo
def servo_targets(rng):
    """Tep rows for Te = I: the zyx gimbal band of both dtypes, near identity, the angle-axis cut ln = 1e-6 (1 -+ 1e-2),
    near and exactly half turns, yaw / roll exactly +-pi"""
    Rs = []
    for dt in DTYPES:
        d0 = M.sqrt(20 * ref.EPS[dt])
        for delta in (0, d0 * M.mpf("0.99"), d0 * M.mpf("1.01")):
            for s in (1, -1):
                Rs += [ref.rpy2r(M.mpf("0.3"), s * (M.pi / 2 - delta), M.mpf("-1.1"), "zyx"),
                       ref.rpy2r(M.pi, s * (M.pi / 2 - delta), M.mpf("2.5"), "zyx")]
    for k in AXES:
        Rs += [ref.rot(k, M.mpf(float(a))) for a in np.logspace(-12, -1, 12)]
        Rs += [ref.rot(k, M.asin(M.mpf("5e-7") * f)) for f in (M.mpf("0.99"), M.mpf("1.01"))]  # ln = 2 sin(theta) = 1e-6 (1 -+ 1e-2)
        Rs += [ref.rot(k, M.pi), ref.rot(k, M.pi - M.mpf("1e-3")), ref.rot(k, M.pi - M.mpf("1e-9"))]
    for a, b in ((M.pi, M.mpf("0.4")), (-M.pi, M.mpf("-2")), (M.mpf("0.4"), M.pi), (M.mpf("-1"), -M.pi), (M.pi, M.pi)):
        Rs += [ref.rpy2r(a, M.mpf("0.2"), b, "zyx")]  # roll = a, yaw = b
    return Rs


SERVO = {"rpy": "b2k_p_servo_rpy", "angle-axis": "b2k_p_servo"}


def run_servo(method, Te, Tep, stride, gain, threshold):
    dt = Te.dtype.type
    N = len(Te)
    Ted, Tpd = dev(Te, dt), dev(Tep, dt)
    out = nan_buffer(N * 6, dt)
    arr = torch.full((N + 2 * GUARD,), -7, dtype=torch.int32, device="cuda")
    g = None if gain is None else rtb._lib.dptr(np.ascontiguousarray(gain, dtype=np.float64))
    fn = getattr(rtb._lib.lib(), SERVO[method])
    rtb._lib.check(fn(B.code(Te.dtype), B.ptr(Ted), B.ptr(Tpd), N, stride, g, threshold, B.ptr(out[GUARD:]),
                      B.ptr(arr[GUARD:]), B.stream_ptr(Ted)))
    a = arr.cpu().numpy()
    assert (a[:GUARD] == -7).all() and (a[GUARD + N:] == -7).all()
    return unguard(out, N * 6, method).reshape(N, 6), a[GUARD:GUARD + N]


def run_angle_axis(Te, Tep, stride):
    dt = Te.dtype.type
    N = len(Te)
    Ted, Tpd = dev(Te, dt), dev(Tep, dt)
    out = nan_buffer(N * 6, dt)
    rtb._lib.check(rtb._lib.lib().b2k_angle_axis(B.code(Te.dtype), B.ptr(Ted), B.ptr(Tpd), N, stride, B.ptr(out[GUARD:]),
                                                 B.stream_ptr(Ted)))
    return unguard(out, N * 6, "angle_axis").reshape(N, 6)


def servo_ref(method, Te, Tep, gain, threshold, dt):
    g = 1.0 if gain is None else gain
    if method == "rpy":
        v, arrived, tot, kap = ref.p_servo_rpy(Te, Tep, g, threshold, dt)
    else:
        v, arrived, tot, ln = ref.angle_axis(Te, Tep, g, threshold, dt)
        kap = np.maximum(1.0, 1.0 / np.maximum(ln, 1e-300))  # the axis l / ln of a rounded R: eps / ln
    return v, arrived, tot, kap


@pytest.mark.parametrize("method", ["rpy", "angle-axis"])
def test_servo_edges(method):
    rng = np.random.default_rng(30)
    Rs = servo_targets(rng)
    wrap = [0, 0, 0] + [2 * np.pi] * 3 if method == "rpy" else None
    for dt in DTYPES:
        tag = (SERVO[method], "edges", np.dtype(dt).name)
        # Te = I: Re^T Rep (rpy) and Rep Re^T (angle-axis) are Rep exactly, so the branch the kernel takes is the one
        # the reference computes from Tep
        Tep = np.stack([ref.pose(R, rng.normal(size=3), dt) for R in Rs])
        Te = np.broadcast_to(np.eye(4, dtype=dt), Tep.shape).copy()
        for gain in (None, np.array([1, 2, 3, 0.5, 0.25, 4.0]), np.array([-1.5, 0.1, 7, -3, 1, 0.3])):
            gw = 1.0 if gain is None else gain.astype(dt)
            v, arrived = run_servo(method, Te, Tep, 16, gain, 2.5)
            wv, wa, tot, _ = servo_ref(method, Te, Tep, gain, 2.5, dt)
            check_rows(v, wv, dt, tag, wrap=None if wrap is None else np.abs(np.asarray(wrap) * gw))
            far = np.abs(tot - 2.5) > 8 * TOL[dt][0] * np.maximum(tot, 1)
            assert (arrived[far] == wa[far]).all() and far.sum() > len(far) // 2, tag
            if method == "angle-axis" and gain is None:
                e = run_angle_axis(Te, Tep, 16)
                np.testing.assert_array_equal(e, v, err_msg=f"{tag}: b2k_angle_axis != b2k_p_servo with unit gain")
        # one target for every row (tep_stride 0): each row of Te against Tep[k]
        for k in (0, len(Rs) // 2, len(Rs) - 1):
            Te_r = np.stack([ref.pose(ref.rot(rng.normal(size=3), rng.uniform(0, 3)), rng.normal(size=3), dt) for _ in range(7)])
            v, _ = run_servo(method, Te_r, Tep[k], 0, None, 1.0)
            v16, _ = run_servo(method, Te_r, np.broadcast_to(Tep[k], Te_r.shape).copy(), 16, None, 1.0)
            np.testing.assert_array_equal(v, v16, err_msg=f"{tag}: tep_stride 0 vs 16")
        # arrived at the threshold: pure translations with an exactly representable sum |e| = 0.875, thresholds a
        # few ulps either side of it (sum < threshold is strict)
        Tt = np.broadcast_to(np.eye(4, dtype=dt), (3, 4, 4)).copy()
        Tt[:, :3, 3] = [[0.25, 0.5, 0.125], [-0.5, 0.25, -0.125], [0.875, 0, 0]]
        for k in range(-3, 4):
            thr = float(np.float64(dt(0.875)) + k * float(np.spacing(dt(0.875))))
            _, arrived = run_servo(method, np.broadcast_to(np.eye(4, dtype=dt), Tt.shape).copy(), Tt, 16, None, thr)
            assert (arrived == (1 if k > 0 else 0)).all(), (tag, k, arrived)


@pytest.mark.parametrize("method", ["rpy", "angle-axis"])
def test_servo_random_pairs(method):
    """generic (Te, Tep): Re^T Rep is now rounded in the kernel, so roll / yaw carry kappa = 1/|cos pitch| and the
    angle-axis direction 1/ln (the error of l = vex(R - R^T) is ~ eps absolute); both stay small away from the bands"""
    rng = np.random.default_rng(31)
    N = 513
    Rs = [ref.rot(rng.normal(size=3), rng.uniform(0, float(M.pi))) for _ in range(2 * N)]
    wrap = [0, 0, 0] + [2 * np.pi] * 3 if method == "rpy" else None
    gain = np.array([1, 2, 3, 0.5, 0.25, 4.0])
    for dt in DTYPES:
        tag = (SERVO[method], "random", np.dtype(dt).name)
        Te = np.stack([ref.pose(R, rng.normal(size=3), dt) for R in Rs[:N]])
        Tep = np.stack([ref.pose(R, rng.normal(size=3), dt) for R in Rs[N:]])
        thr = 6.0
        v, arrived = run_servo(method, Te, Tep, 16, gain, thr)
        wv, wa, tot, kap = servo_ref(method, Te, Tep, gain, thr, dt)
        ok = kap <= KMAX[dt]
        assert ok.sum() >= N - 5, (tag, (~ok).sum())
        check_rows(v, wv, dt, tag, kap=kap, wrap=None if wrap is None else np.abs(np.asarray(wrap) * gain.astype(dt)), rows=ok)
        far = np.abs(tot - thr) > 8 * TOL[dt][0] * kap * np.maximum(tot, 1)
        assert (arrived[far] == wa[far]).all() and 0 < arrived.sum() < N, tag


# ------------------------------------------------------------------ 3. b2k_ctraj
def ctraj_ends(rng):
    """(T0, T1) pairs: T0 through every branch of host_r2q (trace > 0; trace <= 0 with R00, R11, R22 largest),
    T1 = T0 Rot(k, delta) for delta from 0 to near 2 pi across the point where the shorter arc flips"""
    T0s = [ref.rot((1, 2, 3), M.mpf("0.7")), ref.rot((1, 0.2, 0.1), M.mpf("2.5")), ref.rot((0.1, 1, 0.2), M.mpf("2.5")),
           ref.rot((0.2, 0.1, 1), M.mpf("2.5"))]
    deltas = [M.mpf(0), M.mpf("1e-16"), M.mpf("1e-14"), M.mpf("1e-8"), M.mpf("1e-4"), M.mpf("1.3"), M.pi - M.mpf("1e-6"),
              M.pi, M.pi + M.mpf("1e-6"), 2 * M.pi - M.mpf("1e-3"), 2 * M.pi - M.mpf("1e-8")]
    pairs = []
    for R0 in T0s:
        for d in deltas:
            R1 = ref.mul(R0, ref.rot(rng.normal(size=3), d))
            pairs.append((ref.pose(R0, rng.normal(size=3)), ref.pose(R1, rng.normal(size=3)), d))
    return pairs


def run_ctraj(T0, T1, s, offset=0):
    dt = s.dtype.type
    N = len(s)
    sd = dev(s, dt)
    out = nan_buffer(N * 16 + offset, dt)
    rtb._lib.check(rtb._lib.lib().b2k_ctraj(B.code(s.dtype), rtb._lib.dptr(np.ascontiguousarray(T0)),
                                            rtb._lib.dptr(np.ascontiguousarray(T1)), B.ptr(sd), N,
                                            B.ptr(out[GUARD + offset:]), B.stream_ptr(sd)))
    b = unguard(out, N * 16 + offset, "ctraj")
    assert np.isnan(b[:offset]).all()
    return b[offset:].reshape(N, 4, 4)


@pytest.mark.parametrize("dt", DTYPES, ids=["f64", "f32"])
def test_ctraj_edges(dt):
    rng = np.random.default_rng(40)
    pairs = ctraj_ends(rng)
    seen_branches = set()
    for T0, _, _ in pairs:
        R = T0[:3, :3]
        tr = np.trace(R)
        seen_branches.add("trace" if tr > 0 else int(np.argmax(np.diag(R))))
    assert seen_branches == {"trace", 0, 1, 2}
    tag = ("ctraj", np.dtype(dt).name)
    s = np.r_[0.0, -0.0, 1e-300, np.finfo(dt).tiny, np.nextafter(dt(1), dt(0)), 1.0, -1e-3, -0.5, 1 + 1e-3, 1.5,
              rng.uniform(0, 1, 40), rng.uniform(-0.2, 1.2, 20)].astype(dt)
    for T0, T1, d in pairs:
        got = run_ctraj(T0, T1, s)
        np.testing.assert_array_equal(run_ctraj(T0, T1, s, offset=1), got, err_msg=f"{tag}: unaligned output")
        want = ref.ctraj(T0, T1, s)
        if abs(ref.ctraj_dot(T0, T1)) < 1e-9:  # a half turn apart: either arc is as short; each row on one of them
            err, scale = row_errors(got, want)
            other, _ = row_errors(got, ref.ctraj(T0, T1, s, other_arc=True))
            rtol, atol = TOL[dt]
            assert (np.minimum(err, other) <= rtol * scale + atol).all(), (tag, float(d))
        else:
            try:
                check_rows(got, want, dt, tag)
            except AssertionError as e:
                raise AssertionError(f"delta = {float(d):.3g}: {e}") from None
