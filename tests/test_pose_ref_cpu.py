"""The pose-representation reference without a GPU: pose_ref.py -- the mpmath restatement test_gpu_pose_edges.py checks
the kernels of b2k_pose.cu and the angle-axis error against -- agrees with the oracle's float64 restatements at generic
rows and satisfies the defining identities in mpmath; and the C entry points of those kernels reject bad arguments with
B2K_ERR_INVALID before any CUDA call."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import b2kin as rtb
from oracle import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pose_ref as ref  # noqa: E402

M = ref.M


def random_rotations(rng, N):
    """N rotations about random axes by angles in [0.1, pi - 0.1], in mpmath"""
    return [ref.rot(rng.normal(size=3), rng.uniform(0.1, np.pi - 0.1)) for _ in range(N)]


def generic(Rs, rep):
    """rows away from the representation's singularity, where both restatements are well-conditioned"""
    return [R for R in Rs if ref.kappa(ref.r2x(R, rep), rep) < 10]


def test_reference_matches_the_oracle_at_generic_rows():
    rng = np.random.default_rng(0)
    Rs = random_rotations(rng, 40)
    for rep in ref.REPS:
        rows = generic(Rs, rep)
        assert len(rows) >= 20, rep
        for Rm in rows:
            R = ref.to_np(Rm)
            g = ref.r2x(R, rep)
            np.testing.assert_allclose([float(x) for x in g], orc.r2x(R, rep), rtol=0, atol=1e-12, err_msg=rep)
            A = np.array([[float(x) for x in r] for r in ref.rotvel_inverse(g, rep)])
            np.testing.assert_allclose(A, orc.rotvelxform_inv(orc.r2x(R, rep), rep), rtol=0, atol=1e-12 * np.abs(A).max())
        T = np.stack([ref.pose(Rm, rng.normal(size=3)) for Rm in rows])
        J = rng.normal(size=(len(T), 6, 7))
        Ja, kap = ref.jacob0_analytical(T, J, rep)
        want = orc.jacob0_analytical(T, J, rep)
        assert (kap < 10).all()
        np.testing.assert_allclose(Ja, want, rtol=0, atol=1e-12 * np.abs(want).max(), err_msg=rep)
    Te = np.stack([ref.pose(R, rng.normal(size=3)) for R in Rs[:20]])
    Tep = np.stack([ref.pose(R, rng.normal(size=3)) for R in Rs[20:]])
    gain = np.array([1, 2, 3, 0.5, 0.25, 4.0])
    thr = float(np.median(ref.p_servo_rpy(Te, Tep, gain, 0.0)[2]))
    v, arrived, tot, kap = ref.p_servo_rpy(Te, Tep, gain, thr)
    wv, wa = orc.p_servo_rpy(Te, Tep, gain, thr)
    ok = kap < 10
    assert ok.sum() >= 10
    d = (v - wv)[ok]
    d[:, 3:] = (d[:, 3:] / gain[3:] + np.pi) % (2 * np.pi) - np.pi  # roll / yaw at +-pi: either side is the same angle
    assert np.abs(d).max() < 1e-12
    far = np.abs(tot - thr) > 1e-9
    assert (arrived == wa)[far].all() and 0 < arrived.sum() < len(Te)
    e, _, _, _ = ref.angle_axis(Te, Tep)
    np.testing.assert_allclose(e, np.stack([orc.angle_axis(a, b) for a, b in zip(Te, Tep)]), rtol=0, atol=1e-12)
    s = np.r_[0.0, 1.0, -0.5, 1.5, rng.uniform(0, 1, 20)]
    for k in range(5):
        np.testing.assert_allclose(ref.ctraj(Te[k], Tep[k], s), orc.ctraj_poses(Te[k], Tep[k], s), rtol=0, atol=1e-12)


@pytest.mark.parametrize("rep", ref.REPS)
def test_representation_round_trips_in_mpmath(rep):
    """R -> Gamma -> R on exact rotations outside the singular bands (to 1e-30), and on the bands' own branches (rpy at
    pitch +-pi/2, eul at theta 0 and pi, exp at pi) where the representation is still one of R -- to 1e-20 there: those
    branches take asin at 1 or the square root of (R_ii + 1) / 2 at 0, which turn 50 digits into 25"""
    rng = np.random.default_rng(1)
    Rs = random_rotations(rng, 12)
    if rep == "exp":
        Rs += [ref.rot((1, 2, 3), 0), ref.rot((1, 2, 3), 1e-8)]
    if rep.startswith("rpy"):
        band = [ref.rpy2r(0.3, s * M.pi / 2, -1.1, rep[4:]) for s in (1, -1)]
    elif rep == "eul":
        band = [ref.eul2r(0.4, 0, 0.9), ref.eul2r(0.4, M.pi, 0.9)]
    else:
        band = [ref.rot((1, 2, 3), M.pi), ref.rot((1, 0, 0), M.pi), ref.rot((1, 1, 1), M.pi)]
    for R, tol in [(R, 1e-30) for R in Rs] + [(R, 1e-20) for R in band]:
        back = ref.x2r(ref.r2x(R, rep), rep)
        assert max(abs(back[i][j] - R[i][j]) for i in range(3) for j in range(3)) < tol, rep


@pytest.mark.parametrize("rep", ref.REPS)
def test_rotvel_inverse_inverts_rotvelxform(rep):
    rng = np.random.default_rng(2)
    gs = [rng.uniform(-3, 3, 3) for _ in range(10)]
    if rep == "exp":  # every angle scale down to the smallest, and a half turn
        gs += [v / np.linalg.norm(v) * th for v, th in zip(rng.normal(size=(12, 3)), np.r_[np.logspace(-12, -1, 11), np.pi])]
    for g in gs:
        A, Ai = ref.rotvelxform(g, rep), ref.rotvel_inverse(g, rep)
        P = ref.mul(Ai, A)
        assert max(abs(P[i][j] - (i == j)) for i in range(3) for j in range(3)) < 1e-30, (rep, g)


def test_k2_matches_its_series():
    """Where both apply, the closed form from x cot x and the series agree to the series' first omitted term,
    theta^8 / 47900160; at theta = 0 the closed form is the limit 1/12."""
    for th in np.logspace(-9, -1, 33):
        d = abs(ref.k2(th) - ref.k2_series(th))
        assert d <= 1.01 * M.mpf(th) ** 8 / 47900160 + M.mpf(10) ** -45, th
    assert ref.k2(0) == M.mpf(1) / 12
    assert abs(ref.k2(M.pi) - 1 / M.pi ** 2) < M.mpf(10) ** -45  # x = pi/2: cot x = 0


def test_branch_predicates_follow_the_dtype():
    """A rotation between the fp32 and the fp64 thresholds takes each dtype's own branch."""
    R = ref.to_np(ref.rot((0.3, -0.2, 0.9), 1e-7))  # ln = 2e-7: above fp64's 1e-9, below fp32's 1e-6
    assert all(x == 0 for x in ref.trlog(R, np.float32)) and abs(ref.trlog(R, np.float64)[2]) > 9e-8
    R = ref.to_np(ref.rpy2r(0.3, M.pi / 2 - 1e-5, 0.2, "zyx"))  # |R20| = 1 - 5e-11: inside 10 eps of fp32 only
    assert ref.tr2rpy(R, "zyx", np.float32)[0] == 0 and ref.tr2rpy(R, "zyx", np.float64)[0] != 0


# ------------------------------------------------------------------ the C ABI validates before launching
def _launches_nothing(call, msg):
    lib = rtb._lib.lib()
    n0 = lib.b2k_launch_count()
    assert call(lib) == -1
    assert msg in lib.b2k_last_error(), lib.b2k_last_error()
    assert lib.b2k_launch_count() == n0


P = np.zeros(64)  # stands in for a (never dereferenced) device pointer
p = P.ctypes.data


@pytest.mark.parametrize("n", [-1, 0, 11])
def test_jacob0_analytical_rejects_a_bad_joint_count(n):
    _launches_nothing(lambda lib: lib.b2k_jacob0_analytical(1, n, p, p, 4, 3, p, None), b"n must be")


@pytest.mark.parametrize("rep", [-1, 4, 99])
def test_jacob0_analytical_rejects_a_bad_representation(rep):
    _launches_nothing(lambda lib: lib.b2k_jacob0_analytical(1, 7, p, p, 4, rep, p, None), b"representation")


@pytest.mark.parametrize("args", [(-1, p, p, p), (4, None, p, p), (4, p, None, p), (4, p, p, None)])
def test_jacob0_analytical_rejects_bad_rows_or_pointers(args):
    N, T, J, Ja = args
    _launches_nothing(lambda lib: lib.b2k_jacob0_analytical(1, 7, T, J, N, 0, Ja, None), b"bad arguments")


def test_jacob0_analytical_rejects_a_bad_dtype():
    _launches_nothing(lambda lib: lib.b2k_jacob0_analytical(7, 7, p, p, 4, 0, p, None), b"dtype")


@pytest.mark.parametrize("stride", [-16, 1, 4, 15, 17, 32])
def test_p_servo_rpy_rejects_a_bad_target_stride(stride):
    _launches_nothing(lambda lib: lib.b2k_p_servo_rpy(1, p, p, 4, stride, None, 0.1, p, p, None), b"tep_stride")


@pytest.mark.parametrize("args", [(-1, p, p, p, p), (4, None, p, p, p), (4, p, None, p, p), (4, p, p, None, p),
                                  (4, p, p, p, None)])
def test_p_servo_rpy_rejects_bad_rows_or_pointers(args):
    N, Te, Tep, v, arrived = args
    _launches_nothing(lambda lib: lib.b2k_p_servo_rpy(1, Te, Tep, N, 16, None, 0.1, v, arrived, None), b"bad arguments")


@pytest.mark.parametrize("which", ["T0", "T1"])
def test_ctraj_rejects_a_null_end_pose(which):
    T = np.eye(4)
    dp = rtb._lib.dptr
    T0, T1 = (None, dp(T)) if which == "T0" else (dp(T), None)
    _launches_nothing(lambda lib: lib.b2k_ctraj(1, T0, T1, p, 4, p, None), b"NULL")


@pytest.mark.parametrize("args", [(-1, p, p), (4, None, p), (4, p, None)])
def test_ctraj_rejects_bad_rows_or_pointers(args):
    N, s, out = args
    T = np.eye(4)
    dp = rtb._lib.dptr
    _launches_nothing(lambda lib: lib.b2k_ctraj(1, dp(T), dp(T), s, N, out, None), b"bad arguments")


# ---- the eight pose-error and trajectory entry points on one table of bad arguments.  Each call has valid arguments
# except the ones a case names; a host buffer stands in for the (never dereferenced) device arrays.  Without a device, a
# call that reached the CUDA runtime would report a CUDA error instead.
POSE_SIG = {"b2k_angle_axis": "dtype Te Tep N tep_stride e",
            "b2k_p_servo": "dtype Te Tep N tep_stride gain threshold v arrived",
            "b2k_p_servo_rpy": "dtype Te Tep N tep_stride gain threshold v arrived",
            "b2k_jacob0_analytical": "dtype n T J N representation Ja",
            "b2k_jtraj": "dtype n q0 qf qd0 qd1 N t tscal q qd qdd",
            "b2k_mtraj": "dtype kind n q0 qf qd0 qdf V N t tf s sd sdd tblend",
            "b2k_ctraj": "dtype T0 T1 s N T",
            "b2k_mstraj": "dtype n npieces row0 rows kind tscal t0 dt coef N q"}
# the device arrays in the order they are checked, and the required ones; the host tables that must not be NULL; the
# entry point's own scalars as (name, bad value, good value); nmax: the joint-count range, None: no joint count
POSE_DEV = {"b2k_angle_axis": "Te Tep e", "b2k_p_servo": "Te Tep v arrived", "b2k_p_servo_rpy": "Te Tep v arrived",
            "b2k_jacob0_analytical": "T J Ja", "b2k_jtraj": "t q qd qdd", "b2k_mtraj": "t s sd sdd", "b2k_ctraj": "s T",
            "b2k_mstraj": "q"}
POSE_OPTIONAL = ("t", "qd", "qdd", "sd", "sdd")
POSE_HOST = {"b2k_jtraj": "q0 qf", "b2k_mtraj": "q0 qf", "b2k_ctraj": "T0 T1", "b2k_mstraj": "row0 rows kind tscal t0 dt coef"}
POSE_SCALARS = {"b2k_angle_axis": [("tep_stride", 1, 16)], "b2k_p_servo": [("tep_stride", 32, 16)],
                "b2k_p_servo_rpy": [("tep_stride", -16, 16)], "b2k_jacob0_analytical": [("representation", 4, 0)],
                "b2k_jtraj": [("tscal", 0.0, 1.0)], "b2k_mtraj": [("kind", 2, 0), ("tf", 0.0, 3.0)]}
POSE_NMAX = {"b2k_jacob0_analytical": 10, "b2k_jtraj": 10, "b2k_mtraj": 10, "b2k_mstraj": 16}
_HOST = np.zeros(64)  # q0, qf, T0, T1 and the mstraj tables of fp64
_HD = _HOST.ctypes.data_as(rtb._lib.dp)


def _pose_call(fn, **kw):
    """fn's status and message; row0 / rows / kind of b2k_mstraj are numpy arrays (one piece of N rows by default)"""
    lib = rtb._lib.lib()
    a = dict(dtype=1, n=4, N=4, tep_stride=16, gain=None, threshold=0.1, representation=0, qd0=None, qd1=None, qdf=None,
             V=None, tblend=None, tscal=1.0, kind=0, tf=3.0, npieces=1, q0=_HD, qf=_HD, T0=_HD, T1=_HD, t0=_HD, dt=_HD,
             coef=_HD)
    a.update({d: p for d in "Te Tep e v arrived T J Ja t q qd qdd s sd sdd".split()})
    if fn == "b2k_mstraj":
        a.update(tscal=_HD, row0=np.zeros(1, np.int64), rows=np.array([max(kw.get("N", 4), 0)], np.int64),
                 kind=np.zeros(1, np.int32))
    a.update(kw)
    if fn == "b2k_mstraj":
        for k, ct in (("row0", C.c_int64), ("rows", C.c_int64), ("kind", C.c_int32)):
            if isinstance(a[k], np.ndarray):
                a[k] = a[k].ctypes.data_as(C.POINTER(ct))
    n0 = lib.b2k_launch_count()
    rc = getattr(lib, fn)(*[a[k] for k in POSE_SIG[fn].split()], None)
    assert lib.b2k_launch_count() == n0, fn
    return rc, lib.b2k_last_error().decode()


def _pose_cases():
    """(fn, case, arguments, what the message says; None: the call is accepted)"""
    for fn in POSE_SIG:
        dev = POSE_DEV[fn].split()
        yield fn, "dtype 2", dict(dtype=2), "dtype"
        if fn in POSE_NMAX:
            for n in (-1, 0, POSE_NMAX[fn] + 1):
                yield fn, f"n {n}", dict(n=n), "n must be"
        yield fn, "N -1", dict(N=-1), "N is negative"
        for name, bad, _ in POSE_SCALARS.get(fn, []):
            yield fn, f"{name} {bad}", {name: bad}, name
        for name in POSE_HOST.get(fn, "").split():
            yield fn, f"{name} NULL", {name: None}, f"{name} is NULL"
            yield fn, f"N 0, {name} NULL", {name: None, "N": 0}, f"{name} is NULL"
        for name in dev:
            if name not in POSE_OPTIONAL:
                yield fn, f"{name} NULL", {name: None}, f"{name} is NULL"
            for dt, half in ((0, 2), (1, 4)):
                yield fn, f"{name} fp{32 * (dt + 1)} +{half}", {"dtype": dt, name: p + (2 if name == "arrived" else half)}, \
                    f"{name} is not aligned"
        yield fn, "N 0, misaligned", {"N": 0, dev[0]: p + 4}, f"{dev[0]} is not aligned"
        yield fn, "N 0, every device array NULL", {"N": 0, **{d: None for d in dev}}, None
        yield fn, "N 0, fp32", dict(N=0, dtype=0), None
    for name, bad in (("npieces", dict(npieces=0)), ("piece 0", dict(row0=np.ones(1, np.int64))),
                      ("piece 0", dict(kind=np.full(1, 2, np.int32))), ("piece 0", dict(rows=np.full(1, -1, np.int64))),
                      ("cover", dict(rows=np.full(1, 3, np.int64)))):
        yield "b2k_mstraj", f"{name}: {bad}", bad, name
    # b2k_mtraj's trapezoidal profiles that do not exist, after the argument check; axis 2 is the one out of range
    qf, V = np.ones(4), np.array([np.nan, 0.5, 0.1, np.nan])
    yield "b2k_mtraj", "V too small", dict(N=0, kind=1, qf=qf.ctypes.data_as(rtb._lib.dp), V=V.ctypes.data_as(rtb._lib.dp)), \
        "b2k_mtraj: axis 2: V too small"
    V2 = np.array([np.nan, 0.5, 0.9, np.nan])
    yield "b2k_mtraj", "V too big", dict(N=4, kind=1, qf=qf.ctypes.data_as(rtb._lib.dp), V=V2.ctypes.data_as(rtb._lib.dp)), \
        "b2k_mtraj: axis 2: V too big"


POSE_CASES = list(_pose_cases())


@pytest.mark.parametrize("fn, case, kw, want", POSE_CASES, ids=[f"{c[0]}-{c[1]}" for c in POSE_CASES])
def test_pose_entry_points_reject_bad_arguments_before_any_cuda_call(fn, case, kw, want):
    rc, msg = _pose_call(fn, **kw)
    if want is None:
        assert rc == 0, msg
    else:
        assert rc == -1 and msg.startswith(fn + ":") and want in msg, msg


@pytest.mark.parametrize("fn", POSE_SIG)
def test_pose_entry_points_check_in_one_order(fn):
    """dtype, n, N, the entry point's scalars, host tables, required device arrays, alignment: with every defect present
    the first one is reported, and repairing it reports the next."""
    dev = POSE_DEV[fn].split()
    args = dict(dtype=2, n=0, N=-1, **{k: bad for k, bad, _ in POSE_SCALARS.get(fn, [])},
                **{k: None for k in POSE_HOST.get(fn, "").split()},
                **{d: (p + 2 if d in POSE_OPTIONAL else None) for d in dev})
    steps = [({}, "dtype"), (dict(dtype=1), "n must be" if fn in POSE_NMAX else "N is negative")]
    if fn in POSE_NMAX:
        steps.append((dict(n=4), "N is negative"))
    fix = dict(N=4)
    for name, _, good in POSE_SCALARS.get(fn, []):
        steps.append((fix, name))
        fix = {name: good}
    tables = dict(row0=np.zeros(1, np.int64), rows=np.full(1, 4, np.int64), kind=np.zeros(1, np.int32))
    for name in POSE_HOST.get(fn, "").split():
        steps.append((fix, f"{name} is NULL"))
        fix = {name: tables[name] if fn == "b2k_mstraj" and name in tables else _HD}
    if fn == "b2k_mstraj":
        steps += [(dict(fix, npieces=0), "npieces"), (dict(npieces=1, row0=np.ones(1, np.int64)), "piece 0"),
                  (dict(row0=np.zeros(1, np.int64), rows=np.full(1, 3, np.int64)), "cover")]
        fix = dict(rows=np.full(1, 4, np.int64))
    for name in dev:
        if name not in POSE_OPTIONAL:
            steps.append((fix, f"{name} is NULL"))
            fix = {name: p + 2}
    for name in dev:
        steps.append((fix, f"{name} is not aligned"))
        fix = {name: p}
    for fix, want in steps:
        args.update(fix)
        rc, msg = _pose_call(fn, **args)
        assert rc == -1 and msg.startswith(fn + ":") and want in msg, (want, msg)
