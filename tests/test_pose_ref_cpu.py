"""The pose-representation reference without a GPU: pose_ref.py -- the mpmath restatement test_gpu_pose_edges.py checks
the kernels of b2k_pose.cu and the angle-axis error against -- agrees with the oracle's float64 restatements at generic
rows and satisfies the defining identities in mpmath; and the C entry points of those kernels reject bad arguments with
B2K_ERR_INVALID before any CUDA call."""
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
