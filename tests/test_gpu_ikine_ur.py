"""GPU tests of the closed-form inverse kinematics of UR-type arms (DHRobot.ikine_ur): the device against the numpy
restatement in ikine_ur_ref.py, all eight configurations from one launch, round trips, branch recovery and the
configuration predicates at 1M rows, wrist-singular and straight-elbow rows, out-of-reach rows, input forms, the
unaligned load path and launch counts."""
import os
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_ur_ref as ref  # noqa: E402

ALL = [ref.letters_of(c) for c in range(8)]


def _robots():
    rng = np.random.default_rng(78)
    return [rtb.models.UR10()] + [ref.random_robot(rtb, rng) for _ in range(3)]


ROBOTS = _robots()


def well_conditioned(c, s5, rm, ax):
    """Rows where the joint angles are a well-conditioned function of the pose: 1 - |c3| > 1e-4 (elbow), |sin theta5| >
    1e-2 (wrist), r - |D| > 1e-4 (shoulder), |X| > 1e-4 (the elbow letter's sign(X)).  Nearer to a boundary an ulp of T
    moves the angles by far more than 1e-9; those rows are held to the pose round trip instead."""
    return (c > 1e-4) & (s5 > 1e-2) & (rm > 1e-4) & (ax > 1e-4)


def dev(a, dt=np.float64, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)


def host(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _solve_c(rob, Td, conf):
    """the C entry point on device poses -> q (N,k,6), ok (N,k) on the host"""
    dh = ref.dh_table(rob)
    conf = np.ascontiguousarray(conf, dtype=np.int32)
    N, k = Td.shape[0], len(conf)
    q = torch.empty((N, k, 6), dtype=Td.dtype, device=Td.device)
    ok = torch.empty((N, k), dtype=torch.int32, device=Td.device)
    L = rtb._lib
    L.check(L.lib().b2k_ikine_ur(L.F64 if Td.dtype == torch.float64 else L.F32, L.dptr(dh), L.dptr(np.ascontiguousarray(rob._base)),
                                 L.dptr(np.ascontiguousarray(rob._tool)), Td.data_ptr(), N, k, conf.ctypes.data_as(L.ip),
                                 q.data_ptr(), ok.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return host(q), host(ok).astype(bool)


@pytest.mark.parametrize("N", [1, 31, 32, 33, 1000, 100001])
@pytest.mark.parametrize("k", range(4))
def test_parity_with_the_restatement_fp64(k, N):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(zlib.crc32(f"ur-{k}-{N}".encode()))
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6)))
    got, gok = _solve_c(rob, dev(T), range(8))
    sol = rob.ikine_ur(dev(T), config=ALL)
    np.testing.assert_array_equal(host(sol.q), got)
    assert sol.success == gok.all()
    for code in range(8):
        want, ok = ref.ikine_ur(dh, rob._base, rob._tool, T, code)
        c, s5, rm, ax = ref.margins(dh, rob._base, rob._tool, T, code)
        # away from the reach boundaries (and from the wrist singularity, which moves O4) the two agree on reach
        clear = (np.abs(c) > 1e-6) & (np.abs(rm) > 1e-6) & (s5 > 1e-6)
        assert (gok[clear, code] == ok[clear]).all()
        assert np.isnan(got[~gok[:, code], code]).all() and np.isfinite(got[gok[:, code], code]).all()
        m = ok & well_conditioned(c, s5, rm, ax)
        assert m.sum() >= 0.9 * ok.sum() - 3
        assert np.abs(ref.wrap(got[m, code] - want[m])).max(initial=0) <= 1e-9


@pytest.mark.parametrize("N", [33, 100001])
@pytest.mark.parametrize("k", range(4))
def test_round_trip_fp32(k, N):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(zlib.crc32(f"ur-{k}-{N}-f32".encode()))
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6))).astype(np.float32).astype(np.float64)
    sol = rob.ikine_ur(dev(T, np.float32), config=ALL)
    assert sol.q.dtype == torch.float32
    got = host(sol.q).astype(np.float64)
    for code in range(8):
        c, s5, rm, ax = ref.margins(dh, rob._base, rob._tool, T, code)
        m = (c > 1e-3) & (s5 > 1e-2) & (rm > 1e-3)
        assert m.sum() >= 0.5 * N
        assert np.isfinite(got[m, code]).all()
        assert np.abs(ref.fk(rob, got[m, code]) - T[m]).max() <= 1e-4
    # dtype= on fp64 input selects the fp32 kernel too
    assert rob.ikine_ur(T[:3], dtype=np.float32).q.dtype == np.float32


def test_all_eight_in_one_launch_equal_eight_launches():
    rob = ROBOTS[1]
    rng = np.random.default_rng(3)
    for dt in (np.float64, np.float32):
        Td = dev(ref.fk(rob, rng.uniform(-np.pi, np.pi, (5000, 6))), dt)
        together = host(rob.ikine_ur(Td, config=ALL).q)
        for code, letters in enumerate(ALL):
            one = host(rob.ikine_ur(Td, config=letters).q)
            assert np.array_equal(one.view(np.uint8), np.ascontiguousarray(together[:, code]).view(np.uint8)), letters
        mixed = host(rob.ikine_ur(Td, config=["rdf", "lun", "rdf"]).q)
        assert np.array_equal(mixed[:, 0], together[:, 7], equal_nan=True)
        assert np.array_equal(mixed[:, 1], together[:, 0], equal_nan=True)
        assert np.array_equal(mixed[:, 2], together[:, 7], equal_nan=True)


@pytest.mark.parametrize("k", [0, 2])
def test_million_row_identities_on_the_device(k):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    ets = rob.ets()
    N = 1_000_000
    rng = np.random.default_rng(90 + k)
    qstar = rng.uniform(-np.pi, np.pi, (N, 6))
    Td = ets.eval(dev(qstar))
    T = host(Td)
    sol = rob.ikine_ur(Td, config=ALL)
    assert sol.q.device == Td.device
    codes = ref.config_code(dh, qstar)
    for code in range(8):
        qc = sol.q[:, code]
        okc = ~torch.isnan(qc[:, 0])
        assert okc[torch.from_numpy(codes == code).to(Td.device)].all()  # every pose is reachable in its own configuration
        qok = qc[okc].contiguous()
        assert (ets.eval(qok) - Td[okc]).abs().max().item() <= 1e-12
        # every well-conditioned solution has the letters it was asked for
        keep = well_conditioned(*ref.margins(dh, rob._base, rob._tool, T, code)) & host(okc)
        assert keep.sum() >= 0.5 * N
        assert (ref.config_code(dh, host(qc)[keep]) == code).all()
        # branch recovery: q* comes back from FK(q*) in the configuration of q*
        sel = keep & (codes == code)
        assert np.abs(ref.wrap(host(qc)[sel] - qstar[sel])).max() <= 1e-9


def test_wrist_singular_and_straight_elbow_rows_round_trip():
    for rob in ROBOTS:
        dh = ref.dh_table(rob)
        rng = np.random.default_rng(11)
        q = rng.uniform(-np.pi, np.pi, (4000, 6))
        # theta5 = 0 or pi with theta6 = 0 (the solver's choice there); theta3 = 0 or pi
        q[:2000, 4] = rng.choice([0.0, np.pi], 2000) - dh[4, 3]
        q[:2000, 5] = -dh[5, 3]
        q[2000:, 2] = rng.choice([0.0, np.pi], 2000) - dh[2, 3]
        Td = dev(ref.fk(rob, q))
        codes = ref.config_code(dh, q)
        got = host(rob.ikine_ur(Td, config=ALL).q)
        own = got[np.arange(len(q)), codes]
        ok = np.isfinite(own[:, 0])
        # a straight elbow is reached within the elbow band; at a singular wrist, |u| and |v| above 10 eps from
        # rounding give theta6 from noise, which moves O4 and may put it out of reach
        assert ok[2000:].mean() >= 0.99 and ok[:2000].mean() >= 0.8
        assert np.abs(ref.fk(rob, own[ok]) - host(Td)[ok]).max() <= 1e-12
        for code in range(8):
            fin = np.isfinite(got[:, code, 0])
            assert np.abs(ref.fk(rob, got[fin, code]) - host(Td)[fin]).max() <= 1e-12
    # UR10's named configurations have a straight elbow, and qz a singular wrist
    u = rtb.models.UR10()
    for name in ("qz", "qr"):
        qn = getattr(u, name)
        Tn = u.fkine(qn).A
        letters = ref.config_of(ref.dh_table(u), qn)[0]
        for dt in (np.float64, np.float32):
            sol = u.ikine_ur(Tn, config=letters, dtype=dt)
            assert sol.success, (name, dt)
            np.testing.assert_allclose(u.fkine(sol.q.astype(np.float64)).A, Tn, atol=1e-12 if dt == np.float64 else 1e-4)
            # at a straight elbow theta3 = acos(c3) moves by sqrt(2 |dc3|): a few eps of c3 give 1e-8 in fp64, 1e-3 in fp32
            np.testing.assert_allclose(ref.wrap(sol.q - qn), 0, atol=1e-7 if dt == np.float64 else 2e-3)


def _mixed_batch(rob, rng, N=4000):
    """FK poses with rows moved onto the first axis (r < |D|) and rows moved beyond reach (|c3| > 1)"""
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6)))
    kind = rng.integers(0, 3, N)
    T[kind == 1, :3, 3] = (0.01, 0.0, 0.5)
    T[kind == 2, :3, 3] = (2.5, 0.5, 0.5) * rng.uniform(0.9, 1.1, ((kind == 2).sum(), 1))
    return T, kind


def test_out_of_reach_rows_get_nan_and_ok_zero():
    rob = rtb.models.UR10()
    dh = ref.dh_table(rob)
    T, kind = _mixed_batch(rob, np.random.default_rng(4))
    N = len(T)
    Td = dev(T)
    q, ok = _solve_c(rob, Td, range(8))
    bad = kind != 0
    assert not ok[bad].any() and np.isnan(q[bad]).all()
    for code in range(8):
        want_ok = ref.ikine_ur(dh, rob._base, rob._tool, T, code)[1]
        assert (ok[:, code] == want_ok).all()
        assert np.isnan(q[~ok[:, code], code]).all() and np.isfinite(q[ok[:, code], code]).all()
    sol = rob.ikine_ur(Td, config=ALL)
    assert not sol.success and sol.reason == f"Out of reach: {8 * N - ok.sum()} of {8 * N} solutions"
    single = rob.ikine_ur(T)  # numpy, one configuration
    assert not single.success and single.reason == f"Out of reach: {N - ok[:, 0].sum()} of {N} rows"
    one = rob.ikine_ur(T[kind == 2][0])
    assert not one.success and one.reason == "Out of reach" and one.q.shape == (6,) and np.isnan(one.q).all()
    one = rob.ikine_ur(T[kind == 1][0], config="rdf")
    assert not one.success and one.reason == "Out of reach"


def test_placement_and_input_forms():
    rob = rtb.models.UR10()
    rng = np.random.default_rng(5)
    q0 = rng.uniform(-np.pi, np.pi, (50, 6))
    T = ref.fk(rob, q0)
    letters = ref.config_of(ref.dh_table(rob), q0[7])[0]
    ref_q = host(rob.ikine_ur(dev(T), config=letters).q)
    got = rob.ikine_ur(T, config=letters)
    assert isinstance(got.q, np.ndarray) and got.q.shape == (50, 6)
    np.testing.assert_array_equal(got.q, ref_q)
    np.testing.assert_array_equal(rob.ikine_ur(rtb.SE3(T), config=letters).q, ref_q)
    for one in (rob.ikine_ur(rtb.SE3(T[7]), config=letters), rob.ikine_ur(T[7], config=letters)):
        assert one.success and one.reason == "Success" and one.q.shape == (6,)
        np.testing.assert_array_equal(one.q, ref_q[7])
    np.testing.assert_allclose(ref.wrap(ref_q[7] - q0[7]), 0, atol=1e-9)
    assert rob.ikine_ur(T[7], config=["lun", "rdn"]).q.shape == (2, 6)
    Td = dev(T)
    t = rob.ikine_ur(Td, config=letters).q
    assert isinstance(t, torch.Tensor) and t.device == Td.device and t.shape == (50, 6)
    if torch.cuda.device_count() < 2:
        return
    torch.cuda.set_device(0)
    d1 = rob.ikine_ur(dev(T, device="cuda:1"), config=letters).q
    assert d1.device == torch.device("cuda:1")
    np.testing.assert_array_equal(host(d1), ref_q)


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
def test_unaligned_poses_take_the_element_load_path(dt):
    """T one element past a 16-byte boundary cannot use the 16-byte loads; the element loads give the same q"""
    rob = ROBOTS[2]
    rng = np.random.default_rng(6)
    N = 1000
    Td = dev(ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6)))).to(dt)
    buf = torch.empty(N * 16 + 1, dtype=dt, device=Td.device)
    Tu = buf[1:].view(N, 4, 4)
    Tu.copy_(Td)
    assert Tu.data_ptr() % 16 != 0 and Td.data_ptr() % 16 == 0
    a = host(rob.ikine_ur(Td, config=ALL).q)
    b = host(rob.ikine_ur(Tu, config=ALL).q)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_one_launch_per_call():
    rob = ROBOTS[3]
    rng = np.random.default_rng(7)
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (300, 6)))
    Td = dev(T)
    for args in ((Td, ALL), (Td, "lun"), (T, ["ruf", "ldn"]), (T[0], "lun")):
        torch.cuda.synchronize()
        n0 = rtb.launch_count()
        rob.ikine_ur(*args)
        torch.cuda.synchronize()
        assert rtb.launch_count() - n0 == 1, args
