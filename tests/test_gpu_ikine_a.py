"""GPU tests of the closed-form inverse kinematics (DHRobot.ikine_a, reference DHRobot.ikine_6s / Puma560.ikine_a): the
device against the numpy restatement in ikine_a_ref.py, all eight configurations from one launch, round trips, branch
recovery and the configuration predicates at 1M rows, out-of-reach rows, placement and launch counts."""
import os
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_a_ref as ref  # noqa: E402

ALL = [ref.letters_of(c) for c in range(8)]


def _robots():
    rng = np.random.default_rng(77)
    return [rtb.models.Puma560()] + [ref.random_robot(rtb, rng, s) for s in (1, -1, 1)]


ROBOTS = _robots()


def well_conditioned(c, s5, rm):
    """Rows where the joint angles are a well-conditioned function of the pose: 1 - |c| > 1e-4 (elbow), |sin theta5| >
    1e-2 (wrist), r - |D| > 1e-4 (shoulder).  Nearer to one of these boundaries -- above all near two at once -- a
    perturbation of T by an ulp moves the restatement's own angles by up to 2e-7 at 1M rows, so no implementation can
    match it to 1e-9 there; those rows are held to the pose round trip instead."""
    return (c < 1 - 1e-4) & (s5 > 1e-2) & (rm > 1e-4)


def dev(a, dt=np.float64, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)


def host(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


@pytest.mark.parametrize("N", [1, 31, 33, 1000, 100001])
@pytest.mark.parametrize("k", range(4))
def test_parity_with_the_restatement_fp64(k, N):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(zlib.crc32(f"{k}-{N}".encode()))
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6)))
    sol = rob.ikine_a(dev(T), config=ALL)
    assert sol.success and sol.reason == "Success"
    got = host(sol.q)
    assert got.shape == (N, 8, 6)
    for code in range(8):
        want, ok = ref.ikine_a(dh, rob._base, rob._tool, T, code)
        m = well_conditioned(*ref.margins(dh, rob._base, rob._tool, T, code))
        assert m.sum() >= 0.9 * N - 3
        assert np.abs(ref.wrap(got[m, code] - want[m])).max(initial=0) <= 1e-9


@pytest.mark.parametrize("N", [33, 100001])
@pytest.mark.parametrize("k", range(4))
def test_round_trip_fp32(k, N):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(zlib.crc32(f"{k}-{N}-f32".encode()))
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6))).astype(np.float32).astype(np.float64)
    sol = rob.ikine_a(dev(T, np.float32), config=ALL)
    assert sol.q.dtype == torch.float32
    got = host(sol.q).astype(np.float64)
    for code in range(8):
        c, s5, rm = ref.margins(dh, rob._base, rob._tool, T, code)
        # rm: a wrist centre within fp32 rounding of the cylinder r = |D| may come out of reach in fp32
        m = (c < 0.999) & (s5 > 1e-2) & (rm > 1e-4)
        assert m.sum() >= 0.8 * N
        assert np.abs(ref.fk(rob, got[m, code]) - T[m]).max() <= 1e-4
    # dtype= on fp64 input selects the fp32 kernel too
    assert rob.ikine_a(T[:3], dtype=np.float32).q.dtype == np.float32


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_all_eight_in_one_launch_equal_eight_launches(dt):
    rob = ROBOTS[1]
    rng = np.random.default_rng(3)
    Td = dev(ref.fk(rob, rng.uniform(-np.pi, np.pi, (5000, 6))), dt)
    together = host(rob.ikine_a(Td, config=ALL).q)
    for code, letters in enumerate(ALL):
        one = host(rob.ikine_a(Td, config=letters).q)
        assert np.array_equal(one.view(np.uint8), np.ascontiguousarray(together[:, code]).view(np.uint8)), letters
    # any order and repetition of configurations
    mixed = host(rob.ikine_a(Td, config=["rdf", "lun", "rdf"]).q)
    assert np.array_equal(mixed[:, 0], together[:, 7]) and np.array_equal(mixed[:, 1], together[:, 0])
    assert np.array_equal(mixed[:, 2], together[:, 7])


@pytest.mark.parametrize("k", [0, 2])
def test_million_row_identities_on_the_device(k):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    ets = rob.ets()
    N = 1_000_000
    rng = np.random.default_rng(90 + k)
    qstar = rng.uniform(-np.pi, np.pi, (N, 6))
    Td = ets.eval(dev(qstar))
    sol = rob.ikine_a(Td, config=ALL)
    assert sol.success and sol.q.device == Td.device
    for code in range(8):
        qc = sol.q[:, code].contiguous()
        assert (ets.eval(qc) - Td).abs().max().item() <= 1e-12
        assert (ref.config_code(dh, host(qc)) == code).all()  # every solution has the letters it was asked for
    # branch recovery: q* comes back from FK(q*) and the configuration of q*
    codes = ref.config_code(dh, qstar)
    T = host(Td)
    for code in range(8):
        sel = codes == code
        keep = well_conditioned(*ref.margins(dh, rob._base, rob._tool, T[sel], code))
        got = host(rob.ikine_a(Td[torch.from_numpy(sel).to(Td.device)], config=ALL[code]).q)
        assert np.abs(ref.wrap(got - qstar[sel]))[keep].max() <= 1e-9


def _mixed_batch(rob, rng, N=4000):
    """FK poses with rows moved onto the shoulder axis (r < |D|) and rows moved beyond reach (|c| > 1)"""
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (N, 6)))
    kind = rng.integers(0, 3, N)
    T[kind == 1, :3, 3] = (0.05, 0.0, 0.67)
    T[kind == 2, :3, 3] = (2.0, 0.0, 0.67) * rng.uniform(0.9, 1.1, ((kind == 2).sum(), 1))
    return T, kind


def test_out_of_reach_rows_get_nan_and_ok_zero():
    rob = rtb.models.Puma560()
    dh = ref.dh_table(rob)
    T, kind = _mixed_batch(rob, np.random.default_rng(4))
    N = len(T)
    Td = dev(T)
    sol = rob.ikine_a(Td, config=ALL)
    q = host(sol.q)
    bad = kind != 0
    assert not sol.success and sol.reason == f"Out of reach: {8 * bad.sum()} of {8 * N} solutions"
    assert np.isnan(q[bad]).all() and np.isfinite(q[~bad]).all()
    single = rob.ikine_a(T)  # numpy, one configuration
    assert not single.success and single.reason == f"Out of reach: {bad.sum()} of {N} rows"
    # the ok flags of the C entry point, against the restatement's
    conf = np.arange(8, dtype=np.int32)
    qo = torch.empty((N, 8, 6), dtype=torch.float64, device="cuda")
    ok = torch.empty((N, 8), dtype=torch.int32, device="cuda")
    rtb._lib.check(rtb._lib.lib().b2k_ikine_6s(rtb._lib.F64, rtb._lib.dptr(np.ascontiguousarray(dh)), None, None, Td.data_ptr(), N, 8,
                                               conf.ctypes.data_as(rtb._lib.ip), qo.data_ptr(), ok.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
    ok = host(ok)
    for code in range(8):
        assert (ok[:, code] == (kind == 0)).all()
        assert (ref.ikine_a(dh, rob._base, rob._tool, T, code)[1] == (kind == 0)).all()
    one = rob.ikine_a(T[kind == 2][0])
    assert not one.success and one.reason == "Out of reach" and one.q.shape == (6,) and np.isnan(one.q).all()
    one = rob.ikine_a(T[kind == 1][0], config="rdf")
    assert not one.success and one.reason == "Out of reach"


def test_placement_and_input_forms():
    rob = rtb.models.Puma560()
    rng = np.random.default_rng(5)
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (50, 6)))
    ref_q = host(rob.ikine_a(dev(T), config="rdn").q)
    got = rob.ikine_a(T, config="rdn")
    assert isinstance(got.q, np.ndarray) and got.q.shape == (50, 6)
    np.testing.assert_array_equal(got.q, ref_q)
    np.testing.assert_array_equal(rob.ikine_a(rtb.SE3(T), config="rdn").q, ref_q)
    one = rob.ikine_a(rtb.SE3(T[7]), config="dr")
    assert one.success and one.reason == "Success" and one.q.shape == (6,)
    np.testing.assert_array_equal(one.q, ref_q[7])
    assert rob.ikine_a(T[7], config=["lun", "rdn"]).q.shape == (2, 6)
    # the reference's own test: fkine(ikine_a(fkine(qn), "lun").q) == fkine(qn)
    Tn = rob.fkine(rob.qn).A
    np.testing.assert_allclose(rob.fkine(rob.ikine_a(Tn, "lun").q).A, Tn, atol=1e-12)
    if torch.cuda.device_count() < 2:
        return
    torch.cuda.set_device(0)
    d1 = rob.ikine_a(dev(T, device="cuda:1"), config="rdn").q
    assert d1.device == torch.device("cuda:1")
    np.testing.assert_array_equal(host(d1), ref_q)


def test_one_launch_per_call():
    rob = ROBOTS[3]
    rng = np.random.default_rng(6)
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (300, 6)))
    Td = dev(T)
    for args in ((Td, ALL), (Td, "lun"), (T, ["ruf", "ldn"]), (T[0], "lun")):
        torch.cuda.synchronize()
        n0 = rtb.launch_count()
        rob.ikine_a(*args)
        torch.cuda.synchronize()
        assert rtb.launch_count() - n0 == 1, args
