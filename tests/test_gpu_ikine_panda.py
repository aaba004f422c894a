"""GPU tests of the closed-form inverse kinematics of Panda-type arms at a given q7 (DHRobot.ikine_panda): the device
against the numpy restatement in ikine_panda_ref.py, all eight configurations from one launch, round trips, branch
recovery and the configuration predicates at 1M rows, per-row q7, singular-shoulder and degenerate-wrist rows,
out-of-reach rows, input forms, the unaligned load path, launch counts, and the iterative ik_LM as an independent
check."""
import os
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ikine_panda_ref as ref  # noqa: E402

ALL = [ref.letters_of(c) for c in range(8)]
h = np.pi / 2


def _robots():
    rng = np.random.default_rng(79)
    return [rtb.models.PandaMDH()] + [ref.random_robot(rtb, rng) for _ in range(3)]


ROBOTS = _robots()


def well_conditioned(el, wr, sh, hh):
    """Rows where the joint angles are a well-conditioned function of the pose: 1 - |C/rho| > 1e-4 (elbow), 1 - |p/h| >
    1e-4 (wrist), |sin theta2| > 1e-3 (shoulder), h > 1e-3 (O2 away from joint 6's axis).  Nearer to a boundary an ulp
    of T moves the angles by far more than 1e-9; those rows are held to the pose round trip instead."""
    return (el > 1e-4) & (wr > 1e-4) & (sh > 1e-3) & (hh > 1e-3)


def dev(a, dt=np.float64, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)


def host(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _solve_c(rob, Td, q7d, conf):
    """the C entry point on device poses and q7 -> q (N,k,7), ok (N,k) on the host"""
    dh = ref.dh_table(rob)
    conf = np.ascontiguousarray(conf, dtype=np.int32)
    N, k = Td.shape[0], len(conf)
    q = torch.empty((N, k, 7), dtype=Td.dtype, device=Td.device)
    ok = torch.empty((N, k), dtype=torch.int32, device=Td.device)
    L = rtb._lib
    L.check(L.lib().b2k_ikine_panda(L.F64 if Td.dtype == torch.float64 else L.F32, L.dptr(dh),
                                    L.dptr(np.ascontiguousarray(rob._base)), L.dptr(np.ascontiguousarray(rob._tool)),
                                    Td.data_ptr(), q7d.data_ptr(), N, k, conf.ctypes.data_as(L.ip), q.data_ptr(),
                                    ok.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return host(q), host(ok).astype(bool)


@pytest.mark.parametrize("N", [1, 31, 32, 33, 1000, 100001])
@pytest.mark.parametrize("k", range(4))
def test_parity_with_the_restatement_fp64(k, N):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(zlib.crc32(f"panda-{k}-{N}".encode()))
    qs = rng.uniform(-np.pi, np.pi, (N, 7))
    T = ref.fk(rob, qs)
    q7 = qs[:, 6]
    got, gok = _solve_c(rob, dev(T), dev(q7), range(8))
    sol = rob.ikine_panda(dev(T), dev(q7), config=ALL)
    np.testing.assert_array_equal(host(sol.q), got)
    assert sol.success == gok.all()
    for code in range(8):
        want, ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q7, code)
        el, wr, sh, hh = ref.margins(dh, rob._base, rob._tool, T, q7, code)
        # away from the reach boundaries the two agree on reach
        clear = (np.abs(el) > 1e-6) & (np.abs(wr) > 1e-6)
        assert (gok[clear, code] == ok[clear]).all()
        assert np.isnan(got[~gok[:, code], code]).all() and np.isfinite(got[gok[:, code], code]).all()
        assert (got[gok[:, code], code, 6] == q7[gok[:, code]]).all()
        m = ok & well_conditioned(el, wr, sh, hh)
        assert m.sum() >= 0.9 * ok.sum() - 3
        assert np.abs(ref.wrap(got[m, code] - want[m])).max(initial=0) <= 1e-9


@pytest.mark.parametrize("N", [33, 100001])
@pytest.mark.parametrize("k", range(4))
def test_round_trip_fp32(k, N):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(zlib.crc32(f"panda-{k}-{N}-f32".encode()))
    qs = rng.uniform(-np.pi, np.pi, (N, 7)).astype(np.float32).astype(np.float64)
    T = ref.fk(rob, qs).astype(np.float32).astype(np.float64)
    sol = rob.ikine_panda(dev(T, np.float32), dev(qs[:, 6], np.float32), config=ALL)
    assert sol.q.dtype == torch.float32
    got = host(sol.q).astype(np.float64)
    for code in range(8):
        el, wr, sh, hh = ref.margins(dh, rob._base, rob._tool, T, qs[:, 6], code)
        m = (el > 1e-3) & (wr > 1e-3) & (hh > 1e-2)
        assert m.sum() >= 0.3 * N
        assert np.isfinite(got[m, code]).all()
        assert np.abs(ref.fk(rob, got[m, code]) - T[m]).max() <= 1e-4
    # dtype= on fp64 input selects the fp32 kernel too
    assert rob.ikine_panda(T[:3], qs[:3, 6], dtype=np.float32).q.dtype == np.float32


def test_all_eight_in_one_launch_equal_eight_launches():
    rob = ROBOTS[1]
    rng = np.random.default_rng(3)
    for dt in (np.float64, np.float32):
        qs = rng.uniform(-np.pi, np.pi, (5000, 7))
        Td, q7 = dev(ref.fk(rob, qs), dt), dev(qs[:, 6], dt)
        together = host(rob.ikine_panda(Td, q7, config=ALL).q)
        for code, letters in enumerate(ALL):
            one = host(rob.ikine_panda(Td, q7, config=letters).q)
            assert np.array_equal(one.view(np.uint8), np.ascontiguousarray(together[:, code]).view(np.uint8)), letters
        mixed = host(rob.ikine_panda(Td, q7, config=["rdf", "lun", "rdf"]).q)
        assert np.array_equal(mixed[:, 0], together[:, 7], equal_nan=True)
        assert np.array_equal(mixed[:, 1], together[:, 0], equal_nan=True)
        assert np.array_equal(mixed[:, 2], together[:, 7], equal_nan=True)


@pytest.mark.parametrize("k", [0, 2])
def test_million_row_identities_on_the_device(k):
    rob = ROBOTS[k]
    dh = ref.dh_table(rob)
    N = 1_000_000
    rng = np.random.default_rng(90 + k)
    qstar = rng.uniform(-np.pi, np.pi, (N, 7))
    qd = dev(qstar)
    ets = rob.ets()
    Td = ets.eval(qd)
    T = host(Td)
    sol = rob.ikine_panda(Td, qd[:, 6].contiguous(), config=ALL)
    assert sol.q.device == Td.device
    codes = ref.config_code(dh, qstar)
    for code in range(8):
        qc = sol.q[:, code]
        okc = ~torch.isnan(qc[:, 0])
        assert okc[torch.from_numpy(codes == code).to(Td.device)].all()  # every pose is reachable in its own configuration
        qok = qc[okc].contiguous()
        assert (ets.eval(qok) - Td[okc]).abs().max().item() <= 1e-12
        keep = well_conditioned(*ref.margins(dh, rob._base, rob._tool, T, qstar[:, 6], code)) & host(okc)
        assert keep.sum() >= 0.3 * N
        assert (ref.config_code(dh, host(qc)[keep]) == code).all()
        sel = keep & (codes == code)
        assert np.abs(ref.wrap(host(qc)[sel] - qstar[sel])).max() <= 1e-9


def test_per_row_q7_equals_scalar_q7():
    rob = ROBOTS[0]
    rng = np.random.default_rng(21)
    T = ref.fk(rob, rng.uniform(-np.pi, np.pi, (3000, 7)))
    Td = dev(T)
    rows = host(rob.ikine_panda(Td, dev(np.full(3000, 0.7)), config=ALL).q)
    for q7 in (0.7, np.float64(0.7), torch.tensor(0.7, dtype=torch.float64), np.array(0.7)):
        assert np.array_equal(host(rob.ikine_panda(Td, q7, config=ALL).q), rows, equal_nan=True)
    # a row's q7 only affects that row
    q7 = rng.uniform(-np.pi, np.pi, 3000)
    mixed = host(rob.ikine_panda(Td, q7, config=ALL).q)
    for j in (0, 1234, 2999):
        one = host(rob.ikine_panda(Td[j:j + 1], q7[j], config=ALL).q)
        assert np.array_equal(one[0], mixed[j], equal_nan=True)
    # non-finite q7 gives NaN rows with ok = 0
    bad = q7.copy()
    bad[[5, 6]] = (np.nan, np.inf)
    q, ok = _solve_c(rob, Td, dev(bad), range(8))
    assert not ok[[5, 6]].any() and np.isnan(q[[5, 6]]).all()
    with pytest.raises(ValueError, match=r"q7 must be a scalar or have shape \(3000,\)"):
        rob.ikine_panda(Td, np.zeros(2999))


def test_singular_shoulder_and_degenerate_wrist_rows_round_trip():
    for rob in ROBOTS:
        dh = ref.dh_table(rob)
        rng = np.random.default_rng(11)
        q = rng.uniform(-np.pi, np.pi, (4000, 7))
        q[:1000, 1] = rng.choice([0.0, np.pi], 1000) - dh[1, 3]  # sin(theta2) = 0
        q[1000:2000, 4] = rng.choice([h, -h], 1000) - dh[4, 3]  # theta5 = +-pi/2: on the wrist boundary
        d3, a4, a5, d5 = dh[2, 0], dh[3, 1], dh[4, 1], dh[4, 0]
        H, g = np.hypot(a4, d3), np.arctan2(d3, a4)
        # O2 on joint 5's axis (theta5 free): H cos(theta4 - gamma) = -a5
        q[2000:3000, 3] = g + rng.choice([-1, 1], 1000) * np.arccos(-a5 / H) - dh[3, 3]
        # theta4 = phi or phi + pi: on the elbow boundary
        q[3000:, 3] = np.arctan2(a4 * d5 - d3 * a5, -a4 * a5 - d3 * d5) + rng.choice([0.0, np.pi], 1000) - dh[3, 3]
        T = ref.fk(rob, q)
        Td = dev(T)
        got = host(rob.ikine_panda(Td, dev(q[:, 6]), config=ALL).q)
        for code in range(8):
            fin = np.isfinite(got[:, code, 0])
            assert np.abs(ref.fk(rob, got[fin, code]) - T[fin]).max() <= 1e-12
        solved = np.isfinite(got[:, :, 0]).any(1)
        assert solved.mean() >= 0.99
    # PandaMDH's qz has a singular shoulder: every configuration round-trips, and the elbow-down ones keep theta2 at 0
    p = rtb.models.PandaMDH()
    Tz = p.fkine(p.qz).A
    for dt in (np.float64, np.float32):
        sol = p.ikine_panda(Tz, 0.0, config=ALL, dtype=dt)
        assert sol.success
        np.testing.assert_allclose(p.fkine(sol.q.astype(np.float64)).A, np.broadcast_to(Tz, (8, 4, 4)),
                                   atol=1e-12 if dt == np.float64 else 1e-5)


def test_o2_on_joint_6_axis_round_trips():
    """h = 0: theta6 is free, the solver takes psi = 0 and reads the wrist equation as p = 0"""
    rng = np.random.default_rng(15)
    dh0 = ref.dh_table(rtb.models.PandaMDH())
    dh0[4, 0] = 0.2  # |d5| < hypot(a4, d3), so that p = 0 can be reached
    rob = rtb.DHRobot([rtb.RevoluteMDH(d=x[0], a=x[1], alpha=x[2], offset=x[3]) for x in dh0], base=ref.random_se3(rng),
                      tool=ref.random_se3(rng, 0.1))
    d3, a4, d5 = dh0[2, 0], dh0[3, 1], dh0[4, 0]
    H, g = np.hypot(a4, d3), np.arctan2(d3, a4)
    q = rng.uniform(-np.pi, np.pi, (2000, 7))
    s = np.arcsin(d5 / H)
    q[:, 3] = g + np.where(rng.random(2000) < 0.5, s, np.pi - s)
    q[:, 4] = rng.choice([h, -h], 2000)
    T = ref.fk(rob, q)
    assert ref.margins(dh0, rob._base, rob._tool, T, q[:, 6], 0)[3].max() <= 1e-14
    got = host(rob.ikine_panda(dev(T), dev(q[:, 6]), config=ALL).q)
    fin = np.isfinite(got[:, :, 0])
    assert fin.any(1).all()
    for code in range(8):
        assert np.abs(ref.fk(rob, got[fin[:, code], code]) - T[fin[:, code]]).max() <= 1e-12


def _mixed_batch(rob, rng, N=4000):
    """FK poses with rows moved beyond reach (|C / rho| > 1)"""
    q = rng.uniform(-np.pi, np.pi, (N, 7))
    T = ref.fk(rob, q)
    kind = rng.integers(0, 2, N)
    T[kind == 1, :3, 3] = (2.5, 0.5, 0.5) * rng.uniform(0.9, 1.1, ((kind == 1).sum(), 1))
    return T, q[:, 6], kind


def test_out_of_reach_rows_get_nan_and_ok_zero():
    rob = rtb.models.PandaMDH()
    dh = ref.dh_table(rob)
    T, q7, kind = _mixed_batch(rob, np.random.default_rng(4))
    N = len(T)
    Td = dev(T)
    q, ok = _solve_c(rob, Td, dev(q7), range(8))
    bad = kind != 0
    assert not ok[bad].any() and np.isnan(q[bad]).all()
    for code in range(8):
        want_ok = ref.ikine_panda(dh, rob._base, rob._tool, T, q7, code)[1]
        el, wr, _, _ = ref.margins(dh, rob._base, rob._tool, T, q7, code)
        clear = (np.abs(el) > 1e-9) & (np.abs(wr) > 1e-9)
        assert (ok[clear, code] == want_ok[clear]).all()
        assert np.isnan(q[~ok[:, code], code]).all() and np.isfinite(q[ok[:, code], code]).all()
    sol = rob.ikine_panda(Td, q7, config=ALL)
    assert not sol.success and sol.reason == f"Out of reach: {8 * N - ok.sum()} of {8 * N} solutions"
    single = rob.ikine_panda(T, q7)  # numpy, one configuration
    assert not single.success and single.reason == f"Out of reach: {N - ok[:, 0].sum()} of {N} rows"
    one = rob.ikine_panda(T[kind == 1][0], 0.0)
    assert not one.success and one.reason == "Out of reach" and one.q.shape == (7,) and np.isnan(one.q).all()


def test_placement_and_input_forms():
    rob = rtb.models.PandaMDH()
    rng = np.random.default_rng(5)
    q0 = rng.uniform(-np.pi, np.pi, (50, 7))
    T = ref.fk(rob, q0)
    letters = ref.config_of(ref.dh_table(rob), q0[7])[0]
    ref_q = host(rob.ikine_panda(dev(T), dev(q0[:, 6]), config=letters).q)
    got = rob.ikine_panda(T, q0[:, 6], config=letters)
    assert isinstance(got.q, np.ndarray) and got.q.shape == (50, 7)
    np.testing.assert_array_equal(got.q, ref_q)
    np.testing.assert_array_equal(rob.ikine_panda(rtb.SE3(T), list(q0[:, 6]), config=letters).q, ref_q)
    for one in (rob.ikine_panda(rtb.SE3(T[7]), q0[7, 6], config=letters), rob.ikine_panda(T[7], q0[7, 6], config=letters)):
        assert one.success and one.reason == "Success" and one.q.shape == (7,)
        np.testing.assert_array_equal(one.q, ref_q[7])
    np.testing.assert_allclose(ref.wrap(ref_q[7] - q0[7]), 0, atol=1e-9)
    assert rob.ikine_panda(T[7], q0[7, 6], config=["lun", "rdn"]).q.shape == (2, 7)
    Td = dev(T)
    t = rob.ikine_panda(Td, dev(q0[:, 6]), config=letters).q
    assert isinstance(t, torch.Tensor) and t.device == Td.device and t.shape == (50, 7)


@pytest.mark.parametrize("dt", [torch.float64, torch.float32])
def test_unaligned_poses_take_the_element_load_path(dt):
    """T one element past a 16-byte boundary cannot use the 16-byte loads; the element loads give the same q"""
    rob = ROBOTS[2]
    rng = np.random.default_rng(6)
    N = 1000
    qs = rng.uniform(-np.pi, np.pi, (N, 7))
    Td = dev(ref.fk(rob, qs)).to(dt)
    q7 = dev(qs[:, 6]).to(dt)
    buf = torch.empty(N * 16 + 1, dtype=dt, device=Td.device)
    Tu = buf[1:].view(N, 4, 4)
    Tu.copy_(Td)
    assert Tu.data_ptr() % 16 != 0 and Td.data_ptr() % 16 == 0
    a = host(rob.ikine_panda(Td, q7, config=ALL).q)
    b = host(rob.ikine_panda(Tu, q7, config=ALL).q)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_one_launch_per_call():
    rob = ROBOTS[3]
    rng = np.random.default_rng(7)
    qs = rng.uniform(-np.pi, np.pi, (300, 7))
    T = ref.fk(rob, qs)
    Td = dev(T)
    for args in ((Td, dev(qs[:, 6]), ALL), (Td, 0.3, "lun"), (T, qs[:, 6], ["ruf", "ldn"]), (T[0], 0.1, "lun")):
        torch.cuda.synchronize()
        n0 = rtb.launch_count()
        rob.ikine_panda(*args)
        torch.cuda.synchronize()
        assert rtb.launch_count() - n0 == 1, args


def test_ik_lm_solutions_are_among_the_closed_form_solutions():
    """an independent solver on the device: every solved PandaMDH.ik_LM row is one of the eight closed-form solutions at
    its own q7.  ik_LM stops at a pose error of its tolerance, so the poses solved in closed form are ik_LM's own,
    FK(q_LM), rather than the targets it was given."""
    rob = rtb.models.PandaMDH()
    dh = ref.dh_table(rob)
    rng = np.random.default_rng(8)
    N = 2000
    ql = rob.qlim
    Tq = dev(ref.fk(rob, rng.uniform(ql[0], ql[1], (N, 7))))
    qlm, ok = rob.ik_LM(Tq)[:2]
    qlm, ok = host(qlm).astype(np.float64), host(ok).astype(bool)
    assert ok.mean() >= 0.9
    qlm = qlm[ok]
    T = ref.fk(rob, qlm)
    sols = host(rob.ikine_panda(dev(T), dev(qlm[:, 6]), config=ALL).q)
    d = np.abs(ref.wrap(sols - qlm[:, None, :]))
    d = np.where(np.isnan(d), np.inf, d).max(-1).min(-1)
    assert d.max() <= 1e-6
    # and the closest one is the solution in ik_LM's own configuration
    codes = ref.config_code(dh, qlm)
    own = np.abs(ref.wrap(sols[np.arange(len(qlm)), codes] - qlm)).max(-1)
    assert np.mean(own <= 1e-6) >= 0.99
