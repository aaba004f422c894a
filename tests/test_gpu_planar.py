"""Planar kinematics on the GPU (b2k_fkine_planar through ETS2 / Robot2) against the float64 restatement in
planar_ref.py: random chains of every joint count with all three joint kinds, flips, constants between joints, permuted
jindices, q wider than the chain, base and tool; tile edges; fp64 and fp32 (on fp32-rounded inputs); fused against
separate calls; every q form."""
import os
import sys

import numpy as np
import pytest

import b2kin as rtb

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import planar_ref as ref  # noqa: E402

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROWS = (1, 31, 32, 33, 1000, 100001)
TOL = {np.float64: dict(rtol=1e-10, atol=1e-12), np.float32: dict(rtol=1e-4, atol=1e-5)}


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", range(1, 11))
def test_random_chains_against_the_restatement(n, dt):
    rng = np.random.default_rng(1000 + n)
    wide = int(rng.integers(0, 4))
    ets = ref.random_chain(rng, n, wide=wide)
    base, tool = ref.random_pose(rng), ref.random_pose(rng)
    Q = rng.uniform(-3.5, 3.5, (max(ROWS), n + wide)).astype(dt)
    Q64 = Q.astype(np.float64)  # the reference sees the rounded inputs
    T_ref = ref.eval_(ets, Q64, base, tool)
    J_ref = ref.jacob0(ets, Q64, tool)
    Je_ref = ref.jacobe(ets, Q64, tool)
    tdt = torch.float64 if dt == np.float64 else torch.float32
    # fp32 positions are sums over the whole chain: the absolute bar is 1e-5 per unit of the chain's reach
    reach = max(1.0, float(np.abs(T_ref[:, :2, 2]).max()))
    tol = dict(TOL[dt], atol=TOL[dt]["atol"] * (reach if dt == np.float32 else 1.0))
    Qd = torch.from_numpy(Q).cuda()
    for N in ROWS:
        q = Qd[:N]  # one row is one configuration: results come back without the batch axis
        T, J = (x.reshape(N, 3, -1) for x in ets.fkine_jacob0(q, base=base, tool=tool))
        assert T.dtype == tdt and T.shape == (N, 3, 3) and J.shape == (N, 3, n)
        np.testing.assert_allclose(T.cpu().numpy(), T_ref[:N], **tol, err_msg=f"T n={n} N={N}")
        np.testing.assert_allclose(J.cpu().numpy(), J_ref[:N], **tol, err_msg=f"J0 n={n} N={N}")
        Je = ets.jacobe(q, tool=tool).reshape(N, 3, n)
        np.testing.assert_allclose(Je.cpu().numpy(), Je_ref[:N], **tol, err_msg=f"Je n={n} N={N}")
        # the fused call equals the separate ones bit for bit
        assert torch.equal(T, ets.eval(q, base=base, tool=tool).reshape(N, 3, 3))
        assert torch.equal(J, ets.jacob0(q, tool=tool).reshape(N, 3, n))
        # jacobe = blkdiag(R^T, 1) jacob0 on the kernel's own outputs
        R = ets.eval(q, tool=tool).reshape(N, 3, 3)[:, :2, :2]
        np.testing.assert_allclose(Je[:, :2].cpu().numpy(), (R.transpose(1, 2) @ J[:, :2]).cpu().numpy(), **tol)
        assert torch.equal(Je[:, 2], J[:, 2])


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_base_is_on_the_pose_only_and_include_base(dt):
    rng = np.random.default_rng(7)
    ets = ref.random_chain(rng, 4, wide=1)
    base = ref.random_pose(rng)
    q = torch.from_numpy(rng.uniform(-2, 2, (100, 5)).astype(dt)).cuda()
    T = ets.eval(q, base=base)
    np.testing.assert_allclose(T.cpu().numpy(), ref.eval_(ets, q.double().cpu().numpy(), base), **TOL[dt])
    assert torch.equal(ets.eval(q, base=base, include_base=False), ets.eval(q))
    T2, J2 = ets.fkine_jacob0(q, base=base)
    assert torch.equal(T2, T) and torch.equal(J2, ets.jacob0(q))


def test_planar2_hand_derived_values():
    r = rtb.models.ETS.Planar2()
    np.testing.assert_allclose(r.eval(r.qz), [[1, 0, 2], [0, 1, 0], [0, 0, 1]], atol=1e-15)
    np.testing.assert_allclose(r.jacob0(r.qz), [[0, 0], [2, 1], [1, 1]], atol=1e-15)
    np.testing.assert_allclose(r.jacobe(r.qz), [[0, 0], [2, 1], [1, 1]], atol=1e-15)
    # q = (pi/2, -pi/2): the first link points along y, the second along x
    q = [np.pi / 2, -np.pi / 2]
    np.testing.assert_allclose(r.eval(q), [[1, 0, 1], [0, 1, 1], [0, 0, 1]], atol=1e-15)
    np.testing.assert_allclose(r.jacob0(q), [[-1, 0], [1, 1], [1, 1]], atol=1e-15)
    s = r.fkine(np.array([r.qz, q]))
    assert isinstance(s, rtb.SE2) and len(s) == 2
    np.testing.assert_allclose(s.t, [[2, 0], [1, 1]], atol=1e-15)
    # the robot's base and tool enter like explicit ones
    r.base = ref.random_pose(np.random.default_rng(1))
    r.tool = ref.random_pose(np.random.default_rng(2))
    qq = np.random.default_rng(3).uniform(-3, 3, (50, 2))
    np.testing.assert_allclose(r.eval(qq), ref.eval_(r.ets(), qq, r.base.A, r.tool.A), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(r.jacob0(qq), ref.jacob0(r.ets(), qq, r.tool.A), rtol=1e-10, atol=1e-12)
    T, J = r.fkine_jacob0(qq)
    np.testing.assert_array_equal(T, r.eval(qq))
    np.testing.assert_array_equal(J, r.jacob0(qq))


def test_every_q_form():
    r = rtb.models.ETS.Planar2()
    e = r.ets()
    q = [0.3, -1.1]
    want = ref.eval_(e, np.array([q]))[0]
    for form in (q, np.array(q), np.array([q]), np.array(q).reshape(2, 1), np.array(q, dtype=np.float32)):
        T = e.eval(form)
        assert isinstance(T, np.ndarray) and T.shape == (3, 3), type(form)
        np.testing.assert_allclose(T, want, rtol=1e-4 if getattr(form, "dtype", None) == np.float32 else 1e-12, atol=1e-6)
    for tdt in (torch.float64, torch.float32):
        for form in (torch.tensor(q, dtype=tdt).cuda(), torch.tensor([q], dtype=tdt).cuda()):
            T = e.eval(form)
            assert torch.is_tensor(T) and T.is_cuda and T.dtype == tdt and T.shape == (3, 3)
            np.testing.assert_allclose(T.cpu().numpy(), want, rtol=1e-4, atol=1e-6)
        J = e.jacob0(torch.tensor([q, q], dtype=tdt).cuda())
        assert J.shape == (2, 3, 2) and J.dtype == tdt
    Jh = e.jacob0(np.array([q, q, q]))
    assert isinstance(Jh, np.ndarray) and Jh.shape == (3, 3, 2)
    # a 1-joint chain: (N, 1) is a batch
    one = rtb.ETS2([rtb.ET2.R(), rtb.ET2.tx(1.0)])
    Tb = one.eval(np.array([[0.0], [np.pi / 2], [np.pi]]))
    assert Tb.shape == (3, 3, 3)
    np.testing.assert_allclose(Tb[:, :2, 2], [[1, 0], [0, 1], [-1, 0]], atol=1e-15)
    # an explicit dtype converts the input
    assert e.eval(np.array([q]), dtype=np.float32).dtype == np.float32


def test_non_planar_chain_adds_no_launch():
    e3 = rtb.ETS([rtb.ET.Rz(), rtb.ET.tx(1.0), rtb.ET.Ry()])
    q = torch.zeros((64, 2), dtype=torch.float64, device="cuda")
    T = torch.empty((64, 3, 3), dtype=torch.float64, device="cuda")
    L = rtb._lib.lib()
    n0 = rtb.launch_count()
    rc = L.b2k_fkine_planar(e3._chain, 1, q.data_ptr(), 64, 2, None, None, 0, T.data_ptr(), None,
                            torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"joint 1 is Ry" in L.b2k_last_error()
    assert rtb.launch_count() == n0
    e = rtb.models.ETS.Planar2().ets()
    n0 = rtb.launch_count()
    e.fkine_jacob0(q)
    assert rtb.launch_count() == n0 + 1  # pose and Jacobian from one launch
