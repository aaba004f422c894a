"""The regressor reference of tests/regressor_ref.py, without a GPU: Y_ref @ pi reproduces the oracle's rne, pi follows
the parallel-axis convention, the structural zeros hold; and the C ABI of the regressor is exported and refuses bad
arguments before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

import b2kin as rtb
import regressor_ref as RR
import rne_derivs_ref as R
from oracle import chains as ch
from oracle import oracle as orc

GRAV = np.array([1.5, -2.0, 9.81])  # the vector handed to the kernel: minus the robot's gravity


def robots():
    out = [("puma560", ch.pack_rne(ch.puma560_links()), 0), ("panda_mdh", ch.pack_rne(ch.panda_mdh_links()), 1)]
    for n in range(1, 11):
        for mdh in (0, 1):
            for pris in (False, True):
                out.append((f"n{n}_{'mdh' if mdh else 'dh'}_{'pris' if pris else 'rev'}",
                            R.robot(n, mdh, pris, True, 700 + 10 * n + 2 * mdh + pris), mdh))
    return out


ROBOTS = robots()


def rel(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1.0))


@pytest.mark.parametrize("name,L,mdh", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_reference_regressor_times_parameters_is_rne(name, L, mdh):
    """Y_ref @ pi == rne to 1e-12 at both signs of qd and exact zeros, with the default and a custom gravity; pi from
    DHRobot.dynamic_parameters of the same links."""
    q, qd, qdd = RR.states(L, 12, 3)
    pi = R.dhrobot(L, mdh).dynamic_parameters()
    np.testing.assert_array_equal(pi, RR.parameters(L))
    for g in (np.array([0.0, 0.0, 9.81]), GRAV):
        Y = RR.regressor(L, mdh, g, q, qd, qdd)
        tau = orc.rne(len(L) // 24, mdh, L, g, q, qd, qdd)
        assert rel(Y @ pi, tau) < 1e-12, (name, rel(Y @ pi, tau))


@pytest.mark.parametrize("name,L,mdh", ROBOTS[:8], ids=[r[0] for r in ROBOTS[:8]])
def test_structural_zeros_are_exact(name, L, mdh):
    q, qd, qdd = RR.states(L, 6, 4)
    Y = RR.regressor(L, mdh, GRAV, q, qd, qdd)
    n = len(L) // 24
    assert np.all(Y[:, RR.structural_mask(n)] == 0.0)
    # and the friction columns of the own joint are the closed forms
    G = np.asarray(L).reshape(-1, 24)[:, 20]
    for j in range(n):
        np.testing.assert_allclose(Y[:, j, 14 * j + 10], G[j] ** 2 * qdd[:, j], rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(Y[:, j, 14 * j + 11], G[j] ** 2 * qd[:, j], rtol=1e-13, atol=1e-13)
        np.testing.assert_array_equal(Y[:, j, 14 * j + 12], np.where(qd[:, j] > 0, abs(G[j]), 0.0))
        np.testing.assert_array_equal(Y[:, j, 14 * j + 13], np.where(qd[:, j] < 0, abs(G[j]), 0.0))


def test_dynamic_parameters_moves_the_inertia_to_the_frame_origin():
    r = np.array([0.1, -0.2, 0.3])
    I = np.array([[0.5, 0.01, -0.02], [0.01, 0.4, 0.03], [-0.02, 0.03, 0.3]])
    link = rtb.DHLink(a=0.2, alpha=0.3, m=2.0, r=r, I=I, Jm=1e-4, G=-50.0, B=2e-3, Tc=[0.3, -0.4])
    pi = rtb.DHRobot([link]).dynamic_parameters()
    Io = I + 2.0 * (r @ r * np.eye(3) - np.outer(r, r))  # the parallel-axis theorem
    want = [2.0, 0.2, -0.4, 0.6, Io[0, 0], Io[1, 1], Io[2, 2], Io[0, 1], Io[1, 2], Io[0, 2], 1e-4, 2e-3, 0.3, -0.4]
    np.testing.assert_allclose(pi, want, rtol=1e-15, atol=1e-17)
    # the 6-vector form of I takes the same order
    link6 = rtb.DHLink(a=0.2, alpha=0.3, m=0.0, I=[1, 2, 3, 4, 5, 6])
    np.testing.assert_array_equal(rtb.DHRobot([link6]).dynamic_parameters()[4:10], [1, 2, 3, 4, 5, 6])


def test_regressor_symbols_are_exported():
    lib = rtb._lib.lib()
    for sym in ("b2k_rne_regressor", "b2k_rne_regressor_gram"):
        assert sym in rtb._lib.EXPORTED_SYMBOLS
        getattr(lib, sym)


def test_kernel_info_names_the_generic_regressor_kernel():
    puma = rtb.models.Puma560()
    s = puma.rne_kernel_info(op="rne_regressor")
    assert s.startswith("generic k_rne_regressor<double, n=6, DH, all-revolute>"), s
    assert "float" in rtb.models.PandaMDH().rne_kernel_info(op="rne_regressor", dtype=np.float32)


# ------------------------------------------------------------------ the C ABI refuses bad arguments before any CUDA call
@pytest.fixture(scope="module")
def puma():
    lib = rtb._lib.lib()
    h = rtb._lib.vp()
    L = ch.pack_rne(ch.puma560_links())
    assert lib.b2k_rne_create(6, 0, L.ctypes.data_as(rtb._lib.dp), C.byref(h)) == 0
    yield h
    lib.b2k_rne_destroy(h)


def _refused(fn, call, needle):
    lib = rtb._lib.lib()
    assert call() == -1, (fn, needle)
    msg = lib.b2k_last_error().decode()
    assert msg.startswith(fn + ":") and needle in msg, (fn, msg)


def test_bad_arguments_are_refused_before_any_cuda_call(puma):
    lib = rtb._lib.lib()
    buf = np.zeros(8192)
    p = buf.ctypes.data + (-buf.ctypes.data) % 64
    g = rtb._lib.dptr(np.array([0.0, 0.0, 9.81]))
    w_ok = np.ones(6)
    n0 = lib.b2k_launch_count()

    def reg(h=puma, dt=1, q=p, qd=p, qdd=p, N=4, grav=g, Y=p):
        return lambda: lib.b2k_rne_regressor(h, dt, q, qd, qdd, N, grav, Y, None)

    def gram(h=puma, dt=1, q=p, qd=p, qdd=p, tau=p, N=4, grav=g, w=w_ok, G=p, b=p, s=p):
        return lambda: lib.b2k_rne_regressor_gram(h, dt, q, qd, qdd, tau, N, grav, rtb._lib.dptr(w), G, b, s, None)

    for fn, mk in (("b2k_rne_regressor", reg), ("b2k_rne_regressor_gram", gram)):
        _refused(fn, mk(h=None), "rne handle is NULL")
        _refused(fn, mk(dt=2), "dtype must be B2K_F32 or B2K_F64")
        _refused(fn, mk(N=-1), "N is negative")
        _refused(fn, mk(grav=None), "grav is NULL")
        _refused(fn, mk(q=None), "q is NULL")
        _refused(fn, mk(qd=None), "qd is NULL")
        _refused(fn, mk(qdd=None), "qdd is NULL")
        _refused(fn, mk(qd=p + 4), "qd must be 8-byte aligned")
        _refused(fn, mk(dt=0, qdd=p + 2), "qdd must be 4-byte aligned")
    # Y's rows (14 n^2 reals: 4032 bytes in fp64, 2016 in fp32) are copied in 16-byte pieces
    _refused("b2k_rne_regressor", reg(Y=None), "Y is NULL")
    _refused("b2k_rne_regressor", reg(Y=p + 8), "Y must be 16-byte aligned")
    _refused("b2k_rne_regressor", reg(dt=0, Y=p + 8), "Y must be 16-byte aligned")
    fn = "b2k_rne_regressor_gram"
    _refused(fn, gram(tau=None), "tau is NULL")
    _refused(fn, gram(tau=p + 4), "tau must be 8-byte aligned")
    for bad in (-1.0, np.nan, np.inf):
        w = w_ok.copy(); w[3] = bad
        _refused(fn, gram(w=w), "weights[3]")
    for name in ("G", "b", "s"):
        _refused(fn, gram(**{name: None}), f"{name} is NULL")
        _refused(fn, gram(**{name: p + 4}), f"{name} must be 8-byte aligned")
        _refused(fn, gram(N=0, q=None, qd=None, qdd=None, tau=None, **{name: None}), f"{name} is NULL")  # written at N = 0 too
    # N = 0 touches no device for the regressor, whatever the pointers
    assert reg(q=None, qd=None, qdd=None, N=0, Y=None)() == 0
    assert lib.b2k_launch_count() == n0


def test_the_regressor_code_is_no_tree_or_specialised_operation(puma):
    """B2K_GEN_RNE_REGRESSOR (9) follows B2K_GEN_ACCEL_DERIV; the tree entry points and the DH specialiser's info and
    code generator reject it."""
    lib = rtb._lib.lib()
    buf = C.create_string_buffer(4096)
    g = np.array([0.0, 0.0, 9.81])
    assert lib.b2k_rne_codegen(puma, 9, 7, 0, buf, 4096, None, 0, None, None) == -1
    assert lib.b2k_last_error().decode().startswith("b2k_rne_codegen: ")
    rc = lib.b2k_rne_spec_info(puma, 9, 1, rtb._lib.dptr(g), 0, buf, 4096)
    assert rc == -1 or "k_rne_spec" not in buf.value.decode(), buf.value.decode()
    import os
    arm = rtb.Robot.URDF(os.path.join(os.path.dirname(__file__), "golden", "urdf", "two_arm.urdf"))
    h = arm._tree_handle()
    cbuf = (C.c_double * 64)()
    p = C.cast(cbuf, C.c_void_p)
    assert lib.b2k_tree_dyn(h, 9, 1, p, p, p, 1, rtb._lib.dptr(g), p, None) == -1
    assert "is not one of B2K_DYN_*" in lib.b2k_last_error().decode()
    assert lib.b2k_tree_derivatives(h, 9, 1, p, p, p, 1, rtb._lib.dptr(g), p, p, None, None) == -1
    assert lib.b2k_tree_info(h, 9, 1, rtb._lib.dptr(g), buf, 4096) == -1
    assert "is not one of B2K_DYN_*" in lib.b2k_last_error().decode()
    assert lib.b2k_tree_codegen(h, 9, 7, buf, 4096, None, 0, None, None) == -1
