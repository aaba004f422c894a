"""The float64 derivative reference of tests/rne_derivs_ref.py, without a GPU: pinned to identities of rigid-body dynamics
that need no step size, and the argument checks of b2k_rne_derivatives / b2k_rne_accel_derivatives, which must refuse
bad input before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

import b2kin as rtb
import rne_derivs_ref as R
from oracle import chains as ch
from oracle import oracle as orc

GRAV = np.array([1.5, -2.0, 9.81])  # the vector handed to the kernel: minus the robot's gravity


def robots():
    """(name, L, mdh): DH and MDH, all-revolute and with prismatic joints, friction on and off, a few joint counts."""
    out = [("puma560", ch.pack_rne(ch.puma560_links()), 0), ("panda_mdh", ch.pack_rne(ch.panda_mdh_links()), 1)]
    for n in (1, 3, 6, 10):
        for mdh in (0, 1):
            for pris in (False, True):
                for fr in (False, True):
                    out.append((f"n{n}_{'mdh' if mdh else 'dh'}_{'pris' if pris else 'rev'}_{'fric' if fr else 'nofric'}",
                                R.robot(n, mdh, pris, fr, 100 * n + 10 * mdh + 2 * pris + fr), mdh))
    return out


ROBOTS = robots()


mdh_prismatic_first = R.mdh_prismatic_first
# the MDH prismatic-first arms again, with that joint made revolute
ROBOTS += [(name + "_revfirst", R.revolute_first(L), mdh) for name, L, mdh in ROBOTS if mdh_prismatic_first(L, mdh)]


def rel(a, b):
    """Largest difference relative to the largest entry of b, or absolute when that is below 1."""
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1.0))


def test_accel_restatement_matches_the_oracle():
    for name, L, mdh in ROBOTS[:6]:
        n = len(L) // 24
        q, qd, _, tq = R.states(L, 5, 1)
        want = orc.dyn_accel(lambda a, b, c, g: orc.rne(n, mdh, L, g, a, b, c), n, q, qd, tq, GRAV)
        np.testing.assert_allclose(R.accel(L, mdh, GRAV, q, qd, tq), want, rtol=1e-12, atol=1e-12, err_msg=name)


def test_reference_matches_a_known_linear_case():
    """One prismatic joint along gravity: tau = (m + G^2 Jm) qdd + m g + G^2 B qd + |G| Tc, so dtau/dq = 0 and
    dtau/dqd = G^2 B exactly."""
    L = np.zeros(24)
    L[4], L[6], L[19], L[20], L[21], L[22], L[23] = 1, 2.5, 1e-4, 30.0, 1e-3, 0.2, -0.3
    q, qd, qdd = np.array([[0.3]]), np.array([[0.7]]), np.array([[-1.2]])
    dq, dqd = R.rne_derivatives(L, 0, np.array([0, 0, 9.81]), q, qd, qdd)
    assert abs(dq[0, 0, 0]) < 1e-10  # the rounding of a difference quotient, eps |tau| / H
    assert abs(dqd[0, 0, 0] - 900 * 1e-3) < 1e-10


@pytest.mark.parametrize("name,L,mdh", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_velocity_terms_are_quadratic_in_qd(name, L, mdh):
    """Without a tip wrench, tau(qd) - friction = Coriolis/centripetal part, homogeneous of degree 2 in qd, so
    dtau_dqd @ qd = 2 (rne(q, qd, 0, g=0) + friction(qd)) + G^2 B qd -- at any qdd and gravity."""
    q, qd, qdd, _ = R.states(L, 8, 2)
    _, dqd = R.rne_derivatives(L, mdh, GRAV, q, qd, qdd)
    lhs = np.einsum("rik,rk->ri", dqd, qd)
    rhs = 2 * (R.rne(L, mdh, np.zeros(3), q, qd, np.zeros_like(q)) + R.friction(L, qd)) + R.viscous(L) * qd
    assert rel(lhs, rhs) < 1e-9, (name, rel(lhs, rhs))


@pytest.mark.parametrize("name,L,mdh", ROBOTS, ids=[r[0] for r in ROBOTS])
def test_gravity_load_derivative_is_symmetric(name, L, mdh):
    """At qd = qdd = 0 without a tip wrench tau is the gradient of the potential energy: dtau_dq is its Hessian.  The
    MDH prismatic first joint, whose recursion the reference keeps as it is, is made revolute here."""
    if mdh_prismatic_first(L, mdh):
        L = R.revolute_first(L)
    q, _, _, _ = R.states(L, 8, 3)
    z = np.zeros_like(q)
    dq, _ = R.rne_derivatives(L, mdh, GRAV, q, z, z)
    assert rel(dq, np.swapaxes(dq, 1, 2)) < 1e-9, name


CONSISTENT = [r for r in ROBOTS if not mdh_prismatic_first(r[1], r[2])]


@pytest.mark.parametrize("name,L,mdh", CONSISTENT, ids=[r[0] for r in CONSISTENT])
def test_forward_and_inverse_derivatives_agree(name, L, mdh):
    """dqdd_dtau @ inertia(q) = I, and dqdd_dx = -M^-1 dtau_dx at qdd* = accel(q, qd, torque) for x = q, qd, where the
    forward derivatives are differences of accel: everywhere but on MDH arms with a prismatic first joint, whose
    reference accel is not the inverse of rne.  The differences of accel carry M's condition number kappa."""
    q, qd, _, tq = R.states(L, 6, 4)
    fq, fqd, ft = R.accel_derivatives(L, mdh, GRAV, q, qd, tq)
    M = R.inertia(L, mdh, q)
    n = q.shape[1]
    w = max(1.0, float(np.max(np.linalg.cond(M))) / 100)
    assert rel(ft @ M, np.broadcast_to(np.eye(n), M.shape)) < 1e-8 * w, name
    qdd = R.accel(L, mdh, GRAV, q, qd, tq)
    iq, iqd = R.rne_derivatives(L, mdh, GRAV, q, qd, qdd)
    Minv = np.linalg.inv(M)
    assert rel(fq, -Minv @ iq) < 1e-8 * w, (name, rel(fq, -Minv @ iq))
    assert rel(fqd, -Minv @ iqd) < 1e-8 * w, (name, rel(fqd, -Minv @ iqd))


# ------------------------------------------------------------------ the C ABI refuses bad arguments before any CUDA call
@pytest.fixture(scope="module")
def puma():
    lib = rtb._lib.lib()
    h = rtb._lib.vp()
    L = ch.pack_rne(ch.puma560_links())
    assert lib.b2k_rne_create(6, 0, L.ctypes.data_as(rtb._lib.dp), C.byref(h)) == 0
    yield h
    lib.b2k_rne_destroy(h)


def _calls(h, dt, p, N, g, ins=None, outs=None):
    """Both entry points with every pointer p unless replaced by ins / outs."""
    i0, i1, i2 = ins or (p, p, p)
    lib = rtb._lib.lib()
    o = outs or (p, p, p)
    return {"b2k_rne_derivatives": lambda: lib.b2k_rne_derivatives(h, dt, i0, i1, i2, N, g, None, o[0], o[1], None),
            "b2k_rne_accel_derivatives": lambda: lib.b2k_rne_accel_derivatives(h, dt, i0, i1, i2, N, g, o[0], o[1], o[2], None)}


def _refused(fn, call, needle):
    lib = rtb._lib.lib()
    assert call() == -1, fn
    msg = lib.b2k_last_error().decode()
    assert msg.startswith(fn + ":") and needle in msg, (fn, msg)


def test_bad_arguments_are_refused_before_any_cuda_call(puma):
    lib = rtb._lib.lib()
    buf = np.zeros(4096)
    p = buf.ctypes.data + (-buf.ctypes.data) % 64
    g = rtb._lib.dptr(np.array([0.0, 0.0, 9.81]))
    n0 = lib.b2k_launch_count()
    cases = [
        (_calls(None, 1, p, 4, g), "rne handle is NULL"),
        (_calls(puma, 2, p, 4, g), "dtype must be B2K_F32 or B2K_F64"),
        (_calls(puma, 1, p, -1, g), "N is negative"),
        (_calls(puma, 1, p, 4, None), "grav is NULL"),
        (_calls(puma, 1, p, 4, g, ins=(None, p, p)), "q is NULL"),
        (_calls(puma, 1, p, 4, g, ins=(p, None, p)), "qd is NULL"),
        (_calls(puma, 1, p, 4, g, ins=(p, p + 4, p)), "qd must be 8-byte aligned"),
        (_calls(puma, 1, p, 4, g, outs=(None, p, p)), "_dq is NULL"),
        (_calls(puma, 1, p, 4, g, outs=(p, None, p)), "_dqd is NULL"),
        # a 6 x 6 fp64 row is 288 bytes: outputs are copied in 16-byte pieces; in fp32 (144 bytes) too
        (_calls(puma, 1, p, 4, g, outs=(p + 8, p, p)), "_dq must be 16-byte aligned"),
        (_calls(puma, 0, p, 4, g, outs=(p, p + 8, p)), "_dqd must be 16-byte aligned"),
    ]
    for calls, needle in cases:
        for fn, call in calls.items():
            _refused(fn, call, needle)
    inv = _calls(puma, 1, p, 4, g, ins=(p, p, None))
    _refused("b2k_rne_derivatives", inv["b2k_rne_derivatives"], "qdd is NULL")
    _refused("b2k_rne_accel_derivatives", inv["b2k_rne_accel_derivatives"], "torque is NULL")
    fwd = _calls(puma, 1, p, 4, g, outs=(p, p, None))["b2k_rne_accel_derivatives"]
    _refused("b2k_rne_accel_derivatives", fwd, "dqdd_dtau is NULL")
    fwd = _calls(puma, 1, p, 4, g, outs=(p, p, p + 8))["b2k_rne_accel_derivatives"]
    _refused("b2k_rne_accel_derivatives", fwd, "dqdd_dtau must be 16-byte aligned")
    # N = 0 touches no device, whatever the pointers
    for call in _calls(puma, 1, None, 0, g, ins=(None, None, None), outs=(None, None, None)).values():
        assert call() == 0
    assert lib.b2k_launch_count() == n0


def test_kernel_info_names_the_generic_derivative_kernel():
    puma = rtb.models.Puma560()
    for op, mode in (("rne_derivatives", "inverse"), ("accel_derivatives", "forward")):
        s = puma.rne_kernel_info(op=op)
        assert s.startswith("generic k_rne_deriv<double, n=6, DH, all-revolute, " + mode + ">"), s
        assert "generates no derivative kernels" in s
    assert "float" in puma.rne_kernel_info(op="rne_derivatives", dtype=np.float32)
