"""The long-double dynamics reference of tests/dyn_ref.py, without a GPU: pinned to the compiled-reference fixtures and
the oracle, checked against the identities of rigid-body dynamics, and shown to catch plausible kernel defects with the
same fp64 bars the GPU tests apply.  Also the C ABI's output-alignment contract of b2k_rne and the fan-outs."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import b2kin as rtb
import dyn_ref as D
from oracle import chains as ch
from oracle import oracle as orc

G = os.path.join(os.path.dirname(__file__), "golden")
LD = D.LD


def f64(x):
    return np.asarray(x).astype(np.float64)


def standard_set():
    """(name, L, mdh): the two model arms and random arms with prismatic joints (one first), both conventions."""
    out = [("puma560", ch.pack_rne(ch.puma560_links()), 0), ("panda_mdh", ch.pack_rne(ch.panda_mdh_links()), 1)]
    for mdh in (0, 1):
        for prof in D.PROFILES:
            out.append((f"rand{'_mdh' if mdh else ''}_{prof}", D.robot(6, mdh, prof, True, True, 40 + mdh), mdh))
    return out


def test_reference_reproduces_the_compiled_rne_fixtures():
    z = np.load(os.path.join(G, "puma_rne.npz"))
    a = (z["q"], z["qd"], z["qdd"])
    for want, g, fx in ((z["tau"], z["gravity"], None), (z["tau_fext"], z["gravity"], z["fext"]),
                        (z["tau_zerog"], np.zeros(3), None), (z["tau_g2"], z["g2"], z["fext"])):
        np.testing.assert_allclose(f64(D.rne3(z["L"], 0, -g, *a, fext=fx)[0]), want, rtol=1e-12, atol=1e-12)
    z = np.load(os.path.join(G, "panda_mdh_rne.npz"))
    for want, fx in ((z["tau"], None), (z["tau_fext"], z["fext"])):
        np.testing.assert_allclose(f64(D.rne3(z["L"], 1, -z["gravity"], z["q"], z["qd"], z["qdd"], fext=fx)[0]), want,
                                   rtol=1e-12, atol=1e-12)
    z = np.load(os.path.join(G, "random_rne.npz"))
    for c in range(int(z["ncases"])):  # includes prismatic joints and an MDH prismatic first joint
        k = lambda s: z[f"c{c}_{s}"]  # noqa: E731
        got = f64(D.rne3(k("L"), int(k("mdh")), -k("gravity"), k("q"), k("qd"), k("qdd"), fext=k("fext"))[0])
        np.testing.assert_allclose(got, k("tau"), rtol=1e-12, atol=1e-11 * max(1.0, np.abs(k("tau")).max()))


def test_reference_reproduces_the_compiled_dynamics_fixtures():
    z = np.load(os.path.join(G, "puma_dynamics.npz"))
    L, g = z["L"], -z["gravity"]
    tol = dict(rtol=1e-11, atol=1e-11)
    np.testing.assert_allclose(f64(D.op3("inertia", L, 0, g, z["q"])[0]), z["inertia"], **tol)
    np.testing.assert_allclose(f64(D.op3("gravload", L, 0, g, z["q"])[0]), z["gravload"], **tol)
    np.testing.assert_allclose(f64(D.op3("itorque", L, 0, g, z["q"], x=z["qdd"])[0]), z["itorque"], **tol)
    np.testing.assert_allclose(f64(D.op3("coriolis", L, 0, g, z["q"], qd=z["qd"])[0]), z["coriolis"], **tol)
    np.testing.assert_allclose(f64(D.op3("accel", L, 0, g, z["q"], qd=z["qd"], x=z["torque"])[0]), z["accel"], rtol=1e-10, atol=1e-10)


def test_reference_reproduces_the_puma_kats():
    kat = json.load(open(os.path.join(G, "reference_kats.json")))
    L, qn = ch.pack_rne(ch.puma560_links()), np.atleast_2d(ch.PUMA_QN)
    k = kat["puma560_rne"]
    for c in k["cases"]:
        g = np.array(c.get("gravity", [0, 0, -9.81]), dtype=float)
        tau = D.rne3(L, 0, -g, qn, np.full((1, 6), float(c["qd"])), np.full((1, 6), float(c["qdd"])), fext=c.get("fext"))[0]
        np.testing.assert_array_almost_equal(f64(tau[0]), np.array(c["tau"], dtype=float), decimal=k["decimal"])
    k, g = kat["puma560_dynamics"], np.array([0, 0, 9.81])
    dec = k["decimal"]
    np.testing.assert_array_almost_equal(f64(D.op3("inertia", L, 0, g, qn)[0][0]), np.array(k["inertia"]), decimal=dec)
    np.testing.assert_array_almost_equal(f64(D.op3("gravload", L, 0, g, qn)[0][0]), np.array(k["gravload"], dtype=float), decimal=dec)
    np.testing.assert_array_almost_equal(f64(D.op3("itorque", L, 0, g, qn, x=[k["itorque"]["qdd"]])[0][0]), k["itorque"]["taui"], decimal=dec)
    np.testing.assert_array_almost_equal(f64(D.op3("coriolis", L, 0, g, qn, qd=[k["coriolis"]["qd"]])[0][0]), np.array(k["coriolis"]["C"], dtype=float), decimal=dec)
    np.testing.assert_array_almost_equal(f64(D.op3("accel", L, 0, g, qn, qd=[k["accel"]["qd"]], x=[k["accel"]["torque"]])[0][0]), k["accel"]["qdd"], decimal=dec)


@pytest.mark.parametrize("name,L,mdh", standard_set(), ids=[s[0] for s in standard_set()])
def test_reference_agrees_with_the_oracle_and_its_bars_cover_the_oracle(name, L, mdh):
    """The oracle is the same recursion as the kernels, in fp64: it must sit inside the fp64 bars, and agree to about
    1e-12 relative."""
    n = len(L) // 24
    q, qd, qdd, tq = D.inputs(L, 48, np.float64, 3)
    g = np.array([0.4, -1.5, 9.81])
    fx = np.array([1.0, -2.0, 0.5, 0.3, 0.2, -0.1])
    f = lambda a, b, c, gg: orc.rne(n, mdh, L, gg, a, b, c)  # noqa: E731
    fnf = lambda a, b, c, gg: orc.rne(n, mdh, orc.nofriction_L(L), gg, a, b, c)  # noqa: E731
    cases = (("rne", orc.rne(n, mdh, L, g, q, qd, qdd, fx), dict(qd=qd, x=qdd, fext=fx)),
             ("inertia", orc.dyn_inertia(f, n, q), {}), ("gravload", orc.dyn_gravload(f, n, q, g), {}),
             ("itorque", orc.dyn_itorque(f, n, q, qdd), dict(x=qdd)), ("coriolis", orc.dyn_coriolis(fnf, n, q, qd), dict(qd=qd)),
             ("accel", orc.dyn_accel(f, n, q, qd, tq, g), dict(qd=qd, x=tq)))
    for op, want, kw in cases:
        v, bar = D.op3(op, L, mdh, g, q, **kw)
        err = np.abs(f64(v) - want)
        assert np.all(err <= bar), (op, float(np.max(err - bar)))
        scale = np.abs(want).max(axis=tuple(range(1, want.ndim)), keepdims=True)
        small = np.abs(q).max(1) < 4  # rows at |q| up to 1e6 differ by the fp64 rounding of the angle, inside the bar
        assert np.all((err <= 1e-12 * np.maximum(scale, 1) * (1e3 if op == "accel" else 1))[small]), (op, float(err[small].max()))


@pytest.mark.parametrize("name,L,mdh", standard_set()[:4], ids=[s[0] for s in standard_set()[:4]])
def test_dynamics_identities_in_long_double(name, L, mdh):
    """M symmetric positive definite; itorque = M qdd; rne = M qdd + C qd + g + friction (no fext)."""
    n = len(L) // 24
    q, qd, qdd, _ = D.inputs(L, 24, np.float64, 5)
    g = np.array([0.0, 0.0, 9.81])
    M = D.op3("inertia", L, mdh, g, q)[0]
    scale = np.abs(M).max()
    assert np.abs(M - M.transpose(0, 2, 1)).max() < 1e-16 * scale
    A = M.copy()  # LDL^T pivots of an SPD matrix are positive
    for c in range(n):
        assert np.all(A[:, c, c] > 0)
        A[:, c + 1:, c + 1:] -= A[:, c + 1:, c, None] * A[:, c, None, c + 1:] / A[:, c, c, None, None]
    Mq = np.einsum("nik,ni->nk", M, qdd.astype(LD))  # row i of M: torques of a unit acceleration of joint i
    taui = D.op3("itorque", L, mdh, g, q, x=qdd)[0]
    assert np.abs(taui - Mq).max() < 1e-15 * max(1.0, float(np.abs(taui).max()))
    Cm = D.op3("coriolis", L, mdh, g, q, qd=qd)[0]
    grav = D.op3("gravload", L, mdh, g, q)[0]
    Lr = np.asarray(L).reshape(-1, 24)
    Gr, qdl = Lr[:, 20].astype(LD), qd.astype(LD)
    fric = (Gr * Gr * Lr[:, 21] * qdl + np.where(qdl > 0, np.abs(Gr) * Lr[:, 22], 0) + np.where(qdl < 0, np.abs(Gr) * Lr[:, 23], 0))
    tau = D.rne3(L, mdh, g, q, qd, qdd)[0]
    rhs = Mq + np.einsum("nkj,nj->nk", Cm, qdl) + grav + fric
    assert np.abs(tau - rhs).max() < 1e-14 * max(1.0, float(np.abs(tau).max()))


def _near_quarter_turn_robot():
    L = D.robot(6, 0, "struct", False, True, 77).reshape(-1, 24).copy()
    L[:, 0] = np.pi / 2 + 1e-7 * np.array([1, -1, 1, -1, 1, -1])
    return L.ravel()


DEFECT_OPS = {"coulomb_at_zero": ("rne",), "signed_G": ("rne",), "jm_G": ("rne", "inertia"), "mdh_ps_sign": ("rne",),
              "coriolis_friction": ("coriolis",), "accel_nofriction": ("accel",), "loose_snap": ("rne",)}


@pytest.mark.parametrize("defect", D.DEFECTS)
def test_every_plausible_defect_crosses_the_fp64_bar(defect):
    """A kernel with the defect would fail the GPU tests: on the standard set, at least one entry moves by more than
    the fp64 bar of the correct reference."""
    robots = [(L, mdh) for _, L, mdh in standard_set()] + [(_near_quarter_turn_robot(), 0)]
    worst = 0.0
    for L, mdh in robots:
        if defect == "mdh_ps_sign" and not mdh:
            continue
        q, qd, qdd, tq = D.inputs(L, 32, np.float64, 9)
        g = np.array([0.0, 0.0, 9.81])
        for op in DEFECT_OPS[defect]:
            kw = dict(qd=qd, x={"rne": qdd, "accel": tq}.get(op))
            good, bar = D.op3(op, L, mdh, g, q, **kw)
            bad, _ = D.op3(op, L, mdh, g, q, defect=defect, **kw)
            worst = max(worst, float(np.max(np.abs(f64(bad) - f64(good)) / np.maximum(bar, 1e-300))))
    assert worst > 1.0, (defect, worst)


# ------------------------------------------------------------------ output alignment of the C ABI
def _puma_handle():
    h = rtb._lib.vp()
    L = ch.pack_rne(ch.puma560_links())
    assert rtb._lib.lib().b2k_rne_create(6, 0, L.ctypes.data_as(rtb._lib.dp), C.byref(h)) == 0
    return h


def test_outputs_off_their_stage_unit_are_rejected_before_any_cuda_call():
    """A 6-joint fp64 row is 48 bytes: tau, gravload, itorque and accel outputs are copied in 16-byte pieces, the 6x6
    inertia and Coriolis matrices (288 bytes) too.  An output at 8 mod 16 is element-aligned, and must be refused up
    front with a message naming it (the alternative is a launch-time failure after the device guard)."""
    lib = rtb._lib.lib()
    h = _puma_handle()
    buf = np.zeros(512)
    p = buf.ctypes.data + (-buf.ctypes.data) % 64
    g = np.array([0.0, 0.0, 9.81])
    gp = rtb._lib.dptr(g)
    n0 = lib.b2k_launch_count()
    assert lib.b2k_rne(h, 1, p, p, p, 4, gp, None, p + 8, None) == -1
    assert b"tau must be 16-byte aligned" in lib.b2k_last_error(), lib.b2k_last_error()
    for fn, args in (("b2k_rne_inertia", (p, 4)), ("b2k_rne_gravload", (p, 4, gp)), ("b2k_rne_itorque", (p, p, 4)),
                     ("b2k_rne_coriolis", (p, p, 4)), ("b2k_rne_accel", (p, p, p, 4, gp))):
        assert getattr(lib, fn)(h, 1, *args, p + 8, None) == -1, fn
        assert b"output must be 16-byte aligned" in lib.b2k_last_error(), (fn, lib.b2k_last_error())
    # fp32: a 6-joint row is 24 bytes, copied in 8-byte pieces
    assert lib.b2k_rne(h, 0, p, p, p, 4, gp, None, p + 4, None) == -1
    assert b"tau must be 8-byte aligned" in lib.b2k_last_error()
    assert lib.b2k_launch_count() == n0
    lib.b2k_rne_destroy(h)
