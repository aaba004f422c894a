"""Rollouts without a device: the RK4 restatement and its chained sensitivities against differences of the whole
rollout, the double-integrator identity at rest, the generated DH derivative rows compiled for the host (g++) against
the reference, the text of the existing generator modes against the parent's, the NVRTC build of the rollout kernel at
every joint count, and every refusal of the C ABI and the Python front end."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import time

import numpy as np
import pytest

import b2kin as rtb
import rne_derivs_ref as dref
import rollout_ref as ref
import tree_derivs_ref as tref
from test_codegen_cpu import random_tree, tree_handle
from test_tree_derivs_cpu import regular_tree

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "codegen_sha256.json")
NVRTC = any(os.path.exists(p) for p in ("/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"))


def dh_model(n, mdh, friction, seed):
    L = dref.robot(n, mdh, False, friction, seed)
    return L, ref.dh(L, mdh, np.array([0.3, -0.2, 9.81]))


def fd(f, x, h=1e-5):
    """Jacobian (N, m, k) of f: (N, k) -> (N, m) by central differences."""
    cols = []
    for j in range(x.shape[1]):
        e = np.zeros(x.shape[1])
        e[j] = h
        cols.append((f(x + e) - f(x - e)) / (2 * h))
    return np.stack(cols, axis=-1)


@pytest.mark.parametrize("family", ["dh", "tree"])
def test_reference_sensitivities_against_differences_of_the_rollout(family):
    rng = np.random.default_rng(1)
    if family == "dh":
        L, model = dh_model(3, 0, False, 5)
        n = 3
    else:
        desc = regular_tree(rng, 4)
        model, n = ref.tree(desc, np.array([0.0, 0.0, -9.81])), 4
    N, K, h = 2, 3, 0.02
    q0, qd0, tau = rng.uniform(-1, 1, (N, n)), rng.uniform(-1, 1, (N, n)), rng.normal(size=(N, K, n))
    q, qd, A, B = ref.rollout(model, q0, qd0, tau, h)
    x = np.concatenate([q, qd], axis=2)
    for k in range(K):
        wA = fd(lambda y: ref.step(model[0], y, tau[:, k], h), x[:, k])
        wB = fd(lambda u: ref.step(model[0], x[:, k], u, h), tau[:, k])
        np.testing.assert_allclose(A[:, k], wA, rtol=0, atol=1e-6 * max(1, np.abs(wA).max()))
        np.testing.assert_allclose(B[:, k], wB, rtol=0, atol=1e-6 * max(1, np.abs(wB).max()))
        if family == "tree":  # the complex step of the whole map: no composition formula, no step size
            cA, cB = ref.complex_step(model[0], x[:, k], tau[:, k], h)
            np.testing.assert_allclose(A[:, k], cA, rtol=0, atol=1e-12 * max(1, np.abs(cA).max()))
            np.testing.assert_allclose(B[:, k], cB, rtol=0, atol=1e-12 * max(1, np.abs(cB).max()))

    def xK(x0):
        qq, qqd, _, _ = ref.rollout(model, x0[:, :n], x0[:, n:], tau, h, sensitivities=False)
        return np.concatenate([qq[:, -1], qqd[:, -1]], axis=1)

    P = A[:, 0]
    for k in range(1, K):
        P = A[:, k] @ P
    want = fd(xK, x[:, 0])
    np.testing.assert_allclose(P, want, rtol=0, atol=1e-6 * max(1, np.abs(want).max()))


@pytest.mark.parametrize("family", ["dh", "tree"])
def test_double_integrator_identity_at_rest(family):
    """Friction-free, at rest, no gravity, no torque: nothing moves, A = [[I, dt I], [0, I]], B = [[dt^2/2 M^-1], [dt M^-1]]."""
    rng = np.random.default_rng(2)
    if family == "dh":
        L = dref.robot(5, 1, False, False, 7)
        model, Mi = ref.dh(L, 1, np.zeros(3)), np.linalg.inv(dref.inertia(L, 1, np.zeros((1, 5)) + 0.4))
        n = 5
    else:
        desc = regular_tree(rng, 5)
        model, n = ref.tree(desc, np.zeros(3)), 5
        Mi = np.linalg.inv(tref.inertia(desc, np.zeros(5) + 0.4))[None]
    for h in (1e-3, 0.05, 0.7):
        q0 = np.zeros((1, n)) + 0.4
        q, qd, A, B = ref.rollout(model, q0, np.zeros((1, n)), np.zeros((1, 2, n)), h)
        np.testing.assert_array_equal(q[0], np.broadcast_to(q0, (3, n)))
        np.testing.assert_array_equal(qd, 0)
        I, Z = np.eye(n), np.zeros((n, n))
        np.testing.assert_allclose(A[0, 1], np.block([[I, h * I], [Z, I]]), rtol=0, atol=1e-9 * max(1, h))
        np.testing.assert_allclose(B[0, 1], np.vstack([h * h / 2 * Mi[0], h * Mi[0]]), rtol=0, atol=1e-9 * np.abs(Mi).max())


HARNESS = r"""
#include <cmath>
#define __device__
#define __forceinline__ inline
typedef double real;
using std::fma;
static inline real step_pos(real x) { return x > 0 ? 1 : 0; }
static inline real step_neg(real x) { return x < 0 ? 1 : 0; }
%s
extern "C" void eval(const double *Cst, const double *grav, int n, const double *th, const double *qd, const double *qdd, long N,
                     double *out)
{
    double fext[6] = {0};
    for (long i = 0; i < N; i++) {
        double st[16], ct[16];
        for (int j = 0; j < n; j++) { st[j] = std::sin(th[i * n + j]); ct[j] = std::cos(th[i * n + j]); }
        rne_deriv_row(Cst, grav, fext, st, ct, th + i * n, qd + i * n, qdd + i * n, out + i * 2 * n * n, out + i * 2 * n * n + n * n);
    }
}
"""


def codegen_dh(h, mode, gm, fext=0):
    lib = rtb._lib.lib()
    src = C.create_string_buffer(1 << 24)
    consts = np.zeros(16384)
    nc = C.c_int32()
    rtb._lib.check(lib.b2k_rne_codegen(h, mode, gm, fext, src, len(src), rtb._lib.dptr(consts), 16384, C.byref(nc), None))
    return src.value.decode(), consts[:nc.value].copy()


@pytest.mark.parametrize("mdh", [0, 1])
def test_generated_dh_derivative_rows_equal_the_reference(tmp_path, mdh):
    """n = 1..10 with friction (the Coulomb term has a zero tangent: compared against the table without it), qd of both
    signs and exact zeros, gravity masks 7 / 4 / 0; the ACCEL_DERIV program is the ACCEL row followed by the same row."""
    dp = C.POINTER(C.c_double)
    for n in range(1, 11):
        L = dref.robot(n, mdh, False, True, 300 + n)
        rob = dref.dhrobot(L, mdh)
        h = rob._rne_handle()
        nocoul = L.reshape(-1, 24).copy()
        nocoul[:, 22:24] = 0
        rng = np.random.default_rng(n)
        for gm, grav in ((7, np.array([0.5, -1.0, 9.81])), (4, np.array([0, 0, 9.81])), (0, np.zeros(3))):
            for op in (7, 8):
                text, cst = codegen_dh(h, op, gm)
                if op == 8:
                    accel_text = codegen_dh(h, 5, gm)[0]
                    assert text.startswith(accel_text) and text.count("rne_deriv_row(") == 1
                cpp, so = tmp_path / f"d{mdh}_{n}_{gm}_{op}.cpp", tmp_path / f"d{mdh}_{n}_{gm}_{op}.so"
                cpp.write_text(HARNESS % text)
                subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", str(cpp), "-o", str(so)])
                lib = C.CDLL(str(so))
                lib.eval.argtypes = [dp, dp, C.c_int, dp, dp, dp, C.c_long, dp]
                N = 3
                q, qd, qdd, _ = dref.states(L, N, n + gm)
                qd[1, ::2] = 0.0  # exact zeros: the Coulomb step of the generated row must not show
                th = q + L.reshape(-1, 24)[:, 5]
                out = np.zeros((N, 2, n, n))
                a = [np.ascontiguousarray(x, dtype=np.float64) for x in (cst, grav, th, qd, qdd)]
                lib.eval(*(x.ctypes.data_as(dp) for x in a[:2]), n, *(x.ctypes.data_as(dp) for x in a[2:]), N, out.ctypes.data_as(dp))
                wq, wqd = dref.rne_derivatives(nocoul.ravel(), mdh, grav, q, qd, qdd)
                scale = max(1.0, np.abs(wq).max(), np.abs(wqd).max())
                np.testing.assert_allclose(out[:, 0], wq, rtol=0, atol=1e-8 * scale, err_msg=f"n={n} gm={gm} op={op}")
                np.testing.assert_allclose(out[:, 1], wqd, rtol=0, atol=1e-8 * scale, err_msg=f"n={n} gm={gm} op={op}")
        del rng


def codegen_digests():
    """sha256 over the generated text (or the refusal) of every existing mode, per robot: DH modes 0-6 and 9 (gravity
    masks 0 / 4 / 7, tip wrench off / on), tree modes 0-10 (masks 0 / 4 / 7)."""
    lib = rtb._lib.lib()
    buf = C.create_string_buffer(1 << 25)
    out = {}
    dh = [(name, getattr(rtb.models, name)()) for name in ("Puma560", "PandaMDH", "UR10")]
    dh += [(f"rand{n}_{mdh}", dref.dhrobot(dref.robot(n, mdh, False, True, 900 + n), mdh)) for n in range(1, 11) for mdh in (0, 1)]
    for name, r in dh:
        d = hashlib.sha256()
        for mode in (0, 1, 2, 3, 4, 5, 6, 9):
            for gm in (0, 4, 7):
                for fx in (0, 1):
                    rc = lib.b2k_rne_codegen(r._rne_handle(), mode, gm, fx, buf, len(buf), None, 0, None, None)
                    d.update(str(rc).encode() + (buf.value if rc == 0 else lib.b2k_last_error()))
        out[f"dh/{name}"] = d.hexdigest()
    for n in range(1, 17):
        h = tree_handle(random_tree(np.random.default_rng(700 + n), n, n > 2))
        d = hashlib.sha256()
        for mode in range(11):
            for gm in (0, 4, 7):
                rc = lib.b2k_tree_codegen(h, mode, gm, buf, len(buf), None, 0, None, None)
                d.update(str(rc).encode() + (buf.value if rc == 0 else lib.b2k_last_error()))
        lib.b2k_tree_destroy(h)
        out[f"tree/{n}"] = d.hexdigest()
    return out


def test_existing_generator_modes_are_byte_identical():
    """The digests in tests/golden/codegen_sha256.json were taken from the generator before it served the DH derivative
    modes."""
    with open(GOLDEN) as f:
        want = json.load(f)
    assert codegen_digests() == want


@pytest.mark.skipif(not NVRTC, reason="NVRTC not installed")
@pytest.mark.parametrize("n", range(1, 17))
def test_rollout_kernels_build_at_every_joint_count(n):
    lib = rtb._lib.lib()
    tree = random_tree(np.random.default_rng(600 + n), n, True)
    h = tree_handle(tree)
    robots = [("tree", h)]
    if n <= 10:
        robots.append(("dh", dref.dhrobot(dref.robot(n, n % 2, False, True, 600 + n), n % 2)))
    for kind, r in robots:
        for dt in (rtb._lib.F64, rtb._lib.F32):
            for mode in (305, 308):
                buf = C.create_string_buffer(4096)
                t0 = time.perf_counter()
                if kind == "tree":
                    rtb._lib.check(lib.b2k_tree_info(h, mode, dt, rtb._lib.dptr(np.array([0.5, -1.0, 3.0])), buf, 4096))
                    want = f"k_rollout<{'double' if dt == rtb._lib.F64 else 'float'},tree n={n},mode={mode}>"
                else:
                    rtb._lib.check(lib.b2k_rne_spec_info(r._rne_handle(), mode, dt, rtb._lib.dptr(np.array([0.5, -1.0, 3.0])), 0,
                                                         buf, 4096))
                    want = f"k_rollout<{'double' if dt == rtb._lib.F64 else 'float'},n={n},mode={mode}>"
                info = buf.value.decode()
                assert info.startswith(want), info[:600]
                if os.environ.get("B2K_PRINT_BUILD_TIMES"):
                    print(f"{kind} n={n} mode={mode} dtype={dt}: {time.perf_counter() - t0:.2f} s")
    lib.b2k_tree_destroy(h)


def test_c_abi_refusals_launch_nothing():
    lib = rtb._lib.lib()
    puma = rtb.models.Puma560()
    dh_h = puma._rne_handle()
    tr = tree_handle(random_tree(np.random.default_rng(1), 3, False))
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    mis = C.c_void_p(p.value + 4)
    g = rtb._lib.dptr(np.array([0.0, 0.0, 9.81]))
    n0 = rtb.launch_count()
    for fn, h, n, name in ((lib.b2k_rne_rollout, dh_h, 6, "b2k_rne_rollout"), (lib.b2k_tree_rollout, tr, 3, "b2k_tree_rollout")):
        ok = dict(h=h, dt_=1, q0=p, qd0=p, N=1, K=2, dt=0.01, g=g, tau=p, stride=0, q=p, qd=p, A=p, B=p)

        def err(**kw):
            a = dict(ok, **kw)
            assert fn(a["h"], a["dt_"], a["q0"], a["qd0"], a["N"], a["K"], a["dt"], a["g"], a["tau"], a["stride"], a["q"], a["qd"],
                      a["A"], a["B"], None) == -1, kw
            assert lib.b2k_last_error().decode().startswith(name + ": "), lib.b2k_last_error()

        err(h=None)
        err(dt_=2)
        err(N=-1)
        err(K=0)
        for bad in (0.0, -0.01, float("inf"), float("nan")):
            err(dt=bad)
        err(g=None)
        err(stride=2 * n + 1)
        err(A=None)
        err(B=None)
        for k in ("q0", "tau", "q", "qd"):
            err(**{k: None})
        for k in ("q0", "qd0", "tau", "q", "qd", "A", "B"):
            err(**{k: mis})
        err(dt_=0, q0=C.c_void_p(p.value + 2))  # fp32 needs 4-byte alignment
        # N = 0: no launch, no CUDA call; NULL arrays are fine
        assert fn(h, 1, None, None, 0, 2, 0.01, g, None, 0, None, None, None, None, None) == 0
    # a prismatic DH arm is refused
    L = dref.robot(3, 0, True, False, 3)
    pr = dref.dhrobot(L, 0)
    assert lib.b2k_rne_rollout(pr._rne_handle(), 1, p, p, 1, 2, 0.01, g, p, 0, p, p, None, None, None) == -1
    assert "prismatic" in lib.b2k_last_error().decode()
    assert rtb.launch_count() == n0
    lib.b2k_tree_destroy(tr)


def test_python_refusals():
    L = dref.robot(3, 0, True, False, 3)
    pr = dref.dhrobot(L, 0)
    with pytest.raises(ValueError, match="all-revolute"):
        pr.rollout(np.zeros(3), np.zeros((2, 3)), 0.01)
    puma = rtb.models.Puma560()
    for bad in (0.0, -1.0, float("nan"), float("inf"), np.array([0.1, 0.2])):
        with pytest.raises(ValueError, match="dt"):
            puma.rollout(np.zeros(6), np.zeros((2, 6)), bad)


RNE_HARNESS = r"""
#include <cmath>
#define __device__
#define __forceinline__ inline
typedef double real;
using std::fma;
static inline real step_pos(real x) { return x > 0 ? 1 : 0; }
static inline real step_neg(real x) { return x < 0 ? 1 : 0; }
%s
extern "C" void eval(const double *Cst, const double *grav, const double *th, const double *qd, const double *qdd, double *out)
{
    double fext[6] = {0}, st[1] = {std::sin(th[0])}, ct[1] = {std::cos(th[0])};
    rne_row(Cst, grav, fext, st, ct, th, qd, qdd, out);
}
"""


def test_generator_serves_a_joint_whose_only_torque_is_coulomb_friction(tmp_path):
    """One MDH link with no mass, inertia, armature or viscous friction: its torque before the Coulomb term is a structural
    zero.  Every mode generates; rne is the Coulomb torque and its derivatives are 0."""
    L = np.zeros(24)
    L[20], L[22:24] = 1.0, (0.3, -0.2)
    rob = dref.dhrobot(L, 1)
    h = rob._rne_handle()
    for mode in (0, 1, 2, 3, 4, 5, 6, 7, 8):
        codegen_dh(h, mode, 0)
    dp = C.POINTER(C.c_double)
    text, cst = codegen_dh(h, 0, 0)
    cpp, so = tmp_path / "c0.cpp", tmp_path / "c0.so"
    cpp.write_text(RNE_HARNESS % text)
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", str(cpp), "-o", str(so)])
    lib = C.CDLL(str(so))
    text7, cst7 = codegen_dh(h, 7, 0)
    cpp7, so7 = tmp_path / "c7.cpp", tmp_path / "c7.so"
    cpp7.write_text(HARNESS % text7)
    subprocess.check_call(["g++", "-O1", "-shared", "-fPIC", str(cpp7), "-o", str(so7)])
    lib7 = C.CDLL(str(so7))
    lib7.eval.argtypes = [dp, dp, C.c_int, dp, dp, dp, C.c_long, dp]
    for qd, want in ((0.5, 0.3), (-0.5, -0.2), (0.0, 0.0)):
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in (cst, np.zeros(3), [0.7], [qd], [1.3], np.zeros(1))]
        lib.eval(*(x.ctypes.data_as(dp) for x in a))
        assert a[-1][0] == want
        d = np.ones((1, 2, 1, 1))
        b = [np.ascontiguousarray(x, dtype=np.float64) for x in (cst7, np.zeros(3), [0.7], [qd], [1.3])]
        lib7.eval(*(x.ctypes.data_as(dp) for x in b[:2]), 1, *(x.ctypes.data_as(dp) for x in b[2:]), 1, d.ctypes.data_as(dp))
        np.testing.assert_array_equal(d, 0.0)


def test_dh_derivative_operations_stay_on_the_generic_kernel():
    """The generated DH derivative rows serve rollouts only: b2k_rne_spec_info reports the generic kernel for modes 7, 8."""
    lib = rtb._lib.lib()
    h = rtb.models.Puma560()._rne_handle()
    buf = C.create_string_buffer(1024)
    for mode in (7, 8):
        rtb._lib.check(lib.b2k_rne_spec_info(h, mode, rtb._lib.F64, rtb._lib.dptr(np.array([0, 0, 9.81])), 0, buf, 1024))
        assert buf.value.decode() == "generic (the derivatives of DH arms are served by the generic kernel)"
