"""Derivatives of tree-robot dynamics without a device: the complex-step reference against the Featherstone oracle and
Richardson differences, identities that need no step size, the generated RNE_DERIV / ACCEL_DERIV row functions compiled
for the host (g++) against the reference, the library's NVRTC build of both kernels at every joint count, and the C ABI's
argument checks."""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

import b2kin as rtb
import tree_derivs_ref as ref
from oracle import chains as ch
from oracle import oracle as orc
from test_codegen_cpu import random_tree, tree_handle

DERIV_HARNESS = r"""
#include <cmath>
#define __device__
#define __forceinline__ inline
typedef double real;
using std::fma;
%s
extern "C" void eval(const double *Cst, const double *grav, int n, const double *q, const double *qd, const double *qdd, long N,
                     double *out)
{
    double fext[6] = {0};
    for (long i = 0; i < N; i++) {
        double st[16], ct[16];
        for (int j = 0; j < n; j++) { st[j] = std::sin(q[i * n + j]); ct[j] = std::cos(q[i * n + j]); }
        rne_deriv_row(Cst, grav, fext, st, ct, q + i * n, qd + i * n, qdd + i * n, out + i * 2 * n * n, out + i * 2 * n * n + n * n);
    }
}
"""


def deriv_host_fn(tmp_path, tag, h, grav_mask, op=7):
    """The generated derivative row of operation op (7 RNE_DERIV, 8 ACCEL_DERIV: the same row, which the kernel evaluates
    at qdd*) compiled for the host: run(a_grav, q, qd, qdd) -> (dtau_dq, dtau_dqd), each (N, n, n)."""
    lib = rtb._lib.lib()
    src = C.create_string_buffer(1 << 24)
    consts = np.zeros(16384)
    nc = C.c_int32()
    counts = (C.c_int32 * 3)()
    rtb._lib.check(lib.b2k_tree_codegen(h, op, grav_mask, src, len(src), rtb._lib.dptr(consts), 16384, C.byref(nc), counts))
    text = src.value.decode()
    assert text.count("rne_deriv_row(") == 1 and text.count("void rne_row(") == (op == 8)
    cpp, so = tmp_path / f"{tag}.cpp", tmp_path / f"{tag}.so"
    cpp.write_text(DERIV_HARNESS % text)
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", str(cpp), "-o", str(so)])
    L = C.CDLL(str(so))
    dp = C.POINTER(C.c_double)
    L.eval.argtypes = [dp, dp, C.c_int, dp, dp, dp, C.c_long, dp]
    cst = consts[:nc.value].copy()

    def run(agrav, q, qd, qdd):
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in (cst, agrav, q, qd, qdd)]
        N, n = a[2].shape
        out = np.zeros((N, 2, n, n))
        L.eval(a[0].ctypes.data_as(dp), a[1].ctypes.data_as(dp), n, a[2].ctypes.data_as(dp), a[3].ctypes.data_as(dp),
               a[4].ctypes.data_as(dp), N, out.ctypes.data_as(dp))
        return out[:, 0], out[:, 1]

    return run


def spong():
    return dict(parent=[-1, 0], axis=[1, 1], flip=[0, 0], jindex=[0, 1], C=[np.eye(4), ch.transl(1, 0, 0)],
                I6=[orc.spatial_inertia(1, [0.5, 0, 0])] * 2)


def regular_tree(rng, n, branched=True):
    """A tree whose inertia matrix is regular: off-axis point masses on every group, revolute joints."""
    tree = random_tree(rng, n, branched)
    tree["I6"] = [orc.spatial_inertia(rng.uniform(0.5, 2), rng.uniform(0.1, 0.3, 3) * rng.choice([-1, 1], 3))
                  + orc.spatial_inertia(rng.uniform(0.5, 2), rng.uniform(0.1, 0.3, 3) * rng.choice([-1, 1], 3)) for _ in range(n)]
    tree["axis"] = [int(a) for a in rng.integers(0, 3, n)]
    return tree


def test_reference_restates_the_oracle_and_agrees_with_richardson_differences():
    rng = np.random.default_rng(1)
    for n, branched in ((1, False), (4, False), (7, True)):
        tree = random_tree(rng, n, branched)
        tree["flip"][0] = 1
        grav = np.array([0.3, -0.7, -9.81])
        for _ in range(3):
            q, qd, qdd = rng.uniform(-3, 3, n), rng.normal(size=n), rng.normal(size=n)
            want = orc.tree_rne(tree, q, qd, qdd, grav)[0]
            np.testing.assert_allclose(ref.rne(tree, q, qd, qdd, grav), want, rtol=0, atol=1e-14 * max(1, np.abs(want).max()))
            dq, dqd = ref.rne_derivatives(tree, q, qd, qdd, grav)
            for k in range(n):
                rq = ref.richardson(lambda x: ref.rne(tree, x, qd, qdd, grav), q, k)
                rqd = ref.richardson(lambda x: ref.rne(tree, q, x, qdd, grav), qd, k)
                scale = max(1.0, np.abs(dq).max(), np.abs(dqd).max())
                np.testing.assert_allclose(dq[:, k], rq, rtol=0, atol=1e-7 * scale)
                np.testing.assert_allclose(dqd[:, k], rqd, rtol=0, atol=1e-7 * scale)


def _check_identities(tree, dq_fn, q, qd, grav):
    """dtau_dqd qd = 2 rne(q, qd, 0, g = 0); at qd = qdd = 0 the gravity Jacobian, rows in q order and flipped rows negated,
    is the (symmetric) Hessian of the potential energy."""
    n = len(q)
    z = np.zeros(n)
    _, dqd = dq_fn(q, qd, z, grav)
    want = 2 * ref.rne(tree, q, qd, z, np.zeros(3))
    np.testing.assert_allclose(dqd @ qd, want, rtol=0, atol=1e-11 * max(1, np.abs(want).max()))
    dq, _ = dq_fn(q, z, z, grav)
    K = np.zeros((n, n))
    for j in range(n):
        K[tree["jindex"][j]] = -dq[j] if tree["flip"][j] else dq[j]
    np.testing.assert_allclose(K, K.T, rtol=0, atol=1e-11 * max(1, np.abs(K).max()))


def test_identities_of_the_reference_and_the_generated_row(tmp_path):
    rng = np.random.default_rng(2)
    for k, (n, branched, permute) in enumerate(((3, False, False), (6, True, True), (9, True, False))):
        tree = random_tree(rng, n, branched)
        tree["flip"] = [int(f) for f in rng.integers(0, 2, n)]
        if permute:
            tree["jindex"] = [int(i) for i in rng.permutation(n)]
        grav = np.array([0.4, -0.2, -9.81])
        h = tree_handle(tree)
        f = deriv_host_fn(tmp_path, f"id{k}", h, 7)
        gen = lambda q, qd, qdd, g: tuple(x[0] for x in f(-g, q[None], qd[None], qdd[None]))  # noqa: E731
        cs = lambda q, qd, qdd, g: ref.rne_derivatives(tree, q, qd, qdd, g)  # noqa: E731
        for _ in range(3):
            q, qd = rng.uniform(-3, 3, n), rng.normal(size=n)
            _check_identities(tree, cs, q, qd, grav)
            _check_identities(tree, gen, q, qd, grav)
        rtb._lib.lib().b2k_tree_destroy(h)
    # the forward mode: M dqdd_dtau = I and dqdd_dq = -dqdd_dtau dtau_dq at qdd*
    tree = regular_tree(rng, 5)
    q, qd, tq = rng.uniform(-3, 3, 5), rng.normal(size=5), rng.normal(size=5)
    grav = np.array([0, 0, -9.81])
    aq, aqd, at = ref.accel_derivatives(tree, q, qd, tq, grav)
    np.testing.assert_allclose(ref.inertia(tree, q) @ at, np.eye(5), rtol=0, atol=1e-12)
    dq, dqd = ref.rne_derivatives(tree, q, qd, ref.accel(tree, q, qd, tq, grav), grav)
    np.testing.assert_allclose(aq, -at @ dq, rtol=0, atol=1e-12 * np.abs(aq).max())
    np.testing.assert_allclose(aqd, -at @ dqd, rtol=0, atol=1e-12 * np.abs(aqd).max())
    # and against Richardson differences of accel itself
    for k in range(5):
        r = ref.richardson(lambda x: ref.accel(tree, x, qd, tq, grav), q, k)
        np.testing.assert_allclose(aq[:, k], r, rtol=0, atol=1e-6 * max(1, np.abs(aq).max()))


@pytest.mark.parametrize("op", [7, 8])
def test_generated_derivative_rows_equal_the_complex_step_reference(tmp_path, op):
    """random trees n = 1, 3, 6 (branched), 9, 16 with flipped and prismatic joints, gravity masks 7 / 4 / 0, a permuted
    jindex; the ACCEL_DERIV row at a given qdd (the kernel evaluates it at qdd*)."""
    rng = np.random.default_rng(70 + op)
    cases = [(1, False, False), (3, False, False), (6, True, False), (9, True, True), (16, True, False)]
    for k, (n, branched, permute) in enumerate(cases):
        tree = random_tree(rng, n, branched)
        tree["flip"][n // 2] = 1
        tree["axis"][-1] = 3 + int(rng.integers(0, 3))  # at least one prismatic joint
        if permute:
            tree["jindex"] = [int(i) for i in rng.permutation(n)]
        h = tree_handle(tree)
        for gm, grav in ((7, np.array([0.5, -1.0, -9.81])), (4, np.array([0, 0, -9.81])), (0, np.zeros(3))):
            f = deriv_host_fn(tmp_path, f"r{op}_{k}_{gm}", h, gm, op=op)
            N = 4
            q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
            gq, gqd = f(-grav, q, qd, qdd)
            for i in range(N):
                wq, wqd = ref.rne_derivatives(tree, q[i], qd[i], qdd[i], grav)
                scale = max(1.0, np.abs(wq).max(), np.abs(wqd).max())
                np.testing.assert_allclose(gq[i], wq, rtol=0, atol=1e-10 * scale, err_msg=f"n={n} gm={gm} dq")
                np.testing.assert_allclose(gqd[i], wqd, rtol=0, atol=1e-10 * scale, err_msg=f"n={n} gm={gm} dqd")
        rtb._lib.lib().b2k_tree_destroy(h)


def test_spong_two_link_closed_form(tmp_path):
    """tau_1 = d11 qdd1 + d12 qdd2 + h qd2^2 + 2 h qd1 qd2 + g1, tau_2 = d12 qdd1 + d22 qdd2 - h qd1^2 + g2 with
    d11 = 1.5 + cos q2, d12 = 0.25 + 0.5 cos q2, d22 = 0.25, h = -0.5 sin q2, g1 = -G (1.5 cos q1 + 0.5 cos(q1 + q2)),
    g2 = -0.5 G cos(q1 + q2) (the Spong arm of the reference's tests, gravity -G z)."""
    G = 9.81
    h = tree_handle(spong())
    f = deriv_host_fn(tmp_path, "spong", h, 4)
    rng = np.random.default_rng(3)
    for _ in range(5):
        q, qd, qdd = rng.uniform(-3, 3, 2), rng.normal(size=2), rng.normal(size=2)
        s2, c2, s12 = np.sin(q[1]), np.cos(q[1]), np.sin(q[0] + q[1])
        hh, dh = -0.5 * s2, -0.5 * c2
        dq = np.array([[G * (1.5 * np.sin(q[0]) + 0.5 * s12),
                        -s2 * qdd[0] - 0.5 * s2 * qdd[1] + dh * qd[1] ** 2 + 2 * dh * qd[0] * qd[1] + 0.5 * G * s12],
                       [0.5 * G * s12, -0.5 * s2 * qdd[0] - dh * qd[0] ** 2 + 0.5 * G * s12]])
        dqd = np.array([[2 * hh * qd[1], 2 * hh * qd[1] + 2 * hh * qd[0]], [-2 * hh * qd[0], 0.0]])
        gq, gqd = f(np.array([0, 0, G]), q[None], qd[None], qdd[None])
        np.testing.assert_allclose(gq[0], dq, rtol=0, atol=1e-12)
        np.testing.assert_allclose(gqd[0], dqd, rtol=0, atol=1e-12)
    rtb._lib.lib().b2k_tree_destroy(h)


NVRTC = any(os.path.exists(p) for p in ("/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"))


@pytest.mark.skipif(not NVRTC, reason="NVRTC not installed")
@pytest.mark.parametrize("n", range(1, 17))
def test_derivative_kernels_build_through_the_library_at_every_joint_count(n):
    """Both derivative kernels, fp32 and fp64, build for sm_90a at every n <= 16 (B2K_TREE_MAX): the output stage fits the
    shared memory of an SM (the warps per block follow n)."""
    lib = rtb._lib.lib()
    tree = random_tree(np.random.default_rng(500 + n), n, True)
    h = tree_handle(tree)
    for op in (7, 8):
        for dt in (rtb._lib.F64, rtb._lib.F32):
            buf = C.create_string_buffer(4096)
            t0 = time.perf_counter()
            rtb._lib.check(lib.b2k_tree_info(h, op, dt, rtb._lib.dptr(np.array([0.5, -1.0, 3.0])), buf, 4096))
            info = buf.value.decode()
            assert info.startswith(f"k_rne_deriv_spec<{'double' if dt == rtb._lib.F64 else 'float'},tree n={n},mode={op}>"), info[:600]
            if os.environ.get("B2K_PRINT_BUILD_TIMES"):
                print(f"n={n} op={op} dtype={dt}: {time.perf_counter() - t0:.2f} s: {info}")
    lib.b2k_tree_destroy(h)


def test_tree_derivatives_rejects_bad_arguments_before_any_cuda_call():
    lib = rtb._lib.lib()
    h = tree_handle(spong())
    buf = (C.c_double * 64)()
    p = C.cast(buf, C.c_void_p)
    mis = C.c_void_p(p.value + 8)
    g = rtb._lib.dptr(np.array([0.0, 0.0, 9.81]))
    D = lib.b2k_tree_derivatives

    def err(*a):
        assert D(*a) == -1, a
        assert lib.b2k_last_error().decode().startswith("b2k_tree_derivatives: ")

    err(None, 7, 1, p, p, p, 1, g, p, p, None, None)                         # handle
    for op in (0, 5, 6, 9, -1):                                               # op
        err(h, op, 1, p, p, p, 1, g, p, p, p, None)
    err(h, 7, 2, p, p, p, 1, g, p, p, None, None)                            # dtype
    err(h, 7, 1, p, p, p, -1, g, p, p, None, None)                           # N < 0
    for k in range(5):                                                        # NULL arrays with N > 0
        a = [p, p, p, p, p]
        a[k] = None
        err(h, 7, 1, a[0], a[1], a[2], 1, g, a[3], a[4], None, None)
    err(h, 8, 1, p, p, p, 1, g, p, p, None, None)                            # op 8 needs out2
    err(h, 7, 1, p, p, p, 1, g, p, p, p, None)                               # op 7 forbids out2
    err(h, 7, 1, p, p, p, 0, g, p, p, p, None)                               # ... at N = 0 too
    for k in range(6):                                                        # 16-byte alignment
        a = [p] * 6
        a[k] = mis
        err(h, 8, 1, a[0], a[1], a[2], 1, g, a[3], a[4], a[5], None)
    err(h, 7, 1, p, p, p, 1, None, p, p, None, None)                         # grav
    assert D(h, 7, 1, None, None, None, 0, g, None, None, None, None) == 0   # an empty batch is a no-op
    # b2k_tree_dyn keeps rejecting the derivative codes
    for op in (7, 8):
        assert lib.b2k_tree_dyn(h, op, 1, p, p, p, 1, g, p, None) == -1
    lib.b2k_tree_destroy(h)
