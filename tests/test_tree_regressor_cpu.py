"""The dynamics regressor of tree robots without a device: the reference (tests/tree_regressor_ref.py) against the
Featherstone oracle, dynamic_parameters on a two-link arm with literal values, the generated B2K_DYN_REGRESSOR row
function compiled for the host (g++) against the reference on every gravity mask, its structural zeros, the NVRTC build
at every joint count, the C ABI's argument checks and the op codes each robot kind rejects."""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

import b2kin as rtb
import tree_regressor_ref as ref
from oracle import oracle as orc
from test_codegen_cpu import random_tree, tree_handle

B2K_DYN_REGRESSOR = 10

REG_HARNESS = r"""
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
    for (long r = 0; r < N; r++) {
        double st[16], ct[16];
        for (int j = 0; j < n; j++) { st[j] = std::sin(q[r * n + j]); ct[j] = std::cos(q[r * n + j]); }
        for (int i = 0; i < n; i++)
            rne_regressor_row(Cst, grav, fext, st, ct, q + r * n, qd + r * n, qdd + r * n, i, out + (r * n + i) * 10 * n);
    }
}
"""


def regressor_host_fn(tmp_path, tag, h, grav_mask):
    """The generated regressor row compiled for the host: run(a_grav, q, qd, qdd) -> Y (N, n, 10n)."""
    lib = rtb._lib.lib()
    src = C.create_string_buffer(1 << 24)
    consts = np.zeros(16384)
    nc = C.c_int32()
    counts = (C.c_int32 * 3)()
    rtb._lib.check(lib.b2k_tree_codegen(h, B2K_DYN_REGRESSOR, grav_mask, src, len(src), rtb._lib.dptr(consts), 16384,
                                        C.byref(nc), counts))
    text = src.value.decode()
    assert text.count("void rne_regressor_row(") == 1
    cpp, so = tmp_path / f"{tag}.cpp", tmp_path / f"{tag}.so"
    cpp.write_text(REG_HARNESS % text)
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", str(cpp), "-o", str(so)])
    L = C.CDLL(str(so))
    dp = C.POINTER(C.c_double)
    L.eval.argtypes = [dp, dp, C.c_int, dp, dp, dp, C.c_long, dp]
    cst = consts[:nc.value].copy()

    def run(agrav, q, qd, qdd):
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in (cst, agrav, q, qd, qdd)]
        N, n = a[2].shape
        out = np.full((N, n, 10 * n), np.nan)
        L.eval(a[0].ctypes.data_as(dp), a[1].ctypes.data_as(dp), n, a[2].ctypes.data_as(dp), a[3].ctypes.data_as(dp),
               a[4].ctypes.data_as(dp), N, out.ctypes.data_as(dp))
        return out

    return run


def sample_tree(rng, n, branched, permute=False):
    """A random tree (tests/test_codegen_cpu.py) with a flipped and a prismatic joint, full rigid-body inertias."""
    tree = random_tree(rng, n, branched)
    tree["flip"][n // 2] = 1
    tree["axis"][-1] = 3 + int(rng.integers(0, 3))
    if permute:
        tree["jindex"] = [int(i) for i in rng.permutation(n)]
    tree["I6"] = [ref.rigid_body_inertia(rng) if rng.random() < 0.7 else np.asarray(I6) for I6 in tree["I6"]]
    return tree


@pytest.mark.parametrize("n", range(1, 17))
def test_reference_times_parameters_is_the_oracle(n):
    rng = np.random.default_rng(900 + n)
    for branched in (False, True):
        tree = sample_tree(rng, n, branched, permute=branched)
        pi = ref.dynamic_parameters(tree)
        for grav in (np.array([0.0, 0.0, -9.81]), np.array([0.7, -1.2, -9.5])):
            q, qd, qdd = rng.uniform(-3, 3, n), rng.normal(size=n), rng.normal(size=n)
            want = orc.tree_rne(tree, q, qd, qdd, grav)[0]
            got = ref.regressor(tree, q, qd, qdd, grav) @ pi
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-12 * max(1.0, np.abs(want).max()))


def test_dynamic_parameters_of_a_two_link_arm():
    """Spong's arm: two unit masses half-way along unit links about y.  Per group m = 1, h = m r = (0.5, 0, 0),
    Ib = m (r.r E - r r^T) = diag(0, 0.25, 0.25)."""
    ET, Link, Robot = rtb.ET, rtb.Link, rtb.Robot
    l0 = Link(ET.Ry(), name="l0", m=1.0, r=[0.5, 0, 0])
    l1 = Link(ET.tx(1.0) * ET.Ry(), name="l1", parent=l0, m=1.0, r=[0.5, 0, 0])
    rob = Robot([l0, l1])
    want = np.array([1.0, 0.5, 0, 0, 0, 0.25, 0.25, 0, 0, 0] * 2)
    np.testing.assert_array_equal(rob.dynamic_parameters(), want)
    assert rob.dynamic_parameters().dtype == np.float64
    np.testing.assert_array_equal(ref.dynamic_parameters(rob.tree_description()), want)
    # a static link in front of a joint travels with it: its mass joins the group (and shifts h and Ib)
    s = Link(ET.tz(0.2), name="s", m=2.0, r=[0, 0, 0.1])
    j = Link(ET.Rz(), name="j", parent=s, m=1.0, r=[0.1, 0, 0])
    pi = Robot([s, j]).dynamic_parameters()
    np.testing.assert_allclose(pi, [3.0, 0.1, 0, 0.2, 0.02 + 0, 0.02 + 0.01, 0.01, 0, 0, 0], rtol=0, atol=1e-15)


@pytest.mark.parametrize("case", [(1, False, False), (2, False, False), (4, True, False), (6, True, True), (9, False, False),
                                  (12, True, False), (16, True, True)])
def test_generated_row_equals_the_reference_on_every_gravity_mask(tmp_path, case):
    n, branched, permute = case
    rng = np.random.default_rng(1000 + n)
    tree = sample_tree(rng, n, branched, permute)
    h = tree_handle(tree)
    for gm in range(8):
        grav = np.array([0.6, -1.1, -9.81]) * [(gm >> k) & 1 for k in range(3)]
        f = regressor_host_fn(tmp_path, f"r{n}_{gm}", h, gm)
        N = 3
        q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
        Y = f(-grav, q, qd, qdd)
        for r in range(N):
            want = ref.regressor(tree, q[r], qd[r], qdd[r], grav)
            np.testing.assert_allclose(Y[r], want, rtol=0, atol=1e-12 * max(1.0, np.abs(want).max()), err_msg=f"n={n} gm={gm}")
            for i in range(n):  # the structural zeros are exact
                out = np.repeat(~ref.below(tree, i), 10)
                assert np.all(Y[r, i, out] == 0.0)
                assert np.all(want[i, out] == 0.0)
    rtb._lib.lib().b2k_tree_destroy(h)


def test_generated_text_does_not_depend_on_the_inertias():
    rng = np.random.default_rng(7)
    tree = sample_tree(rng, 7, True)
    texts = []
    for scale in (1.0, 2.5):
        h = tree_handle(dict(tree, I6=[scale * np.asarray(I6) for I6 in tree["I6"]]))
        src = C.create_string_buffer(1 << 22)
        consts = np.zeros(8192)
        nc = C.c_int32()
        rtb._lib.check(rtb._lib.lib().b2k_tree_codegen(h, B2K_DYN_REGRESSOR, 7, src, len(src), rtb._lib.dptr(consts), 8192,
                                                       C.byref(nc), None))
        texts.append((src.value, consts[:nc.value].tobytes()))
        rtb._lib.lib().b2k_tree_destroy(h)
    assert texts[0] == texts[1]


NVRTC = any(os.path.exists(p) for p in ("/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so"))


@pytest.mark.skipif(not NVRTC, reason="NVRTC not installed")
@pytest.mark.parametrize("n", range(1, 17))
def test_regressor_kernel_builds_through_the_library_at_every_joint_count(n):
    """The regressor kernel builds for sm_90a in fp32 and fp64 at every n <= 16: one joint row's slab per warp fits the
    shared memory of an SM.  B2K_PRINT_BUILD_TIMES=1 prints the NVRTC time of each build."""
    lib = rtb._lib.lib()
    h = tree_handle(random_tree(np.random.default_rng(500 + n), n, True))
    for dt in (rtb._lib.F64, rtb._lib.F32):
        buf = C.create_string_buffer(4096)
        t0 = time.perf_counter()
        rtb._lib.check(lib.b2k_tree_info(h, B2K_DYN_REGRESSOR, dt, rtb._lib.dptr(np.array([0.5, -1.0, 3.0])), buf, 4096))
        info = buf.value.decode()
        assert info.startswith(f"k_rne_regressor_spec<{'double' if dt == rtb._lib.F64 else 'float'},tree n={n},mode=10>"), info[:600]
        if os.environ.get("B2K_PRINT_BUILD_TIMES"):
            print(f"n={n} dtype={dt}: {time.perf_counter() - t0:.2f} s: {info}")
    lib.b2k_tree_destroy(h)


def spong_handle():
    return tree_handle(dict(parent=[-1, 0], axis=[1, 1], flip=[0, 0], jindex=[0, 1], C=[np.eye(4), np.eye(4)],
                            I6=[orc.spatial_inertia(1, [0.5, 0, 0])] * 2))


def test_tree_regressor_rejects_bad_arguments_before_any_cuda_call():
    lib = rtb._lib.lib()
    h = spong_handle()
    buf = (C.c_double * 256)()
    p = C.cast(buf, C.c_void_p)
    mis = C.c_void_p(p.value + 8)
    g = rtb._lib.dptr(np.array([0.0, 0.0, 9.81]))
    n0 = rtb.launch_count()
    R = lib.b2k_tree_regressor

    def err(*a):
        assert R(*a) == -1, a
        assert lib.b2k_last_error().decode().startswith("b2k_tree_regressor: ")

    err(None, 1, p, p, p, 1, g, p, None)                       # handle
    err(h, 2, p, p, p, 1, g, p, None)                          # dtype
    err(h, 1, p, p, p, -1, g, p, None)                         # N < 0
    for k in range(4):                                         # NULL arrays with N > 0
        a = [p] * 4
        a[k] = None
        err(h, 1, a[0], a[1], a[2], 1, g, a[3], None)
    for k in range(4):                                         # 16-byte alignment
        a = [p] * 4
        a[k] = mis
        err(h, 1, a[0], a[1], a[2], 1, g, a[3], None)
    err(h, 1, p, p, p, 1, None, p, None)                       # grav
    assert R(h, 1, None, None, None, 0, g, None, None) == 0    # an empty batch is a no-op

    Gm = lib.b2k_tree_regressor_gram

    def gerr(*a):
        assert Gm(*a) == -1, a
        assert lib.b2k_last_error().decode().startswith("b2k_tree_regressor_gram: ")

    gerr(None, 1, p, p, p, p, 1, g, None, p, p, p, None)       # handle
    gerr(h, 2, p, p, p, p, 1, g, None, p, p, p, None)          # dtype
    gerr(h, 1, p, p, p, p, -1, g, None, p, p, p, None)         # N < 0
    gerr(h, 1, p, p, p, p, 1, None, None, p, p, p, None)       # grav
    for k in range(7):                                         # NULL arrays (G, b, s also at N = 0)
        a = [p] * 7
        a[k] = None
        gerr(h, 1, *a[:4], 1, g, None, *a[4:], None)
        if k >= 4:
            gerr(h, 1, None, None, None, None, 0, g, None, *a[4:], None)
    for k in range(7):                                         # alignment: inputs 16 bytes, tau the element, G / b / s 8
        a = [p] * 7
        a[k] = C.c_void_p(p.value + (4 if k >= 3 else 8))
        gerr(h, 1, *a[:4], 1, g, None, *a[4:], None)
    for bad in (np.array([1.0, -1.0]), np.array([np.nan, 1.0]), np.array([np.inf, 1.0])):  # weights
        gerr(h, 1, p, p, p, p, 1, g, rtb._lib.dptr(bad), p, p, p, None)
    assert rtb.launch_count() == n0
    lib.b2k_tree_destroy(h)


def test_op_codes_each_robot_kind_rejects():
    """B2K_DYN_REGRESSOR (10): b2k_tree_dyn and b2k_tree_derivatives reject it, b2k_tree_codegen and b2k_tree_info take
    it; the DH specialiser's code generator and info do not serve it.  The DH regressor's code 9 stays no tree operation."""
    lib = rtb._lib.lib()
    h = spong_handle()
    cbuf = (C.c_double * 64)()
    p = C.cast(cbuf, C.c_void_p)
    g = rtb._lib.dptr(np.array([0.0, 0.0, 9.81]))
    buf = C.create_string_buffer(1 << 20)
    assert lib.b2k_tree_dyn(h, 10, 1, p, p, p, 1, g, p, None) == -1
    assert "is not one of B2K_DYN_*" in lib.b2k_last_error().decode()
    assert lib.b2k_tree_derivatives(h, 10, 1, p, p, p, 1, g, p, p, None, None) == -1
    assert lib.b2k_tree_codegen(h, 10, 7, buf, len(buf), None, 0, None, None) == 0
    assert "rne_regressor_row(" in buf.value.decode()
    assert lib.b2k_tree_info(h, 10, 1, g, buf, 4096) == 0
    assert lib.b2k_tree_codegen(h, 9, 7, buf, len(buf), None, 0, None, None) == -1
    assert lib.b2k_tree_info(h, 9, 1, g, buf, 4096) == -1
    dh = rtb.models.Puma560()
    r = dh._rne_handle()
    assert lib.b2k_rne_codegen(r, 10, 7, 0, buf, 4096, None, 0, None, None) == -1
    assert lib.b2k_last_error().decode().startswith("b2k_rne_codegen: ")
    rc = lib.b2k_rne_spec_info(r, 10, 1, g, 0, buf, 4096)
    assert rc == -1 or "k_rne_spec" not in buf.value.decode(), buf.value.decode()
    lib.b2k_tree_destroy(h)
