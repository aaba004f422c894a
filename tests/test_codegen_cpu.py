"""The robot-specialised RNE code generator (csrc/b2k_rne_gen.cpp), checked WITHOUT a GPU: the row function it
emits is plain C in terms of `real`, so the same text the library hands to NVRTC is compiled here for the host
(g++) and compared with the oracle -- the C restatement of the reference's ne.c -- on seeded inputs, for every
operation the generator serves (rne + the five dynamics fan-outs), standard and modified DH, the benchmark robots
and random arms with random sparsity.  Also: the generated text compiles for sm_90a through the library's own
NVRTC path (no device needed for that), and what it leaves out (zero terms) is reported."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import b2kin as rtb
from oracle import chains as ch
from oracle import oracle as orc

MODES = {"rne": 0, "inertia": 1, "gravload": 2, "itorque": 3, "coriolis": 4, "accel": 5}

HARNESS = r"""
#include <cmath>
#define __device__
#define __forceinline__ inline
typedef double real;
using std::fma;
static inline real step_pos(real x) { return x > 0 ? 1.0 : 0.0; }
static inline real step_neg(real x) { return x < 0 ? 1.0 : 0.0; }
%s
extern "C" void eval(const double *Cst, const double *grav, const double *fext, const double *offset, int n, int nout,
                     const double *q, const double *a1, const double *a2, long N, double *out)
{
    for (long i = 0; i < N; i++) {
        double st[16], ct[16], th[16], z[16] = {0};
        for (int j = 0; j < n; j++) { th[j] = q[i * n + j] + offset[j]; st[j] = std::sin(th[j]); ct[j] = std::cos(th[j]); }
        rne_row(Cst, grav, fext, st, ct, th, a1 ? a1 + i * n : z, a2 ? a2 + i * n : z, out + i * nout);
    }
}
"""


def handle(n, mdh, L):
    h = C.c_void_p()
    L = np.ascontiguousarray(L, dtype=np.float64)
    rtb._lib.check(rtb._lib.lib().b2k_rne_create(n, int(mdh), rtb._lib.dptr(L), C.byref(h)))
    return h


def codegen(h, mode, grav_mask=7, has_fext=0):
    lib = rtb._lib.lib()
    src = C.create_string_buffer(1 << 21)
    consts = np.zeros(4096)
    nc = C.c_int32()
    counts = (C.c_int32 * 3)()
    rtb._lib.check(lib.b2k_rne_codegen(h, mode, grav_mask, has_fext, src, len(src), rtb._lib.dptr(consts), 4096, C.byref(nc), counts))
    return src.value.decode(), consts[:nc.value].copy(), tuple(counts)


def host_fn(tmp_path, tag, source):
    cpp = tmp_path / f"{tag}.cpp"
    so = tmp_path / f"{tag}.so"
    cpp.write_text(HARNESS % source)
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", str(cpp), "-o", str(so)])
    lib = C.CDLL(str(so))
    dp = C.POINTER(C.c_double)
    lib.eval.argtypes = [dp, dp, dp, dp, C.c_int, C.c_int, dp, dp, dp, C.c_long, dp]

    def run(consts, grav, fext, offset, n, nout, q, a1=None, a2=None):
        q = np.ascontiguousarray(q, dtype=np.float64)
        out = np.zeros((q.shape[0], nout))
        p = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(dp)  # noqa: E731
        keep = [np.ascontiguousarray(x, dtype=np.float64) for x in (consts, grav, fext, offset)]
        lib.eval(*(k.ctypes.data_as(dp) for k in keep), n, nout, q.ctypes.data_as(dp), p(a1), p(a2), q.shape[0], out.ctypes.data_as(dp))
        return out

    return run


def random_links(rng, n, mdh, prismatic=False):
    """Arm with a random mix of structural zeros (alpha = k pi/2, a / d = 0, sparse r and I); with `prismatic`
    about every other joint is translational (theta fixed, d = q + offset)."""
    links = []
    for k in range(n):
        alpha = rng.choice([0.0, np.pi / 2, -np.pi / 2, np.pi, rng.uniform(-1, 1)])
        I6 = rng.uniform(0.01, 0.5, 3).tolist() + (rng.uniform(-0.01, 0.01, 3) * rng.integers(0, 2, 3)).tolist()
        links.append(dict(d=float(rng.choice([0.0, rng.uniform(-0.5, 0.5)])), a=float(rng.choice([0.0, rng.uniform(-0.5, 0.5)])),
                          alpha=float(alpha), offset=float(rng.choice([0.0, rng.uniform(-1, 1)])),
                          I=I6, r=(rng.uniform(-0.3, 0.3, 3) * rng.integers(0, 2, 3)).tolist(), m=float(rng.uniform(0, 5)),
                          Jm=float(rng.choice([0.0, 2e-4])), G=float(rng.choice([0.0, -60.0, 100.0])),
                          B=float(rng.choice([0.0, 1e-3])), Tc=[float(rng.choice([0.0, 0.3])), float(rng.choice([0.0, -0.4]))]))
        if prismatic and (k % 2 == 0 or rng.random() < 0.3):
            links[-1].update(sigma=1, theta=float(rng.choice([0.0, np.pi / 2, rng.uniform(-1, 1)])))
    return links


def robots():
    rng = np.random.default_rng(11)
    out = [("puma560", 6, 0, ch.pack_rne(ch.puma560_links())), ("panda_mdh", 7, 1, ch.pack_rne(ch.panda_mdh_links(), mdh=True))]
    for k, (n, mdh) in enumerate([(3, 0), (7, 0), (5, 1), (2, 1), (1, 0)]):
        out.append((f"random{k}_n{n}_{'mdh' if mdh else 'dh'}", n, mdh, ch.pack_rne(random_links(rng, n, mdh), mdh=bool(mdh))))
    for k, (n, mdh) in enumerate([(4, 0), (5, 1), (1, 1), (3, 1)]):  # chains with prismatic joints (incl. a prismatic FIRST joint under MDH)
        out.append((f"prismatic{k}_n{n}_{'mdh' if mdh else 'dh'}", n, mdh, ch.pack_rne(random_links(rng, n, mdh, True), mdh=bool(mdh))))
    return out


@pytest.mark.parametrize("name,n,mdh,L", robots(), ids=[r[0] for r in robots()])
def test_generated_recursion_equals_the_oracle(tmp_path, name, n, mdh, L):
    rng = np.random.default_rng(abs(hash(name)) % 2**31)
    h = handle(n, mdh, L)
    offset = np.asarray(L).reshape(n, 24)[:, 5]
    N = 200
    q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
    qd[-5:] = 0.0  # Coulomb branch at rest
    tq = rng.normal(size=(N, n))
    Lnf = orc.nofriction_L(L)
    rne = lambda a, b, c, g, fx=None: orc.rne(n, mdh, L, g, a, b, c, fx)  # noqa: E731
    rne_nf = lambda a, b, c, g: orc.rne(n, mdh, Lnf, g, a, b, c)  # noqa: E731
    tol = dict(rtol=1e-9, atol=1e-9)
    z6 = np.zeros(6)

    # rne: full gravity + tip wrench; gravity along z only, no wrench (the common call)
    for gm, g, fx in ((7, np.array([0.3, -0.2, 9.81]), np.array([1.0, 2, 3, 1, 2, 3])), (4, np.array([0, 0, 9.81]), None)):
        src, cst, cnt = codegen(h, MODES["rne"], gm, int(fx is not None))
        f = host_fn(tmp_path, f"rne{gm}", src)
        got = f(cst, g, z6 if fx is None else fx, offset, n, n, q, qd, qdd)
        np.testing.assert_allclose(got, rne(q, qd, qdd, g, fx), **tol)
    g = np.array([0, 0, 9.81])
    src, cst, _ = codegen(h, MODES["gravload"], 4)
    np.testing.assert_allclose(host_fn(tmp_path, "grav", src)(cst, g, z6, offset, n, n, q), orc.dyn_gravload(rne, n, q, g), **tol)
    src, cst, _ = codegen(h, MODES["itorque"], 0)
    np.testing.assert_allclose(host_fn(tmp_path, "itq", src)(cst, g, z6, offset, n, n, q, qdd), orc.dyn_itorque(rne, n, q, qdd), **tol)
    src, cst, _ = codegen(h, MODES["inertia"], 0)
    M = host_fn(tmp_path, "inertia", src)(cst, g, z6, offset, n, n * n, q[:40]).reshape(-1, n, n)
    np.testing.assert_allclose(M, orc.dyn_inertia(rne, n, q[:40]), **tol)
    src, cst, _ = codegen(h, MODES["coriolis"], 0)
    Cm = host_fn(tmp_path, "coriolis", src)(cst, g, z6, offset, n, n * n, q[:20], qd[:20]).reshape(-1, n, n)
    np.testing.assert_allclose(Cm, orc.dyn_coriolis(rne_nf, n, q[:20], qd[:20]), **tol)
    # accel: the generated function returns [M | torque - rne(q, qd, 0)]; the kernel wrapper solves the system
    src, cst, _ = codegen(h, MODES["accel"], 4)
    res = host_fn(tmp_path, "accel", src)(cst, g, z6, offset, n, n * n + n, q[:40], qd[:40], tq[:40])
    Mi = orc.dyn_inertia(rne, n, q[:40])
    np.testing.assert_allclose(res[:, :n * n].reshape(-1, n, n), Mi, **tol)
    np.testing.assert_allclose(res[:, n * n:], tq[:40] - rne(q[:40], qd[:40], np.zeros((40, n)), g), **tol)
    if np.all(np.linalg.cond(Mi) < 1e8):
        np.testing.assert_allclose(np.linalg.solve(res[:, :n * n].reshape(-1, n, n), res[:, n * n:, None])[..., 0],
                                   orc.dyn_accel(rne, n, q[:40], qd[:40], tq[:40], g), rtol=1e-7, atol=1e-7)
    rtb._lib.lib().b2k_rne_destroy(h)


def test_specialisation_drops_the_structural_zeros_of_the_puma():
    """What the generator is for: the Puma560 recursion shrinks from ~750 generic multiply-adds to ~330."""
    h = handle(6, 0, ch.pack_rne(ch.puma560_links()))
    _, _, (mul, fma, add) = codegen(h, MODES["rne"], 4, 0)
    assert mul + fma + add < 360, (mul, fma, add)
    _, _, full = codegen(h, MODES["rne"], 7, 1)
    assert sum(full) > mul + fma + add  # dense gravity and a tip wrench cost extra terms
    _, _, inertia = codegen(h, MODES["inertia"], 0)
    assert sum(inertia) < 6 * 200
    # a dense random arm keeps (nearly) everything
    rng = np.random.default_rng(5)
    dense = [dict(d=0.1 + 0.1 * k, a=0.2, alpha=0.3 + 0.1 * k, offset=0.0, I=rng.uniform(0.01, 0.1, 6).tolist(),
                  r=rng.uniform(-0.1, 0.1, 3).tolist(), m=1.0, Jm=1e-4, G=50.0, B=1e-3, Tc=[0.1, -0.1]) for k in range(6)]
    hd = handle(6, 0, ch.pack_rne(dense))
    _, _, cd = codegen(hd, MODES["rne"], 7, 1)
    assert sum(cd) > 2 * (mul + fma + add)
    rtb._lib.lib().b2k_rne_destroy(h)
    rtb._lib.lib().b2k_rne_destroy(hd)


@pytest.mark.skipif(not any(os.path.exists(p) for p in ("/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so")),
                    reason="NVRTC not installed")
def test_generated_kernels_compile_for_sm_90a_through_the_library():
    """The library's own NVRTC path (needs no device): every operation x dtype builds for Puma560 and Panda MDH."""
    lib = rtb._lib.lib()
    g = np.array([0.0, 0.0, 9.81])
    for n, mdh, L in ((6, 0, ch.pack_rne(ch.puma560_links())), (7, 1, ch.pack_rne(ch.panda_mdh_links(), mdh=True))):
        h = handle(n, mdh, L)
        for mode in list(range(6)) + [205]:  # 205: the forward-dynamics integrator around the accel recursion
            for dt in (rtb._lib.F64, rtb._lib.F32):
                buf = C.create_string_buffer(4096)
                rtb._lib.check(lib.b2k_rne_spec_info(h, mode, dt, rtb._lib.dptr(g), 0, buf, 4096))
                assert buf.value.startswith(b"k_fdyn<" if mode == 205 else b"k_rne_spec<"), buf.value[:600]
        lib.b2k_rne_destroy(h)


@pytest.mark.skipif(not any(os.path.exists(p) for p in ("/usr/local/cuda/lib64/libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so")),
                    reason="NVRTC not installed")
@pytest.mark.parametrize("n", range(1, 11))
def test_fdyn_integrator_compiles_at_every_joint_count(n):
    """k_fdyn carries K[7][2n] and the n*n + n LDL^T scratch per lane: it builds for sm_90a at every joint count the
    device sweep runs (tests/test_gpu_fdyn.py), DH at odd n and MDH at even n, in both dtypes."""
    lib = rtb._lib.lib()
    mdh = n % 2 == 0
    h = handle(n, mdh, ch.pack_rne(random_links(np.random.default_rng(900 + n), n, mdh), mdh=mdh))
    for dt in (rtb._lib.F64, rtb._lib.F32):
        buf = C.create_string_buffer(4096)
        rtb._lib.check(lib.b2k_rne_spec_info(h, 205, dt, rtb._lib.dptr(np.array([0.5, -1.0, 3.0])), 0, buf, 4096))
        assert buf.value.startswith(b"k_fdyn<"), buf.value[:600]
    lib.b2k_rne_destroy(h)


# ------------------------------------------------------------------ rigid-body trees (Robot.rne)
TREE_HARNESS = r"""
#include <cmath>
#define __device__
#define __forceinline__ inline
typedef double real;
using std::fma;
%s
extern "C" void eval(const double *Cst, const double *grav, int n, const double *q, const double *qd, const double *qdd, long N,
                     double *out, int nres)
{
    double fext[6] = {0};
    for (long i = 0; i < N; i++) {
        double st[16], ct[16];
        for (int j = 0; j < n; j++) { st[j] = std::sin(q[i * n + j]); ct[j] = std::cos(q[i * n + j]); }
        rne_row(Cst, grav, fext, st, ct, q + i * n, qd + i * n, qdd + i * n, out + i * nres);
    }
}
"""


def tree_handle(tree):
    n = len(tree["parent"])
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731
    Cm = np.ascontiguousarray(np.asarray(tree["C"], dtype=np.float64)[:, :3, :].reshape(n, 12))
    I6 = np.ascontiguousarray(np.asarray(tree["I6"], dtype=np.float64).reshape(n, 36))
    h = C.c_void_p()
    ip = rtb._lib.ip
    keep = [i32(tree[k]) for k in ("parent", "axis", "flip", "jindex")]
    rtb._lib.check(rtb._lib.lib().b2k_tree_create(n, *(k.ctypes.data_as(ip) for k in keep), rtb._lib.dptr(Cm), rtb._lib.dptr(I6), C.byref(h)))
    return h


def tree_host_fn(tmp_path, tag, h, grav_mask, op=0):
    """The generated row function of operation `op` (0 rne ... 5 accel) compiled for the host: run(grav, q, in1, in2) ->
    (N, nres) with nres = n (rne, gravload, itorque), n*n (inertia, coriolis) or n*n + n (accel: [M | tau - bias])."""
    lib = rtb._lib.lib()
    src = C.create_string_buffer(1 << 23)
    consts = np.zeros(8192)
    nc = C.c_int32()
    counts = (C.c_int32 * 3)()
    rtb._lib.check(lib.b2k_tree_codegen(h, op, grav_mask, src, len(src), rtb._lib.dptr(consts), 8192, C.byref(nc), counts))
    cpp, so = tmp_path / f"{tag}.cpp", tmp_path / f"{tag}.so"
    cpp.write_text(TREE_HARNESS % src.value.decode())
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", str(cpp), "-o", str(so)])
    L = C.CDLL(str(so))
    dp = C.POINTER(C.c_double)
    L.eval.argtypes = [dp, dp, C.c_int, dp, dp, dp, C.c_long, dp, C.c_int]
    cst = consts[:nc.value].copy()

    def run(grav, q, qd, qdd):
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in (cst, grav, q, qd, qdd)]
        n = a[2].shape[1]
        nres = {0: n, 1: n * n, 2: n, 3: n, 4: n * n, 5: n * n + n}[op]
        out = np.zeros((a[2].shape[0], nres))
        L.eval(a[0].ctypes.data_as(dp), a[1].ctypes.data_as(dp), n, a[2].ctypes.data_as(dp), a[3].ctypes.data_as(dp),
               a[4].ctypes.data_as(dp), a[2].shape[0], out.ctypes.data_as(dp), nres)
        return out

    return run, tuple(counts)


def random_tree(rng, n, branched=True):
    parent = [-1] + [int(rng.integers(0, j)) if branched else j - 1 for j in range(1, n)]
    Cs = []
    for _ in range(n):
        if rng.random() < 0.5:  # axis-aligned constant (URDF style: rpy multiples of pi/2) or a general one
            R = ch.trotz(rng.choice([0, np.pi / 2, -np.pi / 2, np.pi])) @ ch.trotx(rng.choice([0, np.pi / 2, -np.pi / 2]))
        else:
            R = ch.trotz(rng.uniform(-3, 3)) @ ch.troty(rng.uniform(-1, 1)) @ ch.trotx(rng.uniform(-3, 3))
        T = R.copy()
        T[:3, 3] = rng.uniform(-0.4, 0.4, 3) * rng.integers(0, 2, 3)
        Cs.append(T)
    I6 = [orc.spatial_inertia(rng.uniform(0.2, 3), rng.uniform(-0.2, 0.2, 3) * rng.integers(0, 2, 3))
          + (orc.spatial_inertia(rng.uniform(0.1, 1), rng.uniform(-0.2, 0.2, 3)) if rng.random() < 0.3 else 0) for _ in range(n)]
    return dict(parent=parent, axis=[int(a) for a in rng.integers(0, 6, n)], flip=[int(f) for f in rng.integers(0, 2, n)],
                jindex=list(range(n)), C=Cs, I6=I6)


def test_generated_tree_recursion_equals_featherstone_oracle(tmp_path):
    """Robot.rne for rigid-body trees: the generated row function against the numpy restatement of the reference's
    spatial-vector recursion (which reproduces the reference's own KATs, tests/test_ERobot.py:100-154: checked here too)."""
    pi = np.pi
    spong = dict(parent=[-1, 0], axis=[1, 1], flip=[0, 0], jindex=[0, 1], C=[np.eye(4), ch.transl(1, 0, 0)],
                 I6=[orc.spatial_inertia(1, [0.5, 0, 0])] * 2)
    h = tree_handle(spong)
    f, cnt = tree_host_fn(tmp_path, "spong", h, 4)
    z = np.zeros((1, 2))
    g = np.array([0, 0, 9.81])  # a_grav = -gravity
    np.testing.assert_allclose(f(g, z, z, z) / 9.81, [[-2, -0.5]], atol=1e-12)
    np.testing.assert_allclose(f(g, [[0.0, -pi / 2]], z, z) / 9.81, [[-1.5, 0]], atol=1e-12)
    np.testing.assert_allclose(f(g, [[-pi / 2, pi / 2]], z, z) / 9.81, [[-0.5, -0.5]], atol=1e-12)
    f0, _ = tree_host_fn(tmp_path, "spong0", h, 0)
    q = np.array([[0, -pi / 2]])
    hh = -0.5 * np.sin(q[0, 1])
    np.testing.assert_allclose(f0(np.zeros(3), q, [[1.0, 1.0]], z), [np.r_[3, -1] * hh], atol=1e-12)
    d11, d12 = 1.5 + np.cos(q[0, 1]), 0.25 + 0.5 * np.cos(q[0, 1])
    np.testing.assert_allclose(f0(np.zeros(3), q, z, [[1.0, 1.0]]), [[d11 + d12, d12 + 0.25]], atol=1e-12)
    rtb._lib.lib().b2k_tree_destroy(h)
    rng = np.random.default_rng(77)
    for k, (n, branched) in enumerate([(1, False), (3, False), (6, True), (9, True), (16, True)]):
        tree = random_tree(rng, n, branched)
        h = tree_handle(tree)
        N = 60
        q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
        for gm, grav in ((7, np.array([0.5, -1.0, -9.81])), (4, np.array([0, 0, -9.81])), (0, np.zeros(3))):
            f, cnt = tree_host_fn(tmp_path, f"t{k}_{gm}", h, gm)
            np.testing.assert_allclose(f(-grav, q, qd, qdd), orc.tree_rne(tree, q, qd, qdd, grav), rtol=1e-9, atol=1e-9,
                                       err_msg=f"tree {k} n={n} gmask={gm}")
        rtb._lib.lib().b2k_tree_destroy(h)
    # validation
    lib = rtb._lib.lib()
    bad = dict(spong, parent=[0, -1])
    with pytest.raises(ValueError, match="precede"):
        tree_handle(bad)
    with pytest.raises(ValueError, match="permutation"):
        tree_handle(dict(spong, jindex=[0, 0]))
    assert lib.b2k_tree_rne(None, 1, None, None, None, 0, None, None, None) == -1


def test_generated_tree_dynamics_operations_equal_the_reference_loops(tmp_path):
    """inertia / gravload / itorque / coriolis / accel for tree robots: the reference's DynamicsMixin loops (restated in
    oracle.dyn_*) over the Featherstone oracle against the generated row functions -- including a tree whose jindex is
    not the group order (inputs are in q order, torques in group order)."""
    rng = np.random.default_rng(99)
    solved = 0
    for k, (n, branched, permute) in enumerate([(2, False, False), (5, True, False), (6, True, True), (4, False, True)]):
        tree = random_tree(rng, n, branched)
        if k >= 2:  # off-axis point masses everywhere: a regular inertia matrix for the accel check (the recursion uses
            # mass and centre of mass only, so a link whose mass sits on its own joint axis makes M singular -- in the
            # reference too)
            tree["I6"] = [orc.spatial_inertia(rng.uniform(0.5, 2), rng.uniform(0.1, 0.3, 3) * rng.choice([-1, 1], 3))
                          + orc.spatial_inertia(rng.uniform(0.5, 2), rng.uniform(0.1, 0.3, 3) * rng.choice([-1, 1], 3)) for _ in range(n)]
            tree["axis"] = [int(a) for a in rng.integers(0, 3, n)]
        if permute:
            tree["jindex"] = [int(i) for i in rng.permutation(n)]
        h = tree_handle(tree)
        N = 12
        q, qd, x = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
        grav = np.array([0.3, -0.7, -9.81])
        z = np.zeros((N, n))

        def rne_fn(a, b, c, g):  # the oracle's calling convention: the gravity argument is the robot's gravity vector
            return orc.tree_rne(tree, np.atleast_2d(a), np.atleast_2d(b), np.atleast_2d(c), g)

        tol = dict(rtol=1e-9, atol=1e-9)
        f, _ = tree_host_fn(tmp_path, f"d{k}_in", h, 0, op=1)
        M = f(np.zeros(3), q, z, z).reshape(N, n, n)
        np.testing.assert_allclose(M, orc.dyn_inertia(rne_fn, n, q), **tol)
        f, _ = tree_host_fn(tmp_path, f"d{k}_gl", h, 7, op=2)
        np.testing.assert_allclose(f(-grav, q, z, z), orc.dyn_gravload(rne_fn, n, q, grav), **tol)
        f, _ = tree_host_fn(tmp_path, f"d{k}_it", h, 0, op=3)
        np.testing.assert_allclose(f(np.zeros(3), q, x, z), orc.dyn_itorque(rne_fn, n, q, x), **tol)
        f, _ = tree_host_fn(tmp_path, f"d{k}_co", h, 0, op=4)
        np.testing.assert_allclose(f(np.zeros(3), q, qd, z).reshape(N, n, n), orc.dyn_coriolis(rne_fn, n, q, qd), **tol)
        f, _ = tree_host_fn(tmp_path, f"d{k}_ac", h, 7, op=5)
        res = f(-grav, q, qd, x)
        Mi, rhs = res[:, :n * n].reshape(N, n, n), res[:, n * n:]
        np.testing.assert_allclose(Mi, orc.dyn_inertia(rne_fn, n, q), **tol)
        # the kernel wrapper solves M^T-free: rows of the generated M are torques for unit accelerations (symmetric matrix)
        if np.linalg.cond(Mi).max() < 1e6:
            qdd = np.stack([np.linalg.solve(Mi[i], rhs[i]) for i in range(N)])
            np.testing.assert_allclose(qdd, orc.dyn_accel(rne_fn, n, q, qd, x, grav), rtol=1e-6, atol=1e-7)
            solved += 1
        rtb._lib.lib().b2k_tree_destroy(h)
    assert solved >= 2
