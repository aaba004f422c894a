"""DHRobot.rne(..., base_wrench=True) without a GPU: the float64 reference of the base wrench (tests/rne_wrench_ref.py)
against two independent physical statements of the same quantity -- whole-robot momentum balance and six virtual joints
in front of the arm -- and the closed form at rest; the generated row function of B2K_GEN_RNE_WRENCH (compiled for the
host, as test_codegen_cpu.py does) against that reference; and the argument checks of the two C entry points."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import b2kin as rtb
import rne_wrench_ref as ref
from oracle import chains as ch
from oracle import oracle as orc

ROBOTS = ref.robots()
IDS = [r[0] for r in ROBOTS]
RNE_WRENCH = 6


def _base_rotation(rng):
    return (ch.trotz(rng.uniform(-3, 3)) @ ch.troty(rng.uniform(-1, 1)) @ ch.trotx(rng.uniform(-3, 3)))[:3, :3]


def _states(rng, N, n):
    return rng.uniform(-2, 2, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))


@pytest.mark.parametrize("name,n,mdh,L,physical", ROBOTS, ids=IDS)
def test_reference_tau_is_the_oracle_and_its_wrench_balances_momentum(name, n, mdh, L, physical):
    """tau of the restatement equals the oracle's rne; its wbase equals dP/dt and dH_O0/dt of the whole robot plus
    gravity and the tip wrench, with a rotated base (gravity enters in frame 0 as base^T g)."""
    rng = np.random.default_rng(sum(map(ord, name)))
    N = 40
    q, qd, qdd = _states(rng, N, n)
    Rb = _base_rotation(rng)
    g_b = Rb.T @ np.array([0.0, 0.0, -9.81])
    fx = rng.normal(size=6)
    tau, wb = ref.rne_wrench(n, mdh, L, -g_b, q, qd, qdd, fx)
    np.testing.assert_allclose(tau, orc.rne(n, mdh, L, -g_b, q, qd, qdd, fx), rtol=1e-12, atol=1e-12)
    want = ref.momentum_balance(n, mdh, L, g_b, q, qd, qdd, fx)
    scale = max(1.0, np.abs(want).max())
    if physical:
        np.testing.assert_allclose(wb, want, rtol=0, atol=2e-6 * scale)
    else:  # MDH, prismatic first joint: ne.c's recursion is not the physical one there, and neither is its wrench
        assert np.abs(wb - want).max() > 1e-3 * scale


@pytest.mark.parametrize("name,n,mdh,L,physical", [r for r in ROBOTS if r[4]], ids=[r[0] for r in ROBOTS if r[4]])
def test_wrench_equals_the_torques_of_six_virtual_joints(name, n, mdh, L, physical):
    """The links behind massless tx, ty, tz, Rx, Ry, Rz joints, assembled as tree groups with their full spatial
    inertia and evaluated at zero virtual coordinates by the oracle's spatial-vector recursion: the six virtual torques
    are the wrench the base exerts, in frame 0, moment about O_0."""
    rng = np.random.default_rng(7 + sum(map(ord, name)))
    N = 12
    q, qd, qdd = _states(rng, N, n)
    g = np.array([0.4, -0.3, -9.81])
    _, wb = ref.rne_wrench(n, mdh, L, -g, q, qd, qdd)
    want = ref.tree_wrench(n, mdh, L, q, qd, qdd, g)
    np.testing.assert_allclose(wb, want, rtol=1e-9, atol=1e-9 * max(1.0, np.abs(want).max()))


@pytest.mark.parametrize("name,n,mdh,L,physical", [r for r in ROBOTS if r[4]], ids=[r[0] for r in ROBOTS if r[4]])
def test_wrench_at_rest_holds_the_robot_up(name, n, mdh, L, physical):
    rng = np.random.default_rng(3)
    q = rng.uniform(-2, 2, (20, n))
    z = np.zeros_like(q)
    g_b = np.array([0.0, 0.0, -9.81])
    _, wb = ref.rne_wrench(n, mdh, L, -g_b, q, z, z)
    np.testing.assert_allclose(wb, ref.at_rest(n, mdh, L, g_b, q), rtol=1e-12, atol=1e-12)
    M = np.asarray(L).reshape(n, 24)[:, 6].sum()
    np.testing.assert_allclose(wb[:, 2], 9.81 * M, rtol=1e-12)  # fz = +9.81 sum m_i
    np.testing.assert_allclose(wb[:, :2], 0, atol=1e-12)


# ------------------------------------------------------------------ the generated row function of B2K_GEN_RNE_WRENCH
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
                     const double *q, const double *qd, const double *qdd, long N, double *out)
{
    for (long i = 0; i < N; i++) {
        double st[16], ct[16], th[16];
        for (int j = 0; j < n; j++) { th[j] = q[i * n + j] + offset[j]; st[j] = std::sin(th[j]); ct[j] = std::cos(th[j]); }
        rne_row(Cst, grav, fext, st, ct, th, qd + i * n, qdd + i * n, out + i * nout);
    }
}
"""


def _handle(n, mdh, L):
    h = C.c_void_p()
    rtb._lib.check(rtb._lib.lib().b2k_rne_create(n, int(mdh), rtb._lib.dptr(np.ascontiguousarray(L, dtype=np.float64)), C.byref(h)))
    return h


def _codegen(h, mode, grav_mask, has_fext):
    src = C.create_string_buffer(1 << 21)
    consts = np.zeros(4096)
    nc = C.c_int32()
    counts = (C.c_int32 * 3)()
    rtb._lib.check(rtb._lib.lib().b2k_rne_codegen(h, mode, grav_mask, has_fext, src, len(src), rtb._lib.dptr(consts), 4096,
                                                  C.byref(nc), counts))
    return src.value.decode(), consts[:nc.value].copy()


def _host_fn(tmp_path, tag, source):
    cpp, so = tmp_path / f"{tag}.cpp", tmp_path / f"{tag}.so"
    cpp.write_text(HARNESS % source)
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", str(cpp), "-o", str(so)])
    lib = C.CDLL(str(so))
    dp = C.POINTER(C.c_double)
    lib.eval.argtypes = [dp, dp, dp, dp, C.c_int, C.c_int, dp, dp, dp, C.c_long, dp]

    def run(consts, grav, fext, offset, n, q, qd, qdd):
        a = [np.ascontiguousarray(x, dtype=np.float64) for x in (consts, grav, fext, offset, q, qd, qdd)]
        out = np.zeros((q.shape[0], n + 6))
        lib.eval(*(x.ctypes.data_as(dp) for x in a[:4]), n, n + 6, *(x.ctypes.data_as(dp) for x in a[4:]), q.shape[0],
                 out.ctypes.data_as(dp))
        return out

    return run


GEN_ROBOTS = [r for r in ROBOTS if r[0] in ("puma560", "ur10", "panda_mdh", "rand_n1_dh", "rand_n3_mdh", "rand_n7_dh",
                                            "rand_n10_mdh", "prismatic1_n5_mdh", "prismatic2_n3_dh", "prismatic_first_mdh_n3")]


@pytest.mark.parametrize("name,n,mdh,L,physical", GEN_ROBOTS, ids=[r[0] for r in GEN_ROBOTS])
def test_generated_wrench_row_equals_the_reference(tmp_path, name, n, mdh, L, physical):
    """Every gravity mask, with and without a tip wrench: out = [tau | wbase] of the generated function."""
    rng = np.random.default_rng(len(name) + n)
    N = 60
    q, qd, qdd = rng.uniform(-3, 3, (N, n)), rng.normal(size=(N, n)), rng.normal(size=(N, n))
    qd[-4:] = 0.0
    h = _handle(n, mdh, L)
    offset = np.asarray(L).reshape(n, 24)[:, 5]
    gfull = np.array([0.3, -0.2, 9.81])
    for gm in range(8):
        g = np.where([gm & 1, gm & 2, gm & 4], gfull, 0.0)
        for fx in (None, rng.normal(size=6)):
            src, cst = _codegen(h, RNE_WRENCH, gm, int(fx is not None))
            got = _host_fn(tmp_path, f"w{gm}{fx is not None}", src)(cst, g, np.zeros(6) if fx is None else fx, offset, n, q, qd, qdd)
            tau, wb = ref.rne_wrench(n, mdh, L, g, q, qd, qdd, fx)
            np.testing.assert_allclose(got[:, :n], tau, rtol=1e-9, atol=1e-9, err_msg=f"tau gmask={gm} fext={fx is not None}")
            np.testing.assert_allclose(got[:, n:], wb, rtol=1e-9, atol=1e-9, err_msg=f"wbase gmask={gm} fext={fx is not None}")
    rtb._lib.lib().b2k_rne_destroy(h)


def test_tree_robots_reject_the_wrench_mode():
    lib = rtb._lib.lib()
    i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)  # noqa: E731
    keep = [i32(x) for x in ([-1, 0], [1, 1], [0, 0], [0, 1])]
    Cm = np.ascontiguousarray(np.stack([np.eye(4)[:3], ch.transl(1, 0, 0)[:3]]).reshape(2, 12))
    I6 = np.ascontiguousarray(np.stack([orc.spatial_inertia(1, [0.5, 0, 0])] * 2).reshape(2, 36))
    h = C.c_void_p()
    rtb._lib.check(lib.b2k_tree_create(2, *(k.ctypes.data_as(rtb._lib.ip) for k in keep), rtb._lib.dptr(Cm), rtb._lib.dptr(I6), C.byref(h)))
    src = C.create_string_buffer(1 << 16)
    consts = np.zeros(256)
    assert lib.b2k_tree_codegen(h, RNE_WRENCH, 7, src, len(src), rtb._lib.dptr(consts), 256, None, None) == -1
    assert b"base wrench" in lib.b2k_last_error()
    g = np.array([0.0, 0.0, 9.81])
    assert lib.b2k_tree_info(h, RNE_WRENCH, 1, rtb._lib.dptr(g), src, len(src)) == -1
    assert lib.b2k_tree_dyn(h, RNE_WRENCH, 1, None, None, None, 0, rtb._lib.dptr(g), None, None) == -1
    # the six existing operations still generate
    for op in range(6):
        rtb._lib.check(lib.b2k_tree_codegen(h, op, 7, src, len(src), rtb._lib.dptr(consts), 256, None, None))
    lib.b2k_tree_destroy(h)


# ------------------------------------------------------------------ C ABI argument checks
def _bad_calls(h, p, g, host):
    """(description, arguments, expected message) for b2k_rne_wrench[_host]; everything else valid, N = 4 rows."""
    tail = (0,) if host else (None,)  # device ordinal / stream
    ok = dict(r=h, dt=1, q=p, qd=p, qdd=p, N=4, grav=g, fext=None, tau=p, wb=p)
    cases = [("NULL handle", dict(r=None), "handle is NULL"), ("bad dtype", dict(dt=7), "dtype"), ("negative N", dict(N=-1), ""),
             ("NULL q", dict(q=None), "NULL"), ("NULL qd", dict(qd=None), "NULL"), ("NULL qdd", dict(qdd=None), "NULL"),
             ("NULL tau", dict(tau=None), "NULL"), ("NULL wbase", dict(wb=None), "NULL"),
             ("misaligned wbase", dict(wb=p + (4 if host else 8)), "wbase must be")]
    if not host:
        cases += [("NULL grav", dict(grav=None), "grav is NULL"), ("misaligned tau", dict(tau=p + 4), "tau must be"),
                  ("misaligned fp32 wbase", dict(dt=0, wb=p + 4), "wbase must be 8-byte")]
    out = []
    for what, over, msg in cases:
        a = dict(ok, **over)
        out.append((what, (a["r"], a["dt"], a["q"], a["qd"], a["qdd"], a["N"], a["grav"], a["fext"], a["tau"], a["wb"]) + tail, msg))
    return out


@pytest.mark.parametrize("entry", ["b2k_rne_wrench", "b2k_rne_wrench_host"])
def test_entry_points_reject_bad_arguments_before_any_cuda_call(entry):
    """The host buffer stands in for a (never dereferenced) device pointer.  Without a device, an entry point that
    reached the CUDA runtime first would report a CUDA error (not -1) and could not be this quick to refuse."""
    lib = rtb._lib.lib()
    h = _handle(6, 0, ch.pack_rne(ch.puma560_links()))
    buf = np.zeros(256)
    p = buf.ctypes.data + (-buf.ctypes.data) % 64
    g = np.array([0.0, 0.0, 9.81])
    n0 = lib.b2k_launch_count()
    for what, args, msg in _bad_calls(h, p, rtb._lib.dptr(g), entry.endswith("_host")):
        assert getattr(lib, entry)(*args) == -1, what
        assert msg.encode() in lib.b2k_last_error(), (what, lib.b2k_last_error())
    assert lib.b2k_launch_count() == n0
    # N = 0 with every array NULL is a valid empty call
    assert getattr(lib, entry)(h, 1, None, None, None, 0, rtb._lib.dptr(g), None, None, None, 0 if entry.endswith("_host") else None) == 0
    lib.b2k_rne_destroy(h)
