"""CPU-side tests of the drop-in boundary and the host logic (no GPU needed):

* libb2kin.so loads and exports every symbol include/b2kin.h declares;
* handle creation / validation paths of the C ABI that never touch a device;
* the host-side mirror of the reference interface (ET / ETS composition, jindex numbering,
  DH -> ETS expansion, RNE packing + dirty tracking, shape sniffing, error behaviour);
* the product never imports the oracle, and fails loudly without a CUDA device;
* row sharding helpers, including a world_size-2 gloo run of the multi-GPU code path.
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import b2kin as rtb
from oracle import chains as ch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
PKG = os.path.join(ROOT, "robotics-toolbox-python_b200")


# ------------------------------------------------------------------ the C ABI
def header_symbols():
    src = open(os.path.join(ROOT, "include", "b2kin.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2k_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = rtb._lib.lib()
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/b2kin.h but not exported by libb2kin.so"
    # and the Python binding covers the whole header
    assert set(syms) == set(rtb._lib.EXPORTED_SYMBOLS)
    assert lib.b2k_version() == 100


def test_library_is_cuda_not_torch():
    """The boundary is a plain C-ABI shared object: no torch / python symbols in its dynamic deps."""
    out = subprocess.run(["ldd", rtb._lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "torch" not in out and "python" not in out
    import shutil

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-lelf", rtb._lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass


def test_chain_create_validation():
    lib = rtb._lib.lib()
    d = ch.panda_ets()
    ip, dp = rtb._lib.ip, rtb._lib.dp
    h = C.c_void_p()
    args = lambda dd: (len(dd["isjoint"]), dd["isjoint"].ctypes.data_as(ip), dd["axis"].ctypes.data_as(ip),  # noqa: E731
                       dd["flip"].ctypes.data_as(ip), dd["jindex"].ctypes.data_as(ip),
                       np.ascontiguousarray(dd["T"]).ctypes.data_as(dp), np.ascontiguousarray(dd["qlim"]).ctypes.data_as(dp))
    assert lib.b2k_chain_create(*args(d), C.byref(h)) == 0 and h.value
    n, m, w = C.c_int(), C.c_int(), C.c_int()
    assert lib.b2k_chain_info(h, C.byref(n), C.byref(m), C.byref(w)) == 0
    assert (n.value, m.value, w.value) == (7, 22, 7)
    assert lib.b2k_chain_destroy(h) == 0
    # too many joints
    rng = np.random.default_rng(0)
    big = ch.random_chain(rng, n_joints=11)
    assert lib.b2k_chain_create(*args(big), C.byref(h)) == -1
    assert b"joints" in lib.b2k_last_error()
    # non-affine constant
    bad = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in d.items()}
    bad["T"][0][3, 0] = 0.5
    assert lib.b2k_chain_create(*args(bad), C.byref(h)) == -1
    assert b"affine" in lib.b2k_last_error()
    # bad axis code
    bad = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in d.items()}
    bad["axis"][1] = 9
    assert lib.b2k_chain_create(*args(bad), C.byref(h)) == -1
    # compute entry points validate before launching anything
    assert lib.b2k_fkine(None, 1, None, 1, 7, None, None, None, None) == -1
    assert b"NULL" in lib.b2k_last_error()


def test_rne_create_validation():
    lib = rtb._lib.lib()
    L = ch.pack_rne(ch.puma560_links())
    h = C.c_void_p()
    assert lib.b2k_rne_create(6, 0, L.ctypes.data_as(rtb._lib.dp), C.byref(h)) == 0
    assert lib.b2k_rne_destroy(h) == 0
    assert lib.b2k_rne_create(6, 2, L.ctypes.data_as(rtb._lib.dp), C.byref(h)) == -1
    L2 = L.copy(); L2[4] = 3  # invalid joint type: frne.c:203-205 raises ValueError
    assert lib.b2k_rne_create(6, 0, L2.ctypes.data_as(rtb._lib.dp), C.byref(h)) == -1
    assert lib.b2k_rne_create(0, 0, L.ctypes.data_as(rtb._lib.dp), C.byref(h)) == -1


def test_widened_entry_points_validate_before_launching():
    """The entry points of the widened rows (SURVEY 8f) reject bad arguments with a status code and a message
    before any CUDA call, like the core ones."""
    lib = rtb._lib.lib()
    dp = rtb._lib.dp
    q0 = np.zeros(6)
    buf = np.zeros(64)  # stands in for a (never dereferenced) device pointer
    p = buf.ctypes.data
    assert lib.b2k_jtraj(1, 0, q0.ctypes.data_as(dp), q0.ctypes.data_as(dp), None, None, 8, None, 1.0, p, p, p, None) == -1
    assert b"n must be" in lib.b2k_last_error()
    assert lib.b2k_jtraj(1, 6, q0.ctypes.data_as(dp), q0.ctypes.data_as(dp), None, None, 8, None, 0.0, p, p, p, None) == -1
    assert b"tscal" in lib.b2k_last_error()
    assert lib.b2k_jtraj(7, 6, q0.ctypes.data_as(dp), q0.ctypes.data_as(dp), None, None, 8, None, 1.0, p, p, p, None) == -1
    assert lib.b2k_jtraj(1, 6, q0.ctypes.data_as(dp), q0.ctypes.data_as(dp), None, None, 0, None, 1.0, None, None, None, None) == 0
    assert lib.b2k_hessian(1, 7, None, 4, None, None) == -1
    # fkine_all's single-walk entry point: frame table validation happens before anything touches the device
    ip = rtb._lib.ip
    panda_ets = rtb.models.Panda().ets()  # owns the handle: keep it alive
    hc = panda_ets._chain
    aft, slt, tl = np.array([0, 3, 2], np.int32), np.array([1, 2, 3], np.int32), np.tile(np.eye(4), (3, 1, 1))
    a_ = lambda x: x.ctypes.data_as(ip)  # noqa: E731
    p32 = (p + 31) & ~31
    assert lib.b2k_fkine_frames(None, 1, p, 4, 7, None, 3, a_(aft), a_(slt), tl.ctypes.data_as(dp), p32, 4, None) == -1
    assert lib.b2k_fkine_frames(hc, 1, p, 4, 7, None, 3, a_(aft), a_(slt), tl.ctypes.data_as(dp), p32, 4, None) == -1
    assert b"ascending" in lib.b2k_last_error()
    aft[:] = [0, 2, 7]
    assert lib.b2k_fkine_frames(hc, 1, p, 4, 7, None, 3, a_(aft), a_(slt), tl.ctypes.data_as(dp), p32, 4, None) == -1
    aft[:] = [-1, 2, 6]; slt[2] = 4
    assert lib.b2k_fkine_frames(hc, 1, p, 4, 7, None, 3, a_(aft), a_(slt), tl.ctypes.data_as(dp), p32, 4, None) == -1
    assert b"slot" in lib.b2k_last_error()
    slt[2] = 3
    assert lib.b2k_fkine_frames(hc, 1, p, 4, 7, None, 3, a_(aft), a_(slt), tl.ctypes.data_as(dp), p32 + 8, 4, None) == -1
    assert b"32-byte" in lib.b2k_last_error()
    assert lib.b2k_fkine_frames(hc, 1, p, 0, 7, None, 3, a_(aft), a_(slt), tl.ctypes.data_as(dp), p32, 4, None) == 0
    assert lib.b2k_manipulability(1, 7, p, 4, 0, p, None) == -1 and b"axis" in lib.b2k_last_error()
    assert lib.b2k_jacobm(1, 7, p, 4, 0, p, None) == -1
    assert lib.b2k_jacob_dot(3, 7, p, p, 4, p, None) == -1
    assert lib.b2k_angle_axis(1, p, p, 4, 5, p, None) == -1 and b"tep_stride" in lib.b2k_last_error()
    assert lib.b2k_p_servo(1, p, p, 4, 16, None, 0.1, p, None, None) == -1 and b"arrived" in lib.b2k_last_error()
    # IK: unknown method code, negative damping for the pseudo-inverse solvers
    d = ch.panda_ets()
    h = C.c_void_p()
    ip = rtb._lib.ip
    assert lib.b2k_chain_create(len(d["isjoint"]), d["isjoint"].ctypes.data_as(ip), d["axis"].ctypes.data_as(ip),
                                d["flip"].ctypes.data_as(ip), d["jindex"].ctypes.data_as(ip),
                                np.ascontiguousarray(d["T"]).ctypes.data_as(dp), np.ascontiguousarray(d["qlim"]).ctypes.data_as(dp),
                                C.byref(h)) == 0
    ik = lambda lam, meth: lib.b2k_ik_lm(h, 1, p, 2, None, 30, 100, 1e-6, 0, None, lam, meth, 0, 0, 1, p, p, p, p, p, None)  # noqa: E731
    assert ik(1.0, 5) == -1 and b"method" in lib.b2k_last_error()
    assert ik(-0.5, rtb._lib.IK_NR) == -1 and b"damping" in lib.b2k_last_error()
    assert lib.b2k_chain_destroy(h) == 0


IK_PANDA = rtb.models.Panda().ets()  # kept alive: the table below passes its chain handle
IK_SHARED = rtb.ET.Rz(jindex=0) * rtb.ET.tx(0.3) * rtb.ET.Ry(jindex=0)  # two joints read q[0]


def _ik_lm_call(chain=None, dtype=1, N=4, ilimit=30, slimit=100, method=0, semantics=0, lam=1.0, Tep=8, q_out=8,
                succ=8, its=8, srch=8, res=8):
    lib = rtb._lib.lib()
    chain = IK_PANDA._chain if chain is None else chain
    rc = lib.b2k_ik_lm(chain, dtype, Tep, N, None, ilimit, slimit, 1e-6, 1, None, lam, method, 0, semantics, 1, q_out,
                       succ, its, srch, res, None)
    return rc, lib.b2k_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(chain=0), "chain handle is NULL"),
    (dict(dtype=2), "dtype must be"),
    (dict(N=-1), "N is negative"),
    (dict(chain=IK_SHARED._chain), "share a jindex"),
    (dict(ilimit=0), "ilimit and slimit"),
    (dict(slimit=0), "ilimit and slimit"),
    (dict(method=-1), "bad method -1"),
    (dict(method=5), "bad method 5"),
    (dict(semantics=2), "bad semantics 2"),
    (dict(Tep=None), "Tep is NULL"),
    (dict(q_out=None), "q_out is NULL"),
    (dict(succ=None), "success is NULL"),
    (dict(its=None), "iterations is NULL"),
    (dict(srch=None), "searches is NULL"),
    (dict(res=None), "residual is NULL"),
    (dict(method=rtb._lib.IK_NR, lam=-0.5), "pinv_damping is negative"),
    (dict(method=rtb._lib.IK_GN, lam=-0.5), "pinv_damping is negative"),
    (dict(N=-1, dtype=2), "dtype must be"),  # the checks run in the order above
    (dict(method=5, res=None), "bad method"),
    (dict(res=None, method=rtb._lib.IK_NR, lam=-0.5), "residual is NULL"),
    (dict(N=0), None),
    (dict(N=0, Tep=None, q_out=None, succ=None, its=None, srch=None, res=None), None),
    (dict(N=0, method=2, semantics=1, lam=-1.0), None),  # the LM damping rules take any lambda
])
def test_ik_lm_rejects_bad_arguments_before_launching(kw, msg):
    rc, err = _ik_lm_call(**kw)
    if msg is None:
        assert rc == 0, err
        return
    assert rc == -1
    assert msg in err, err


# ------------------------------------------------------------------ host-side mirror of the reference interface
def test_models_match_the_reference_tables():
    """Product model tables == the independent restatement used to generate the goldens."""
    for rob, want in ((rtb.models.Panda(), ch.panda_ets()), (rtb.models.UR10(), ch.dh_to_ets(ch.ur10_links())),
                      (rtb.models.Puma560(), ch.dh_to_ets(ch.puma560_links())),
                      (rtb.models.PandaMDH(), ch.dh_to_ets(ch.panda_mdh_links(), mdh=True, tool=ch.panda_mdh_tool()))):
        d = rob.ets().describe()
        for k in ("isjoint", "axis", "flip", "jindex", "T"):
            assert np.array_equal(d[k], want[k]), (rob.name, k)
        sel = d["isjoint"].astype(bool)
        assert np.array_equal(d["qlim"][sel], want["qlim"][sel])
    assert np.array_equal(rtb.models.Puma560()._pack_rne(), ch.pack_rne(ch.puma560_links()))
    assert np.array_equal(rtb.models.PandaMDH()._pack_rne(), ch.pack_rne(ch.panda_mdh_links()))
    assert np.array_equal(rtb.models.UR10()._pack_rne(), ch.pack_rne(ch.ur10_links()))
    assert rtb.models.Panda().ets().m == 22 and rtb.models.UR10().ets().m == 15  # SURVEY 8a


def test_ets_composition_and_jindex_numbering():
    ET = rtb.ET
    e = ET.tz(0.333) * ET.Rz() * ET.Rx(-90, "deg") * ET.Rz() * ET.tx(0.1) * ET.tz()
    assert (e.n, e.m) == (3, 6) and list(e.jindices) == [0, 1, 2] and e.structure == "RRP"
    # explicit jindices are kept (reference tests/test_ETS.py:267-293 builds Panda this way)
    l0 = ET.tz(0.333) * ET.Rz(jindex=0)
    l1 = ET.Rx(-1.57) * ET.Rz(jindex=1)
    r = l0 + l1
    assert list(r.jindices) == [0, 1]
    with pytest.raises(ValueError):
        rtb.ETS([ET.Rz(jindex=0), ET.Rz()  , ET.Rz()])  # some-but-not-all jindices (ETS.py:830-834)
    # qlim defaults the reference hands its C layer (ET.py:109-115)
    np.testing.assert_allclose(e.qlim, np.array([[-np.pi, -np.pi, 0.0], [np.pi, np.pi, 1.0]]))
    # compile() folds constants (ETS.py:857-906)
    c = rtb.models.Panda().ets().compile()
    assert c.n == 7 and c.m == 15
    # flip and deg units
    f = ET.Ry(flip=True)
    np.testing.assert_allclose(f.A(0.3), ch.troty(-0.3))
    np.testing.assert_allclose(ET.Rx(90, "deg").A(), ch.trotx(np.deg2rad(90.0)))
    with pytest.raises(TypeError):
        ET.Rx("theta")  # symbolic values have no GPU path (reference raises TypeError("Symbolic value"))


def test_robot_sub_chain_ets():
    """Robot.ets(start, end) for a serial robot (reference BaseRobot.ets 1554-1652): link ranges, names, jindex kept."""
    panda = rtb.models.Panda()
    L = panda.links
    assert panda.ets() is panda.ets()
    head, tail = panda.ets(end=L[3]), panda.ets(start=L[4], end=L[-1])
    assert len(head) + len(tail) == len(panda.ets()) and head.n == 4 and tail.n == 3
    assert [et.jindex for et in tail if et.isjoint] == [4, 5, 6]
    assert panda.ets(end=L[3].name).n == 4 and panda.ets(start=L[2], end=L[2]).n == L[2].ets.n
    with pytest.raises(ValueError):
        panda.ets(end="nope")
    with pytest.raises(TypeError):
        panda.ets(end=3.5)
    # towards the base: the inverse of the forward range, ET by ET (reference ETS.inv 545-576, ET.inv 506-539);
    # checked with the CPU oracle, which evaluates any chain description
    from oracle import oracle as orc

    q = np.random.default_rng(0).uniform(-2, 2, (5, 7))
    fwd, back = panda.ets(start=L[3], end=L[6]), panda.ets(start=L[6], end=L[2])
    assert [(e.jindex, e.isflip) for e in back if e.isjoint] == [(6, True), (5, True), (4, True), (3, True)]
    prod = orc.Chain(fwd.describe()).fkine(q) @ orc.Chain(back.describe()).fkine(q)
    np.testing.assert_allclose(prod, np.broadcast_to(np.eye(4), prod.shape), atol=1e-14)
    e = rtb.ET.Rz(jindex=2) * rtb.ET.tx(1) * rtb.ET.Rx(jindex=3, flip=True) * rtb.ET.tx(1)
    prod = orc.Chain(e.describe()).fkine(q[:, :4]) @ orc.Chain(e.inv().describe()).fkine(q[:, :4])
    np.testing.assert_allclose(prod, np.broadcast_to(np.eye(4), prod.shape), atol=1e-14)
    assert rtb.ET.tx(0.3).inv().eta == -0.3 and rtb.ET.Rz(jindex=1).inv().isflip


def test_dh_link_expansion_matches_reference_rule():
    for kw in (dict(d=0.2, a=0.3, alpha=0.4, offset=0.5), dict(d=0.0, a=0.0, alpha=0.0), dict(d=0.1, a=0, alpha=-1.0, flip=True)):
        for cls, mdh, sigma in ((rtb.RevoluteDH, False, 0), (rtb.RevoluteMDH, True, 0)):
            link = cls(**kw)
            b = ch.Builder()
            ch.dh_link_to_ets(b, sigma, 0.0, kw.get("d", 0), kw.get("alpha", 0), kw.get("a", 0), kw.get("offset", 0),
                              kw.get("flip", False), mdh)
            want = b.desc()
            got = link.ets.describe()
            for k in ("isjoint", "axis", "flip", "T"):
                assert np.array_equal(got[k], want[k])
    p = rtb.PrismaticDH(theta=0.3, a=0.1, alpha=0.2, offset=0.05)
    assert p.ets.structure == "P" and p.isprismatic


def test_rne_packing_and_dirty_tracking():
    puma = rtb.models.Puma560()
    L = puma._pack_rne()
    assert L.shape == (144,)
    np.testing.assert_allclose(L[24 + 10:24 + 19].reshape(3, 3), np.diag([0.13, 0.524, 0.539]))  # Link.py:733-742
    assert not puma._dynchanged
    puma.links[1].m = 20.0  # @_listen_dyn -> robot.dynchanged() (Link.py:26-59)
    assert puma._dynchanged and puma._pack_rne()[24 + 6] == 20.0
    puma.links[2].Tc = 0.3  # scalar Coulomb -> symmetric pair (Link.py:850-856)
    np.testing.assert_allclose(puma.links[2].Tc, [0.3, -0.3])
    with pytest.raises(ValueError):
        puma.links[0].I = np.array([[1, 2, 0], [0, 1, 0], [0, 0, 1.0]])  # not symmetric
    with pytest.raises(ValueError):
        rtb.DHRobot([rtb.RevoluteDH(), rtb.RevoluteMDH()])  # mixed conventions


def test_ik_solution_protocol():
    s = rtb.IKSolution(q=np.zeros(3), success=True, iterations=4, searches=1, residual=1e-9, reason="Success")
    q, ok, it, sr, res, why = s
    assert ok and it == 4 and "success=True" in str(s)
    assert rtb.IK_LM(method="sugi", k=0.1).method == "sugihara" and rtb.IK_LM(method="wamp").method == "wampler"


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under the product package may reference it."""
    for dirpath, _, files in os.walk(PKG):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")) or f == "Makefile":
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(from|import)\s+oracle", txt, flags=re.M), f
                assert "liboracle" not in txt and "oracle_kin" not in txt.replace("oracle/oracle_kin.c", ""), f
    src = open(os.path.join(ROOT, "b2kin.py")).read()
    assert "oracle" not in src


def test_fails_loudly_without_a_device_or_library():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    e = rtb.models.Panda().ets()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        e.eval(np.zeros(7))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        rtb.models.Puma560().rne(np.zeros(6), np.zeros(6), np.zeros(6))
    # a missing library is an ImportError with build instructions, never a silent fallback
    code = ("import sys; sys.path.insert(0, %r); import importlib; m = importlib.import_module('robotics-toolbox-python_b200._lib');"
            "m.LIB_PATH = '/nonexistent/libb2kin.so'\ntry:\n    m.lib()\nexcept ImportError as e:\n    print('IMPORTERROR', 'no CPU fallback' in str(e).lower() or 'There is no CPU fallback' in str(e))" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert "IMPORTERROR True" in out.stdout, out.stdout + out.stderr


def test_shape_errors_before_any_launch():
    puma = rtb.models.Puma560()
    try:
        import torch
        has = torch.cuda.is_available()
    except Exception:
        has = False
    if not has:
        with pytest.raises((ValueError, RuntimeError)):
            puma.rne(np.zeros((4, 6)), np.zeros((4, 5)), np.zeros((4, 6)))
    with pytest.raises(TypeError):
        puma.rne("q", np.zeros(6), np.zeros(6))
    with pytest.raises(ValueError):
        rtb.models.Panda().ets()._qbatch(np.zeros((3, 3, 3)))
    q2, single = rtb.models.Panda().ets()._qbatch(np.zeros((7, 1)))
    assert single and q2.shape == (1, 7)
    e1 = rtb.ETS([rtb.ET.Rz()])
    q2, single = e1._qbatch(np.zeros((5, 1)))  # 1-joint chain: (N,1) is a batch (documented deviation)
    assert not single and q2.shape == (5, 1)


# ------------------------------------------------------------------ row sharding (multi-GPU host logic)
def test_shard_bounds_cover_and_balance():
    for n in (0, 1, 7, 8, 1_000_000, 8_388_608, 1_000_003):
        for ws in (1, 2, 3, 8):
            spans = [rtb.dist.shard_bounds(n, ws, r) for r in range(ws)]
            assert spans[0][0] == 0 and spans[-1][1] == n
            assert all(spans[i][1] == spans[i + 1][0] for i in range(ws - 1))
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1 and sizes == rtb.dist.shard_sizes(n, ws)
    with pytest.raises(ValueError):
        rtb.dist.shard_bounds(10, 2, 2)


_WORKER = r"""
import os, sys
sys.path.insert(0, {root!r})
import numpy as np, torch, torch.distributed as td
import b2kin as rtb
td.init_process_group("gloo", rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
rank, ws = td.get_rank(), td.get_world_size()
for n_rows in (10, 11):          # even and ragged shards
    full = torch.arange(n_rows * 6, dtype=torch.float64).reshape(n_rows, 2, 3)
    lo, hi = rtb.dist.shard_bounds(n_rows, ws, rank)
    out = rtb.dist.gather_rows(full[lo:hi].clone(), n_rows)
    assert torch.equal(out, full), (rank, n_rows)
    root = rtb.dist.gather_rows(full[lo:hi].clone(), n_rows, dst=0)
    assert (root is None) == (rank != 0)
    if rank == 0:
        assert torch.equal(root, full)
# max-over-ranks timing reduction used by bench.py
t = torch.tensor([1.0 + rank], dtype=torch.float64)
td.all_reduce(t, op=td.ReduceOp.MAX)
assert t.item() == float(ws)
td.barrier()
td.destroy_process_group()
print("RANK_OK", rank)
"""


def test_gather_rows_world_size_2_gloo(tmp_path):
    """The N>1 path on CPU: two processes, gloo, 127.0.0.1 rendezvous."""
    script = tmp_path / "worker.py"
    script.write_text(_WORKER.format(root=ROOT))
    port = 29500 + (os.getpid() % 2000)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=240)
        except subprocess.TimeoutExpired:
            p.kill()
            o, _ = p.communicate()
        outs.append(o)
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"RANK_OK {r}" in o, o


def test_plain_c_program_links_and_fails_loudly_without_a_gpu(tmp_path):
    """examples/cabi_host.c needs nothing but include/b2kin.h and libb2kin.so (no Python, torch or CUDA headers);
    on a box without a CUDA device the library call must return an error code and a message, not fall back."""
    import shutil
    import subprocess

    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    libdir = os.path.join(ROOT, "robotics-toolbox-python_b200", "lib")
    exe = str(tmp_path / "cabi_host")
    subprocess.run(["gcc", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "cabi_host.c"),
                    "-L", libdir, "-lb2kin", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe], check=True)
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    r = subprocess.run([exe, "4"], capture_output=True, text=True)
    if has_gpu:
        assert r.returncode == 0 and len(r.stdout.strip().splitlines()) == 4
    else:
        assert r.returncode == 2 and "CUDA error" in r.stderr and r.stdout == ""


def test_dh_kinematic_setters_invalidate_the_chain_and_the_rne_table():
    """Changing a DH parameter after construction must rebuild the link's ETs, drop the robot's cached ETS
    (whose compiled chain handle goes with it) and mark the packed RNE table dirty -- the reference's
    @_listen_dyn on theta / d / a / alpha / sigma / mdh / offset (DHLink.py:448-563)."""
    r = rtb.models.Puma560()
    e0 = r.ets()
    d0 = e0.describe()
    assert r.ets() is e0  # cached
    r._dynchanged = False
    r.links[2].d = 0.2
    assert r._ets_cache is None and r._dynchanged
    e1 = r.ets()
    assert e1 is not e0
    T0 = np.asarray(d0["T"]).reshape(-1, 4, 4)
    T1 = np.asarray(e1.describe()["T"]).reshape(-1, 4, 4)
    assert T0.shape == T1.shape and not np.array_equal(T0, T1)
    assert np.isclose(T1[:, 2, 3], 0.2).any() and not np.isclose(T0[:, 2, 3], 0.2).any()
    assert r._pack_rne()[24 * 2 + 3] == 0.2
    # a parameter going to zero drops its elementary transform (DHLink._to_ets omits zero terms)
    m_before = len(np.asarray(r.ets().describe()["isjoint"]))
    r.links[2].a = 0.0
    assert len(np.asarray(r.ets().describe()["isjoint"])) == m_before - 1
    # qlim feeds the joint ET
    r.links[0].qlim = [-1.0, 1.0]
    assert np.allclose(r.qlim[:, 0], [-1.0, 1.0])
    ql = np.asarray(r.ets().describe()["qlim"]).reshape(-1, 2)
    assert (np.isclose(ql[:, 0], -1.0) & np.isclose(ql[:, 1], 1.0)).any()
    # links that are not attached to a robot simply rebuild their own ETS
    l = rtb.RevoluteDH(d=0.1, a=0.2, alpha=0.3)
    n0 = len(l.ets)
    l.alpha = 0.0
    assert len(l.ets) == n0 - 1


def test_numa_helpers_are_safe_without_a_gpu():
    assert rtb.dist._parse_cpulist("0-2,5,7-8\n") == {0, 1, 2, 5, 7, 8}
    assert rtb.dist.bind_to_gpu_numa(0) in (None,) or isinstance(rtb.dist.bind_to_gpu_numa(0), dict)


def test_ik_kernels_keep_the_normal_equations_in_registers():
    """Guards the round-2 finding (DESIGN 3.5): `#pragma unroll` once left two columns of the Cholesky as run-time loops,
    which put the whole packed matrix in local memory (144 B stack frame, 22 LDL + 14 STL per evaluation, no spill
    warning).  The resource table of the shipped fp32 Panda / UR10 / Puma kernels must show no stack frame and at most
    128 registers (4 resident blocks); the fp64 ones are held to 168 registers (3 blocks)."""
    import shutil

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", rtb._lib.LIB_PATH], capture_output=True, text=True).stdout
    usage = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+?):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and name:
            usage[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    seen = 0
    for fn, (reg, stack) in usage.items():
        m = re.match(r"_Z(?:7k_ik_lm|13k_ik_restarts)I([fd])Li([67])ELi1E", fn)  # DH-like profile, n = 6 / 7 (LM and NR / GN)
        if not m:
            continue
        seen += 1
        if m.group(1) == "f":
            assert reg <= 128 and stack == 0, (fn, reg, stack)
        else:
            assert reg <= 168, (fn, reg, stack)
    assert seen >= 24, f"only {seen} IK kernels recognised in the resource table"
