"""CPU checks of tests/fkj_ref.py and of the argument checks of the fkj entry points (no GPU needed):

* the long-double reference against the compiled CPU oracle on every chain family at n = 1..10, with and without
  base and tool;
* each family builder produces the kernel classification it claims, under the restated b2k_chain_create rules;
* b2k_fkine_jacobe rejects what the other four fkj entry points reject, and the output alignment the kernels need is
  checked before any CUDA call.
"""
import ctypes as C

import numpy as np
import pytest

import b2kin as rtb
from oracle import chains as ch
from oracle import oracle as orc

import fkj_ref as R  # noqa: E402

BASE = ch.trotz(0.4) @ ch.troty(-0.3) @ ch.transl(0.2, -0.1, 0.5)
TOOL = ch.trotx(0.7) @ ch.transl(0.05, 0.1, 0.2)


def families(n, rng):
    """(name, description, dh_like, dense) of every family at joint count n."""
    out = [(f"dh-{tail}", R.dh_family(n, rng, tail), True, True) for tail in ("ident", "trans", "gen")]
    out.append(("dh-offset0", R.near_dh_family(n, 0, "offset", rng), True, True))  # an offset on link 0 stays in A_0
    for k in range(n):
        out.append((f"flip@{k}", R.near_dh_family(n, k, "flip", rng), False, True))
    for k in range(1, n):
        for br in ("ry", "rz", "gen", "offset"):
            out.append((f"{br}@{k}", R.near_dh_family(n, k, br, rng), False, True))
    out.append(("generic", R.generic_family(n, rng, list(R.ALL_KINDS)), False, True))
    perm = rng.permutation(n + 3)[:n]
    out.append(("dh-jindex", R.with_jindex(R.dh_family(n, rng), perm), True, bool(np.array_equal(perm, np.arange(n)))))
    return out


@pytest.mark.parametrize("n", range(1, 11))
def test_reference_matches_oracle(n):
    rng = np.random.default_rng(100 + n)
    for name, desc, _, _ in families(n, rng):
        Co = orc.Chain(desc)
        w = int(desc["jindex"][desc["isjoint"].astype(bool)].max()) + 1
        Q = rng.uniform(-3, 3, (24, w))
        for base, tool in ((None, None), (BASE, TOOL)):
            ref = R.evaluate(desc, Q, base, tool)
            for got, want in ((ref["T"], Co.fkine(Q, base, tool)), (ref["J0"], Co.jacob0(Q, tool)),
                              (ref["Je"], Co.jacobe(Q, tool))):
                got = got.astype(np.float64)
                scale = max(1.0, float(np.abs(want).max()))
                assert np.abs(got - want).max() <= 1e-13 * scale, (name, n, base is None)
            assert np.array_equal(ref["T"][:, 3], np.broadcast_to([0, 0, 0, 1], (24, 4)))


@pytest.mark.parametrize("n", range(1, 11))
def test_family_classification(n):
    rng = np.random.default_rng(200 + n)
    for name, desc, dh, dense in families(n, rng):
        c = R.compile_chain(desc)
        assert c["n"] == n, name
        assert c["dh_like"] == dh and c["dense_jindex"] == dense, (name, c["dh_like"], c["dense_jindex"])


def test_generic_family_covers_every_constant_class():
    """Across the n = 1..10 sweep the constants ahead of joints 1..n-1 (the ones both walks multiply as constants)
    take every AK_* class with every combination of translation bits."""
    rng = np.random.default_rng(3)
    kinds, seen = list(R.ALL_KINDS), set()
    for n in range(1, 11):
        c = R.compile_chain(R.generic_family(n, rng, kinds))
        seen |= {R.classify34(c["A"][k]) for k in range(1, n)}
    assert seen >= set(R.ALL_KINDS)


def test_classify34_restatement():
    for M, want in ((np.eye(4), R.AK_IDENT), (ch.transl(1, 0, 0), R.AK_TX), (ch.transl(0, 2, 3), R.AK_TY | R.AK_TZ),
                    (ch.trotx(0.3), R.AK_RX), (ch.troty(0.3), R.AK_RY), (ch.trotz(0.3), R.AK_RZ),
                    (ch.trotx(np.pi / 2) @ ch.transl(0, 0, 1), R.AK_RX | R.AK_TY | R.AK_TZ),
                    (ch.trotx(0.3) @ ch.troty(0.2), R.AK_GEN)):
        assert R.classify34(M[:3]) == want
    # every model the project ships takes the DH-like profile
    for rob in (rtb.models.Panda(), rtb.models.PandaMDH(), rtb.models.Puma560(), rtb.models.UR10()):
        assert R.compile_chain(rob.ets().describe())["dh_like"], rob.name


def test_sincos_path_rule():
    x = np.array([[0.5, -7.99], [8.0, 1.0], [1e3, 105614.0], [105615.0, 1.0], [np.nan, 0.0], [np.inf, 0.0]])
    p32, a = R.sincos_path(x, np.float32, True)
    assert list(p32) == [R.PATH_MUFU, R.PATH_POLY, R.PATH_POLY, R.PATH_SLOW, R.PATH_SLOW, R.PATH_SLOW]
    assert list(R.sincos_path(x, np.float64, True)[0]) == [R.PATH_POLY] * 3 + [R.PATH_SLOW] * 3
    assert list(R.sincos_path(x, np.float32, False)[0]) == [R.PATH_POLY] * 3 + [R.PATH_SLOW] * 3
    assert a[0] == 7.99 and np.isinf(a[4])


def test_lean_rule():
    c = R.compile_chain(R.dh_family(7, np.random.default_rng(0)))
    assert R.expected_launches(c, 7, 256, 64) == 1 and R.expected_launches(c, 7, 256, 65) == 2
    assert R.expected_launches(c, 8, 256, 65) == 1  # ldq != n
    assert R.expected_launches(c, 7, 264, 65) == 1  # q not 16-byte aligned
    assert R.expected_launches(c, 7, 256, 31) == 1 and R.expected_launches(c, 7, 256, 65, variant=4) == 1


# ------------------------------------------------------------------ argument checks of the C ABI
def _handle(desc):
    lib = rtb._lib.lib()
    ip, dp = rtb._lib.ip, rtb._lib.dp
    h = C.c_void_p()
    T = np.ascontiguousarray(desc["T"], dtype=np.float64)
    ql = np.ascontiguousarray(desc["qlim"], dtype=np.float64)
    assert lib.b2k_chain_create(len(desc["isjoint"]), desc["isjoint"].ctypes.data_as(ip), desc["axis"].ctypes.data_as(ip),
                                desc["flip"].ctypes.data_as(ip), desc["jindex"].ctypes.data_as(ip), T.ctypes.data_as(dp),
                                ql.ctypes.data_as(dp), C.byref(h)) == 0
    return h


def _calls(lib, h, dt, q, N, ldq, base, tool, T, J):
    """The five fkj entry points with one argument set; the ones that take no base / T ignore those."""
    return {
        "b2k_fkine": lambda: lib.b2k_fkine(h, dt, q, N, ldq, base, tool, T, None),
        "b2k_jacob0": lambda: lib.b2k_jacob0(h, dt, q, N, ldq, tool, J, None),
        "b2k_jacobe": lambda: lib.b2k_jacobe(h, dt, q, N, ldq, tool, J, None),
        "b2k_fkine_jacob0": lambda: lib.b2k_fkine_jacob0(h, dt, q, N, ldq, base, tool, T, J, None),
        "b2k_fkine_jacobe": lambda: lib.b2k_fkine_jacobe(h, dt, q, N, ldq, base, tool, T, J, None),
    }


def test_fkine_jacobe_rejects_what_the_other_entry_points_reject():
    lib = rtb._lib.lib()
    dp = rtb._lib.dp
    h = _handle(ch.panda_ets())
    buf = np.zeros(1024)  # stands in for (never dereferenced) device arrays
    p = (buf.ctypes.data + 255) & ~255
    bad = np.eye(4); bad[3, 0] = 1.0
    eye = np.eye(4)
    cases = [  # (argument overrides, words of the message, which entry points take the argument)
        (dict(h=None), b"NULL", ""),
        (dict(dt=2), b"dtype", ""),
        (dict(N=-1), b"negative", ""),
        (dict(q=None), b"q is NULL", ""),
        (dict(ldq=6), b"row width", ""),
        (dict(ldq=17), b"row width", ""),
        (dict(q=p + 4), b"aligned", ""),
        (dict(tool=bad.ctypes.data_as(dp)), b"tool", ""),
        (dict(T=None), b"T is NULL", "fkine"),
        (dict(base=bad.ctypes.data_as(dp)), b"base", "fkine"),
        (dict(J=None), b"J is NULL", "jacob"),
    ]
    try:
        for over, word, takers in cases:
            args = dict(h=h, dt=1, q=p, N=4, ldq=7, base=eye.ctypes.data_as(dp), tool=eye.ctypes.data_as(dp), T=p, J=p)
            args.update(over)
            for name, call in _calls(lib, **args).items():
                if takers in name:
                    assert call() == -1, (name, over)
                    assert word in lib.b2k_last_error(), (name, over, lib.b2k_last_error())
    finally:
        lib.b2k_chain_destroy(h)


@pytest.mark.parametrize("n", [3, 6, 7])
def test_output_alignment_is_checked_before_any_cuda_call(n):
    """T must be 32-byte aligned and J aligned to the Jacobian stage's copy unit (16 bytes in fp64 and for even n,
    8 bytes for fp32 odd n).  The check comes before the device lookup, so it gives the same status and message on a
    machine without a GPU, where any CUDA call would fail."""
    lib = rtb._lib.lib()
    h = _handle(R.dh_family(n, np.random.default_rng(n)))
    buf = np.zeros(4096)
    p = (buf.ctypes.data + 255) & ~255
    try:
        for dt, es in ((1, 8), (0, 4)):
            jub = 16 if (6 * n * es) % 16 == 0 else 8
            for name, call in _calls(lib, h, dt, p, 4, n, None, None, p + 8, p).items():  # T 8 mod 32
                if "fkine" in name:
                    assert call() == -1, name
                    assert b"T must be 32-byte aligned" in lib.b2k_last_error(), (name, lib.b2k_last_error())
            for name, call in _calls(lib, h, dt, p, 4, n, None, None, p, p + 8).items():  # J 8 mod 16
                if "jacob" in name and jub == 16:
                    assert call() == -1, name
                    assert b"J must be 16-byte aligned" in lib.b2k_last_error(), (name, lib.b2k_last_error())
            for name, call in _calls(lib, h, dt, p, 4, n, None, None, p + 16, p + 4).items():  # T 16 mod 32, J 4 mod 8
                assert call() == -1, name
                err = lib.b2k_last_error()
                assert b"T must be 32-byte aligned" in err if "fkine" in name else b"J must be %d-byte aligned" % jub in err
    finally:
        lib.b2k_chain_destroy(h)
