"""rne and the five dynamics fan-outs (inertia, gravload, itorque, coriolis, accel) on the GPU against the long-double
reference of tests/dyn_ref.py, entry by entry within its error bar, on both kernel paths:

  spec     B2K_RNE_SPEC=2: the robot-specialised kernel (generated per robot, compiled with NVRTC at first use) serves
           the full 32-row tiles and must not fall back; the generic kernel serves the ragged tail;
  generic  B2K_RNE_SPEC=0: the pre-compiled generic kernels serve every row;
  default  B2K_RNE_SPEC unset: the library's own split.

Calls go through the C ABI into NaN-filled outputs framed by guard elements; each checks every entry against its bar,
that no NaN is left and the guards are untouched, and the launch count that proves which kernel ran.  Batch sizes cover
one row, one warp tile, tile edges, the 8-tile block of the fp32 two-tiles-per-warp kernels (256 rows) and its
neighbours.  Inputs hold exact zeros, -0.0 and subnormal joint rates (the Coulomb switch), angles up to 1e6 (the slow
sincos path), and alternate gravity pattern and tip wrench on one robot handle, so a stale specialised program would
be caught.  fp32 kernels are compared with the reference evaluated on the fp32-rounded inputs.

The worst error / bar ratio of every (dtype, path, op) is printed at the end of the module (pytest -s).
Each (robot, operation, dtype, gravity pattern, tip wrench) the specialised path serves is one NVRTC compile; the
number of compiles and their mean time on the machine at hand are printed too.  Measured on an H100 80GB HBM3 host:
144 compiles took 71 s (0.5 s each; up to 2.6 s for the 10-joint inertia and accel), but the 10-joint Coriolis
program (55 recursions unrolled) took 273 s alone, so the 20 003-row 10-joint Coriolis batch runs on the generic
kernel and the specialised Coriolis kernel is exercised up to 7 joints.  The module then runs in about 100 s.
"""
import ctypes as C
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import dyn_ref as D  # noqa: E402
from oracle import chains as ch  # noqa: E402

NS = (1, 31, 32, 33, 63, 64, 65, 255, 256, 257)
GRAVS = (np.zeros(3), np.array([0.0, 0.0, 9.81]), np.array([1.5, -2.0, 9.81]))  # base acceleration = -gravity
FEXT = np.array([3.0, -1.0, 2.0, 0.4, -0.3, 0.2])
PATHS = {"spec": "2", "generic": "0", "default": "1"}
GUARD = 16
WORST = {}
COMPILES = {"keys": set(), "seconds": 0.0}
DT = {np.float64: 1, np.float32: 0}


@pytest.fixture(scope="module", autouse=True)
def report():
    t0 = time.time()
    yield
    print("\nworst error / bar ratio per (dtype, path, op):")
    for k in sorted(WORST, key=str):
        print(f"  {k[0]:8s} {k[1]:8s} {k[2]:9s} {WORST[k]:.3g}")
    n = len(COMPILES["keys"])
    print(f"specialised programs compiled: {n}, first-call time {COMPILES['seconds']:.1f} s in all"
          f" ({COMPILES['seconds'] / max(n, 1):.2f} s each); module {time.time() - t0:.1f} s")


_HANDLES = {}


def handle(L, mdh):
    key = (np.asarray(L).tobytes(), mdh)
    if key not in _HANDLES:
        h = rtb._lib.vp()
        Lc = np.ascontiguousarray(L, dtype=np.float64)
        rtb._lib.check(rtb._lib.lib().b2k_rne_create(len(Lc) // 24, mdh, rtb._lib.dptr(Lc), C.byref(h)))
        _HANDLES[key] = h
    return _HANDLES[key]


def out_rows(op, n):
    return n * n if op in ("inertia", "coriolis") else n


def launch(op, h, n, dt, ins, N, grav, fext):
    """Runs one C ABI call into a NaN-filled output framed by guards; returns (output (N, ...) on the host, launches)."""
    lib = rtb._lib.lib()
    R = out_rows(op, n)
    buf = torch.full((N * R + 2 * GUARD,), float("nan"), dtype=torch.float64 if dt == np.float64 else torch.float32, device="cuda")
    buf[:GUARD] = 7.0
    buf[GUARD + N * R:] = 7.0
    out = buf[GUARD:GUARD + N * R]
    p = [x.data_ptr() for x in ins]
    g = rtb._lib.dptr(np.ascontiguousarray(grav, dtype=np.float64))
    fx = rtb._lib.dptr(np.ascontiguousarray(fext, dtype=np.float64)) if fext is not None else None
    c = DT[dt]
    n0 = rtb.launch_count()
    if op == "rne":
        rc = lib.b2k_rne(h, c, p[0], p[1], p[2], N, g, fx, out.data_ptr(), None)
    elif op == "inertia":
        rc = lib.b2k_rne_inertia(h, c, p[0], N, out.data_ptr(), None)
    elif op == "gravload":
        rc = lib.b2k_rne_gravload(h, c, p[0], N, g, out.data_ptr(), None)
    elif op == "itorque":
        rc = lib.b2k_rne_itorque(h, c, p[0], p[1], N, out.data_ptr(), None)
    elif op == "coriolis":
        rc = lib.b2k_rne_coriolis(h, c, p[0], p[1], N, out.data_ptr(), None)
    else:
        rc = lib.b2k_rne_accel(h, c, p[0], p[1], p[2], N, g, out.data_ptr(), None)
    rtb._lib.check(rc)
    torch.cuda.synchronize()
    launches = rtb.launch_count() - n0
    b = buf.cpu().numpy()
    assert np.all(b[:GUARD] == 7.0) and np.all(b[GUARD + N * R:] == 7.0), f"{op}: a guard element was overwritten"
    o = b[GUARD:GUARD + N * R]
    assert not np.isnan(o).any(), f"{op}: {int(np.isnan(o).sum())} output entries never written"
    return o.reshape((N, n, n) if op in ("inertia", "coriolis") else (N, n)), launches


def op_inputs(op, q, qd, qdd, tq):
    return {"rne": (q, qd, qdd), "inertia": (q,), "gravload": (q,), "itorque": (q, qdd), "coriolis": (q, qd),
            "accel": (q, qd, tq)}[op]


def reference(op, L, mdh, grav, fext, q, qd, qdd, tq, dt):
    kw = dict(rne=dict(qd=qd, x=qdd, fext=fext), itorque=dict(x=qdd), coriolis=dict(qd=qd), accel=dict(qd=qd, x=tq)).get(op, {})
    v, bar = D.op3(op, L, mdh, grav, q, dtype=dt, **kw)
    return v.astype(np.float64), bar


def compare(key, got, want, bar, rows=None):
    """Every entry within its bar; accel rows whose bar leaves no significant digit in fp32 are counted and skipped."""
    err = np.abs(got - want)
    if rows is None:
        rows = np.ones(len(got), bool)
    ratio = np.where(bar > 0, err / np.where(bar > 0, bar, 1), np.where(err > 0, np.inf, 0))[rows]
    if ratio.size:
        WORST[key] = max(WORST.get(key, 0.0), float(ratio.max()))
    bad = np.argwhere(ratio > 1)
    assert not len(bad), f"{key}: {len(bad)} entries outside the bar, first {tuple(bad[0])}: got {got[rows][tuple(bad[0])]!r} " \
                         f"want {want[rows][tuple(bad[0])]!r} bar {bar[rows][tuple(bad[0])]:.3g}"


def accel_rows(L, mdh, q, dt):
    """Rows where the fp32 solve keeps significant digits (cond(M) u < 1e-2); every row in fp64."""
    if dt == np.float64:
        return np.ones(len(q), bool)
    M = D.op3("inertia", L, mdh, np.zeros(3), q)[0]
    return D.cond(M) * float(np.finfo(np.float32).eps) / 2 < 1e-2


def spec_declines(op, L, mdh):
    """accel of an MDH arm with a prismatic first joint: M is not symmetric there, the specialised kernel's pivot-free
    LDL^T cannot solve it, and the generator declines."""
    return op == "accel" and mdh and np.asarray(L)[4] != 0


def expected_launches(path, N, declined=False):
    if path == "generic" or N < 32 or N % 32 == 0 or declined:
        return 1
    return 2


def run_matrix(path, L, mdh, dt, ops, variants, Ns=NS, seed=0):
    """Every op at every N on one handle; variants (grav, fext) alternate from call to call."""
    n = len(L) // 24
    h = handle(L, mdh)
    q, qd, qdd, tq = D.inputs(L, max(Ns), dt, seed)
    dev = [torch.from_numpy(x).cuda() for x in (q, qd, qdd, tq)]
    for op in ops:
        vs = variants if op in ("rne", "gravload", "accel") else [(GRAVS[2], None)]
        if op != "rne":
            vs = [(g, None) for g, _ in vs]
        refs = {}
        rows_ok = accel_rows(L, mdh, q, dt) if op == "accel" else None
        skipped = 0
        for i, N in enumerate(Ns):
            grav, fext = vs[i % len(vs)]
            rk = (grav.tobytes(), fext is not None)
            if rk not in refs:
                refs[rk] = reference(op, L, mdh, grav, fext, q, qd, qdd, tq, dt)
            want, bar = refs[rk]
            key = (op, dt, int((grav != 0) @ [1, 2, 4]) if op in ("rne", "gravload", "accel") else 0, fext is not None)
            declined = spec_declines(op, L, mdh)
            ins = [x[:N] for x in op_inputs(op, *dev)]
            if declined and path == "spec" and N >= 32:
                with pytest.raises(ValueError, match="prismatic first joint"):
                    launch(op, h, n, dt, ins, N, grav, fext)
                continue
            fresh = path != "generic" and N >= 32 and not declined and (id(h), key) not in COMPILES["keys"]
            t0 = time.time()
            got, nl = launch(op, h, n, dt, ins, N, grav, fext)
            if fresh:
                COMPILES["keys"].add((id(h), key))
                COMPILES["seconds"] += time.time() - t0
            assert nl == expected_launches(path, N, declined), (op, N, nl)
            rows = rows_ok[:N] if rows_ok is not None else None
            if rows is not None:
                skipped += int((~rows).sum())
            compare((np.dtype(dt).name, path, op), got, want[:N], bar[:N], rows)
        if op == "accel" and dt == np.float32:
            assert skipped <= 0.25 * sum(Ns), f"accel fp32: {skipped} of {sum(Ns)} rows too ill-conditioned to compare"


@pytest.fixture(params=list(PATHS))
def path(request, monkeypatch):
    monkeypatch.setenv("B2K_RNE_SPEC", PATHS[request.param])
    return request.param


@pytest.mark.parametrize("n", range(1, 11))
def test_rne_and_inertia_at_every_joint_count(path, n):
    """n = 1..10, DH and MDH, the three alpha profiles, mixed revolute / prismatic (first joint prismatic) on every
    third n, friction on two thirds: rne (fext alternating zero / nonzero) and inertia, fp64 and fp32."""
    L = D.robot(n, n % 2, D.PROFILES[n % 3], n % 3 == 1, n % 3 != 0, 100 + n)
    for dt in (np.float64, np.float32):
        run_matrix(path, L, n % 2, dt, ("rne", "inertia"), [(GRAVS[2], None), (GRAVS[2], FEXT)], seed=n)


MATRIX_ROBOTS = {
    "puma560": (ch.pack_rne(ch.puma560_links()), 0),
    "mdh7_near_prismatic": (D.robot(7, 1, "near", True, True, 7), 1),
    "dh5_general_mixed": (D.robot(5, 0, "gen", True, True, 5), 0),
}


@pytest.mark.parametrize("name", list(MATRIX_ROBOTS))
def test_every_operation_gravity_pattern_and_tip_wrench(path, name):
    """The full operation x gravity pattern x fext matrix, alternated on one handle."""
    L, mdh = MATRIX_ROBOTS[name]
    variants = [(GRAVS[0], None), (GRAVS[1], FEXT), (GRAVS[2], None), (GRAVS[0], FEXT), (GRAVS[1], None), (GRAVS[2], FEXT)]
    for dt in (np.float64, np.float32):
        run_matrix(path, L, mdh, dt, D.OPS, variants, seed=11)


def sample_rows(N, k, seed):
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.arange(64), np.arange(N - 67, N), rng.integers(0, N, k)]))


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_multi_wave_batches(monkeypatch, dt):
    """200 003 Puma rows for rne, gravload and itorque in both types; 20 003 rows of a 10-joint arm for inertia,
    coriolis and accel in fp64 (default split: specialised tiles + a 3-row generic tail; coriolis on the generic kernel
    alone, see the module docstring).  Every row is checked for sentinels; the reference is evaluated on the first and
    last two tiles and 2000 (600 for the n x n operations) random rows.  The first call of each operation includes its
    NVRTC compile (printed)."""
    cases = [((ch.pack_rne(ch.puma560_links()), 0), 200_003, ("rne", "gravload", "itorque"), 2000)]
    if dt == np.float64:
        cases.append(((D.robot(10, 0, "gen", False, True, 10), 0), 20_003, ("inertia", "coriolis", "accel"), 600))
    for (L, mdh), N, ops, k in cases:
        n = len(L) // 24
        q, qd, qdd, tq = D.inputs(L, N, dt, 3)
        dev = [torch.from_numpy(x).cuda() for x in (q, qd, qdd, tq)]
        rows = sample_rows(N, k, 4)
        h = handle(L, mdh)
        for op in ops:
            if op == "coriolis":
                monkeypatch.setenv("B2K_RNE_SPEC", "0")
            else:
                monkeypatch.delenv("B2K_RNE_SPEC", raising=False)
            grav = GRAVS[2]
            fext = FEXT if op == "rne" else None
            t0 = time.time()
            got, nl = launch(op, h, n, dt, op_inputs(op, *dev), N, grav, fext)
            print(f"\n{np.dtype(dt).name} {op} n={n} N={N}: first call (compile + run) {time.time() - t0:.1f} s")
            assert nl == (1 if op == "coriolis" else 2), (op, nl)
            want, bar = reference(op, L, mdh, grav, fext, q[rows], qd[rows], qdd[rows], tq[rows], dt)
            keep = accel_rows(L, mdh, q[rows], dt) if op == "accel" else None
            if keep is not None:
                assert keep.mean() >= 0.75, f"accel: {int((~keep).sum())} of {len(keep)} rows too ill-conditioned"
            compare((np.dtype(dt).name, "default", op), got[rows], want, bar, keep)


def test_element_aligned_inputs_take_the_generic_kernel(monkeypatch):
    """q, qd, qdd one element past a 16-byte boundary (as row slices like q[1:] of an odd-width robot are): the
    specialised kernel declines the whole call, one generic launch serves it."""
    monkeypatch.delenv("B2K_RNE_SPEC", raising=False)
    L, mdh = MATRIX_ROBOTS["mdh7_near_prismatic"]
    n, N = 7, 257
    for dt in (np.float64, np.float32):
        q, qd, qdd, tq = D.inputs(L, N, dt, 21)
        dev = []
        for x in (q, qd, qdd, tq):
            t = torch.empty(N * n + 1, dtype=torch.from_numpy(x).dtype, device="cuda")
            t[1:] = torch.from_numpy(x.ravel()).cuda()
            assert t[1:].data_ptr() % 16 != 0
            dev.append(t[1:])
        h = handle(L, mdh)
        for op in D.OPS:
            fext = FEXT if op == "rne" else None
            got, nl = launch(op, h, n, dt, op_inputs(op, *dev), N, GRAVS[2], fext)
            assert nl == 1, (op, nl)
            want, bar = reference(op, L, mdh, GRAVS[2], fext, q, qd, qdd, tq, dt)
            compare((np.dtype(dt).name, "unaligned", op), got, want, bar, accel_rows(L, mdh, q, dt) if op == "accel" else None)


def test_front_end_rotates_gravity_into_the_base_and_passes_row_slices(monkeypatch):
    """DHRobot with a rotated base: rne / gravload / accel hand the kernels -R_base^T g.  rne(q[1:], ...) and
    inertia(q[1:]) on the 7-joint Panda (a 56-byte fp64 row: the slice is only element-aligned)."""
    monkeypatch.delenv("B2K_RNE_SPEC", raising=False)
    c, s = np.cos(0.7), np.sin(0.7)
    base = np.array([[1, 0, 0, 0.1], [0, c, -s, 0.2], [0, s, c, 0.3], [0, 0, 0, 1.0]])
    rob = rtb.models.PandaMDH()
    rob.base = base
    L, n = rob._pack_rne(), rob.n
    g = -(base[:3, :3].T @ rob.gravity)
    q, qd, qdd, tq = D.inputs(L, 101, np.float64, 8)
    dq, dqd, dqdd, dtq = (torch.from_numpy(x).cuda() for x in (q, qd, qdd, tq))
    n0 = rtb.launch_count()
    tau = rob.rne(dq[1:], dqd[1:], dqdd[1:]).cpu().numpy()
    M = rob.inertia(dq[1:]).cpu().numpy()
    assert rtb.launch_count() - n0 == 2  # one generic launch each
    for got, op, kw in ((tau, "rne", dict(qd=qd[1:], x=qdd[1:])), (M, "inertia", {})):
        want, bar = D.op3(op, L, 1, g, q[1:], **kw)
        compare(("float64", "front_end", op), got, want.astype(np.float64), bar)
    puma = rtb.models.Puma560()
    puma.base = base
    Lp, gp = puma._pack_rne(), -(base[:3, :3].T @ puma.gravity)
    q6, qd6, _, tq6 = D.inputs(Lp, 96, np.float64, 9)
    d6 = [torch.from_numpy(x).cuda() for x in (q6, qd6, tq6)]
    for got, op, kw in ((puma.gravload(d6[0]), "gravload", {}), (puma.accel(*d6), "accel", dict(qd=qd6, x=tq6))):
        want, bar = D.op3(op, Lp, 0, gp, q6, **kw)
        compare(("float64", "front_end", op), got.cpu().numpy(), want.astype(np.float64), bar)


def test_misaligned_output_is_refused_without_a_launch():
    """An fp64 Puma tau at 8 mod 16 is element-aligned but not aligned to the 16-byte piece its rows are copied in."""
    lib = rtb._lib.lib()
    h = handle(ch.pack_rne(ch.puma560_links()), 0)
    x = torch.zeros(64 * 6 + 2, dtype=torch.float64, device="cuda")
    out = torch.zeros(64 * 6 + 2, dtype=torch.float64, device="cuda")
    g = np.array([0.0, 0.0, 9.81])
    n0 = rtb.launch_count()
    assert lib.b2k_rne(h, 1, x.data_ptr(), x.data_ptr(), x.data_ptr(), 64, rtb._lib.dptr(g), None, out.data_ptr() + 8, None) == -1
    assert b"tau must be 16-byte aligned" in lib.b2k_last_error()
    assert lib.b2k_rne_inertia(h, 1, x.data_ptr(), 64, out.data_ptr() + 8, None) == -1
    assert rtb.launch_count() == n0
