"""Sweep of the operational-space kernels (csrc/b2k_opspace.cu): every instantiation of k_opspace (B2K_OPS_PINV at
n = 1..10, B2K_OPS_INV at n = 6) and of k_opspace_xdd (n = 1..10), in fp64 and fp32.

a. Synthetic Ja = U diag(s) V^T with well-conditioned, graded and exactly rank-deficient spectra, through the C ABI,
   against the mpmath reference of tests/opspace_mp_ref.py within its error bars (the worst error / bar per dtype,
   joint count, inverse kind and output is printed at the end of the module).
b. One launch writing all six outputs against one launch per output, and outputs fed back as Ji_in / Mx_in: bitwise.
c. N around the 32-row tile up to 100 003 rows, every array a view starting one element past a 16-byte boundary inside
   NaN guards: the guards stay NaN, the written rows hold no NaN and equal those of contiguous arrays bit for bit.
d. A NaN, Inf or zero-pivot row in the middle of a tile changes no other row.  A NaN never passes the Jacobi
   convergence test, so that lane runs all 30 sweeps while the rest of its warp has finished.
e. The robot classes end to end (random revolute DH / MDH arms at n = 1..10 and the xacro tree), against the numpy
   restatement of tests/opspace_ref.py, with the robot-specialised RNE path off (B2K_RNE_SPEC=0): its 10-joint Coriolis
   program takes minutes to compile, and test_gpu_rne_spec.py covers it."""
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
import opspace_mp_ref as R  # noqa: E402
import opspace_ref as ops  # noqa: E402
import rne_derivs_ref as RD  # noqa: E402
from oracle import oracle as orc  # noqa: E402

PINV, INV = rtb._lib.OPS_PINV, rtb._lib.OPS_INV
KINDS = [(n, PINV) for n in range(1, 11)] + [(6, INV)]
KIND_IDS = [f"pinv{n}" if k == PINV else f"inv{n}" for n, k in KINDS]
DTS = [np.float64, np.float32]
OUTS = ("Ji", "Mx", "Cx", "Gx", "qd", "tau")
INS = ("Ja", "Ji_in", "M", "C", "Jd", "G", "Mx_in", "xd", "w")
TORCH = {np.float64: torch.float64, np.float32: torch.float32}
CODE = {np.float64: rtb._lib.F64, np.float32: rtb._lib.F32}
G_CUSTOM = np.array([1.5, -2.0, -9.81])
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nworst error / bar per (dtype, n, kind, output):")
    for k in sorted(WORST, key=str):
        print(f"  {k[0]:8s} {k[1]:3d} {k[2]:5s} {k[3]:4s} {WORST[k]:.3g}")


def shape(name, n):
    return {"Ja": (6, n), "Ji_in": (n, 6), "M": (n, n), "C": (n, n), "Jd": (6, n), "G": (n,), "Mx_in": (6, 6), "xd": (6,),
            "w": (6,), "Ji": (n, 6), "Mx": (6, 6), "Cx": (6, 6), "Gx": (6,), "qd": (n,), "tau": (n,), "qdd": (n,),
            "xdd": (6,)}[name]


def cuda(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=dt)).cuda()


def _p(t):
    return None if t is None else t.data_ptr()


def opspace(dt, n, kind, N, ins, outs, alloc=None):
    """One b2k_opspace launch.  ins: {name: device tensor}; outs: the outputs to request.  Returns {name: tensor}, each
    from alloc(name) (default: NaN-filled contiguous)."""
    alloc = alloc or (lambda k: torch.full((N,) + shape(k, n), float("nan"), dtype=TORCH[dt], device="cuda"))
    res = {k: alloc(k) for k in outs}
    rtb._lib.check(rtb._lib.lib().b2k_opspace(CODE[dt], n, kind, *[_p(ins.get(k)) for k in INS], N,
                                              *[_p(res.get(k)) for k in OUTS], torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return res


def opspace_xdd(dt, n, N, Ja, qdd, Jd, qd, out=None):
    out = torch.full((N, 6), float("nan"), dtype=TORCH[dt], device="cuda") if out is None else out
    rtb._lib.check(rtb._lib.lib().b2k_opspace_xdd(CODE[dt], n, Ja.data_ptr(), qdd.data_ptr(), Jd.data_ptr(), qd.data_ptr(), N,
                                                  out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out


def host(t):
    return t.cpu().numpy().astype(np.float64)


def record(dt, n, kind, out, r):
    key = (np.dtype(dt).name, n, "pinv" if kind == PINV else "inv", out)
    WORST[key] = max(WORST.get(key, 0.0), float(np.max(r, initial=0.0)))


# ------------------------------------------------------------------ a. synthetic operands against the mp reference

@pytest.mark.parametrize("n,kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("dt", DTS, ids=["f64", "f32"])
def test_synthetic_operands_against_the_mp_reference(dt, n, kind):
    """80 rows (two full tiles and a ragged one) cycling through the five spectra of opspace_mp_ref.synthetic; up to 48
    rows, 0, 31, 32 and 79 among them, compared."""
    N = 80
    rng = np.random.default_rng(zlib.crc32(f"sweep{np.dtype(dt).name}{n}{kind}".encode()))
    Ja, names = R.synthetic(n, N, dt, rng)
    o = R.operands(n, N, dt, rng)
    ins = {k: cuda(v, dt) for k, v in o.items()}
    ins["Ja"] = cuda(Ja, dt)
    got = {k: host(v) for k, v in opspace(dt, n, kind, N, ins, OUTS).items()}
    got["xdd"] = host(opspace_xdd(dt, n, N, ins["Ja"], ins["qdd"], ins["Jd"], ins["qd"]))

    rows = R.sample(N, rng)
    pinv = kind == PINV
    names = np.asarray(names)[rows]
    inv = R.inverse(Ja[rows], pinv)
    ref = R.opspace(Ja[rows], pinv, dt, M=o["M"][rows], C=o["C"][rows], Jd=o["Jd"][rows], G=o["G"][rows], xd=o["xd"][rows],
                    w=o["w"][rows], inv=inv)
    ref["xdd"] = R.xdd(Ja[rows], o["qdd"][rows], o["Jd"][rows], o["qd"][rows], dt)
    use = R.compared(Ja[rows], names, pinv, dt, inv)
    assert use.sum() >= 20 if pinv else use.sum() >= 12
    if not pinv:  # an exactly zero pivot: NaN in everything Ji reaches, as in the reference
        nan_rows = np.isin(names, ("zcol", "zrow"))
        assert nan_rows.any() and not np.isfinite(inv[1][nan_rows]).any()
        for k in ("Ji", "Mx", "Cx", "Gx", "qd"):
            assert np.isnan(got[k][rows][nan_rows]).all(), k
    for k, (want, bar) in ref.items():
        sel = slice(None) if k in ("tau", "xdd") else use  # no inverse in these two: every row has an answer
        r = R.ratio(got[k][rows][sel], want[sel], bar[sel])
        assert np.isfinite(r).all(), (k, rows[sel][~np.isfinite(r)])
        record(dt, n, kind, k, r)
        assert r.max() <= 1.0, (k, float(r.max()), int(rows[sel][np.argmax(r)]), names[sel][np.argmax(r)])


# ------------------------------------------------------------------ b. one launch against many

def _random_case(dt, n, N, seed, spectra=("well", "graded")):
    rng = np.random.default_rng(seed)
    Ja, _ = R.synthetic(n, N, dt, rng, spectra=spectra)
    ins = {k: cuda(v, dt) for k, v in R.operands(n, N, dt, rng).items()}
    ins["Ja"] = cuda(Ja, dt)
    return ins


@pytest.mark.parametrize("n,kind", KINDS, ids=KIND_IDS)
@pytest.mark.parametrize("dt", DTS, ids=["f64", "f32"])
def test_one_launch_equals_one_launch_per_output_and_fed_back_outputs(dt, n, kind):
    N = 70
    ins = _random_case(dt, n, N, 500 + n + 20 * kind + (dt == np.float32))
    every = opspace(dt, n, kind, N, ins, OUTS)
    for k, v in every.items():
        assert torch.isfinite(v).all(), k
        assert torch.equal(opspace(dt, n, kind, N, ins, (k,))[k], v), k
    fed = dict(ins, Ja=None, Ji_in=every["Ji"])
    got = opspace(dt, n, kind, N, fed, ("Mx", "Cx", "Gx", "qd"))
    for k, v in got.items():
        assert torch.equal(v, every[k]), f"{k} from Ji_in"
    got = opspace(dt, n, kind, N, dict(ins, M=None, Mx_in=every["Mx"]), ("Cx",))
    assert torch.equal(got["Cx"], every["Cx"]), "Cx from Mx_in"
    # Ja is staged for tau but not inverted when Ji_in is given
    got = opspace(dt, n, kind, N, dict(ins, Ji_in=every["Ji"]), ("tau", "qd", "Gx"))
    for k, v in got.items():
        assert torch.equal(v, every[k]), f"{k} with Ja and Ji_in"


# ------------------------------------------------------------------ c. tile edges and stray writes

def guarded(N, n, name, dt, like=None):
    """(buffer, view): a NaN buffer with two rows of guard on each side; the (N, ...) view starts one element past a
    16-byte boundary (the allocation itself is at least 256-byte aligned).  like: values to copy into the view."""
    row = int(np.prod(shape(name, n)))
    es = np.dtype(dt).itemsize
    k = 16 // es
    lo = -(-2 * row // k) * k + 1
    buf = torch.full((lo + N * row + 2 * row,), float("nan"), dtype=TORCH[dt], device="cuda")
    assert buf.data_ptr() % 256 == 0
    view = buf[lo:lo + N * row].view((N,) + shape(name, n))
    assert view.data_ptr() % 16 == es
    if like is not None:
        view.copy_(like)
    return buf, view, lo, lo + N * row


def guards_intact(buf, lo, hi):
    return bool(torch.isnan(buf[:lo]).all()) and bool(torch.isnan(buf[hi:]).all())


EDGE_KINDS = [(1, PINV), (6, PINV), (6, INV), (7, PINV), (10, PINV)]


@pytest.mark.parametrize("n,kind", EDGE_KINDS, ids=[f"pinv{n}" if k == PINV else f"inv{n}" for n, k in EDGE_KINDS])
@pytest.mark.parametrize("dt", DTS, ids=["f64", "f32"])
def test_tile_edges_leave_the_guards_and_match_contiguous_arrays(dt, n, kind):
    g = torch.Generator(device="cuda")
    g.manual_seed(900 + n + kind)
    for N in (1, 31, 32, 33, 63, 64, 65, 1025, 100_003):
        dense = {k: torch.randn((N,) + shape(k, n), generator=g, dtype=TORCH[dt], device="cuda")
                 for k in ("Ja", "M", "C", "Jd", "G", "xd", "w", "qdd", "qd")}
        want = opspace(dt, n, kind, N, dense, OUTS)
        want_xdd = opspace_xdd(dt, n, N, dense["Ja"], dense["qdd"], dense["Jd"], dense["qd"])
        ins = {k: guarded(N, n, k, dt, v)[1] for k, v in dense.items()}
        bufs = {}

        def alloc(k):
            bufs[k] = guarded(N, n, k, dt)
            return bufs[k][1]

        got = opspace(dt, n, kind, N, ins, OUTS, alloc)
        bufs["xdd"] = guarded(N, n, "xdd", dt)
        got["xdd"] = opspace_xdd(dt, n, N, ins["Ja"], ins["qdd"], ins["Jd"], ins["qd"], out=bufs["xdd"][1])
        for k, v in dict(want, xdd=want_xdd).items():
            buf, _, lo, hi = bufs[k]
            assert guards_intact(buf, lo, hi), (N, k)
            assert not torch.isnan(got[k]).any(), (N, k)
            assert torch.equal(got[k], v), (N, k)


# ------------------------------------------------------------------ d. row isolation

BAD = [("nan", 7, PINV), ("nan", 10, PINV), ("nan", 3, PINV), ("inf", 6, PINV), ("inf", 6, INV), ("nan", 6, INV),
       ("zero_pivot", 6, INV)]


@pytest.mark.parametrize("bad,n,kind", BAD, ids=[f"{b}-{'pinv' if k == PINV else 'inv'}{n}" for b, n, k in BAD])
@pytest.mark.parametrize("dt", DTS, ids=["f64", "f32"])
def test_a_bad_row_changes_only_itself(dt, bad, n, kind):
    N, rows = 96, (45, 77)  # lanes 13 and 13 of the second and third tiles
    ins = _random_case(dt, n, N, 700 + n)
    base = opspace(dt, n, kind, N, ins, OUTS)
    base_xdd = opspace_xdd(dt, n, N, ins["Ja"], ins["qdd"], ins["Jd"], ins["qd"])
    Ja = ins["Ja"].clone()
    for r in rows:
        if bad == "nan":
            Ja[r, 2, n - 1] = float("nan")
        elif bad == "inf":
            Ja[r, 0, 0] = float("inf")
        else:  # an exactly zero column: the elimination's pivot for it is 0
            Ja[r, :, 2] = 0
    bad_ins = dict(ins, Ja=Ja)
    got = opspace(dt, n, kind, N, bad_ins, OUTS)
    got["xdd"] = opspace_xdd(dt, n, N, Ja, ins["qdd"], ins["Jd"], ins["qd"])
    others = torch.ones(N, dtype=torch.bool, device="cuda")
    others[list(rows)] = False
    for k, v in dict(base, xdd=base_xdd).items():
        assert torch.equal(got[k][others], v[others]), k
    if bad == "zero_pivot":
        for k in ("Ji", "Mx", "Cx", "Gx", "qd"):
            assert torch.isnan(got[k][list(rows)]).all(), k
        assert torch.isfinite(got["tau"]).all()
    if bad == "nan" and kind == PINV:
        assert torch.isnan(got["Ji"][list(rows)]).all()


# ------------------------------------------------------------------ e. the robot classes end to end

REPS = ("rpy/xyz", "rpy/zyx", "eul", "exp")
URDF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "urdf", "macro_arm.urdf.xacro")


def _robot(n, mdh):
    if n == "tree":
        rob = rtb.Robot.URDF(URDF)
        tree = rob.tree_description()
        rne = lambda a, b, c, g: orc.tree_rne(tree, np.atleast_2d(a), np.atleast_2d(b), np.atleast_2d(c), g)  # noqa: E731
        return rob, rne, rne
    L = RD.robot(n, mdh, False, True, 1300 + 10 * n + mdh)
    rob = RD.dhrobot(L, mdh)
    Lnf = orc.nofriction_L(L)
    rne = lambda q, qd, qdd, g: orc.rne(n, mdh, L, -np.asarray(g, dtype=float), q, qd, qdd)  # noqa: E731
    rne_nf = lambda q, qd, qdd, g: orc.rne(n, mdh, Lnf, -np.asarray(g, dtype=float), q, qd, qdd)  # noqa: E731
    return rob, rne, rne_nf


def close(got, want, terms=None, tol=None):
    """|got - want| <= tol (per row) * the row's scale: the largest |entry| of want, or of terms (the magnitude of what
    it is a difference of) where given, and at least 1e-3 -- an output that vanishes identically (the gravity load of a
    vertical first axis, the Coriolis terms of a one-joint arm) is compared absolutely"""
    got = host(got) if torch.is_tensor(got) else np.asarray(got, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    g, w = got.reshape(len(got), -1), want.reshape(len(want), -1)
    scale = np.maximum(np.abs(w).max(1), 1e-3)
    if terms is not None:
        scale = np.maximum(scale, np.abs(terms).reshape(len(w), -1).max(1))
    err = np.abs(g - w).max(1) / scale
    assert (err <= tol).all(), f"row-relative error {err.max():.3g} > {tol[np.argmax(err / tol)]:.3g}"


def coriolis_ref(rne, rne_nf, chain, n, q, qd, pinv, rep, Jd):
    """(Cx, |Ji^T C Ji| + |Mx Jd Ji|) from the reference's Ji, C and M and the given Jad"""
    Ji = ops.ji(ops.ja(chain, q, rep), pinv)
    JiT = np.swapaxes(Ji, 1, 2)
    Mx = JiT @ orc.dyn_inertia(rne, n, q) @ Ji
    a, b = JiT @ orc.dyn_coriolis(rne_nf, n, q, qd) @ Ji, Mx @ Jd @ Ji
    return a - b, np.abs(a) + np.abs(b)


ARMS = [(n, mdh) for n in range(1, 11) for mdh in (0, 1)] + [("tree", 0)]


@pytest.mark.parametrize("n,mdh", ARMS, ids=[f"{'mdh' if m else 'dh'}{n}" if n != "tree" else "tree" for n, m in ARMS])
@pytest.mark.parametrize("dt", DTS, ids=["f64", "f32"])
def test_robot_classes_end_to_end(monkeypatch, dt, n, mdh):
    """Four representations on inertia_x / coriolis_x / gravload_x / accel_x, the robot's and a custom gravity, pinv
    at every n and inv at n = 6, on rows with cond(Ja) < 1e4 (fp64) or 1e3 (fp32).  Tolerances, relative to the
    largest entry of the reference row (see `close`), are those of test_gpu_opspace.py widened by max(1, cond / 100).
    The fp32 Coriolis reference takes the device's own Jad: on one- and two-joint arms the Jad term dominates Cx, and the
    fp32 difference step's rounding alone reaches 1e-2 of it."""
    monkeypatch.setenv("B2K_RNE_SPEC", "0")
    rob, rne, rne_nf = _robot(n, mdh)
    n = rob.n
    chain = orc.Chain(rob.ets().describe())
    N = 33
    rng = np.random.default_rng(zlib.crc32(f"e2e{np.dtype(dt).name}{n}{mdh}".encode()))
    r = (lambda a: a.astype(np.float32).astype(np.float64)) if dt == np.float32 else (lambda a: a)
    q, qd = r(rng.uniform(-2.5, 2.5, (N, n))), r(rng.normal(size=(N, n)))
    xd, w = r(rng.normal(size=(N, 6)) * (0.2 if dt == np.float32 else 1.0)), r(rng.normal(size=(N, 6)) * 5)
    qt, qdt, xdt, wt = cuda(q, dt), cuda(qd, dt), cuda(xd, dt), cuda(w, dt)
    h = 1e-3 if dt == np.float32 else 1e-6  # the difference step of ETS.jacob0_dot in that dtype
    for pinv in (True, False) if n == 6 else (True,):
        for i, rep in enumerate(REPS):
            gravity = G_CUSTOM if i % 2 else None
            g = rob.gravity if gravity is None else gravity
            cond = np.linalg.cond(ops.ja(chain, q, rep))
            rows = np.flatnonzero(cond < (1e4 if dt == np.float64 else 1e3))
            assert len(rows) >= 8, (rep, len(rows))
            wide = np.maximum(1.0, cond[rows] / 100)
            base = {np.float64: (1e-8, 1e-7), np.float32: ((5e-3, 5e-3) if pinv else (2e-3, 2e-3))}[dt]
            qs = q[rows]
            close(host(rob.inertia_x(qt, pinv=pinv, representation=rep))[rows],
                  ops.inertia_x(rne, chain, n, qs, pinv, rep), tol=base[0] * wide)
            close(host(rob.gravload_x(qt, gravity=gravity, pinv=pinv, representation=rep))[rows],
                  ops.gravload_x(rne, chain, n, qs, g, pinv, rep), tol=base[0] * wide)
            if dt == np.float64:
                Jd = ops.jad(chain, qs, qd[rows], rep)
            else:  # fp32 jacob0_dot differences Ja at h = 1e-3, good to ~u/h of |Ja| (its own sweep holds it to that)
                Jd = host(rob.jacob0_dot(qt, qdt, representation=rep)).reshape(N, 6, n)[rows]
            close(host(rob.coriolis_x(qt, qdt, pinv=pinv, representation=rep))[rows],
                  *coriolis_ref(rne, rne_nf, chain, n, qs, qd[rows], pinv, rep, Jd), tol=base[1] * wide)
            close(host(rob.accel_x(qt, xdt, wt, gravity=gravity, pinv=pinv, representation=rep))[rows],
                  ops.accel_x(rne, chain, n, qs, xd[rows], w[rows], g, pinv, rep, h), tol=base[1] * wide)
