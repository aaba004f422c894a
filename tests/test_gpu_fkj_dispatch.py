"""The forward-kinematics / Jacobian kernels (b2k_fkj.cuh) at every joint count, chain profile, output mode and tile
edge, against the long-double reference of tests/fkj_ref.py.

Every call goes through one of the five C-ABI entry points into output buffers filled with a NaN sentinel and framed by
guard bytes, and checks: the number of kernel launches (lean kernel + ragged tail, or one kernel: this is what proves
which kernel ran), every output entry within a per-entry error bar derived from the arithmetic (fkj_ref.bars), the
guards untouched and no sentinel left in the outputs.  The largest error of each dtype x family x entry point, as a
fraction of its bar, is printed at the end of the module (run with -s to see it).
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import chains as ch  # noqa: E402

import fkj_ref as R  # noqa: E402

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
SENTINEL = {np.float64: (torch.int64, 0x7FF4DEADBEEF0BAD), np.float32: (torch.int32, 0x7FA0DEAD)}  # signalling NaNs
GUARD = 64  # bytes of guard before and after every output
ENTRIES = ("fkine", "jacob0", "jacobe", "fkine_jacob0", "fkine_jacobe")
BASE = ch.trotz(0.4) @ ch.troty(-0.3) @ ch.transl(0.2, -0.1, 0.5)
TOOL = ch.trotx(0.7) @ ch.transl(0.05, 0.1, 0.2)
REPORT = {}  # (dtype, family, entry) -> largest error / bar


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest error as a fraction of its bar (dtype, family, entry point):")
        for k in sorted(REPORT):
            print(f"  {k[0]:8s} {k[1]:14s} {k[2]:14s} {REPORT[k]:.3f}")


class Chain:
    def __init__(self, desc):
        self.desc = desc
        self.c = R.compile_chain(desc)
        self.n = self.c["n"]
        L = rtb._lib.lib()
        T = np.ascontiguousarray(desc["T"], dtype=np.float64)
        ql = np.ascontiguousarray(desc["qlim"], dtype=np.float64)
        self.h = rtb._lib.vp()
        ip = rtb._lib.ip
        rtb._lib.check(L.b2k_chain_create(len(desc["isjoint"]), desc["isjoint"].ctypes.data_as(ip),
                                          desc["axis"].ctypes.data_as(ip), desc["flip"].ctypes.data_as(ip),
                                          desc["jindex"].ctypes.data_as(ip), T.ctypes.data_as(rtb._lib.dp),
                                          ql.ctypes.data_as(rtb._lib.dp), rtb._lib.C.byref(self.h)))

    def __del__(self):
        rtb._lib.lib().b2k_chain_destroy(self.h)


def _mat(M):
    return None if M is None else np.ascontiguousarray(M, dtype=np.float64)


def guarded(nelem, dt, misalign=0):
    """(raw int tensor, float view of nelem elements): the view starts GUARD + misalign bytes into a 256-byte aligned
    allocation whose every element holds the sentinel bit pattern."""
    it, pat = SENTINEL[dt]
    es = np.dtype(dt).itemsize
    off = (GUARD + misalign) // es
    raw = torch.full((off + nelem + GUARD // es + 1,), pat, dtype=it, device="cuda")
    view = raw.view(torch.float64 if dt == np.float64 else torch.float32)[off:off + nelem]
    return raw, view, off


def check_guards(raw, off, nelem, dt, tag):
    _, pat = SENTINEL[dt]
    r = raw.cpu().numpy()
    assert (r[:off] == pat).all() and (r[off + nelem:] == pat).all(), ("guard overwritten", tag)
    assert not (r[off:off + nelem] == pat).any(), ("an output element was not written", tag)


def device_q(Q, qoff=0):
    """Q (N, ldq) on the device, the first row qoff elements past a 256-byte aligned address."""
    flat = torch.zeros(Q.size + qoff + 1, dtype=torch.float64 if Q.dtype == np.float64 else torch.float32, device="cuda")
    flat[qoff:qoff + Q.size] = torch.from_numpy(np.ascontiguousarray(Q).ravel()).cuda()
    return flat[qoff:qoff + Q.size]


def call(chain, entry, Q, base=None, tool=None, qoff=0, joff=0, variant=0):
    """One C-ABI call; returns (T or None, J or None) on the host after checking the guards and the launch count."""
    L = rtb._lib.lib()
    dt = Q.dtype.type
    N, ldq = Q.shape
    n = chain.n
    code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
    qd = device_q(Q, qoff)
    wt, wj = "fkine" in entry, "jacob" in entry
    Tb = guarded(N * 16, dt) if wt else None
    Jb = guarded(N * 6 * n, dt, joff) if wj else None
    b, t = _mat(base), _mat(tool)
    bp, tp = rtb._lib.dptr(b), rtb._lib.dptr(t)
    st = torch.cuda.current_stream().cuda_stream
    Tp = Tb[1].data_ptr() if wt else None
    Jp = Jb[1].data_ptr() if wj else None
    n0 = rtb.launch_count()
    fn = getattr(L, "b2k_" + entry)
    if entry == "fkine":
        rc = fn(chain.h, code, qd.data_ptr(), N, ldq, bp, tp, Tp, st)
    elif entry in ("jacob0", "jacobe"):
        rc = fn(chain.h, code, qd.data_ptr(), N, ldq, tp, Jp, st)
    else:
        rc = fn(chain.h, code, qd.data_ptr(), N, ldq, bp, tp, Tp, Jp, st)
    rtb._lib.check(rc)
    torch.cuda.synchronize()
    launches = rtb.launch_count() - n0
    if variant == 0:
        want = R.expected_launches(chain.c, ldq, qd.data_ptr(), N, variant)
        assert launches == want, (entry, n, N, ldq, launches, want)
    T = J = None
    if wt:
        check_guards(Tb[0], Tb[2], N * 16, dt, entry + " T")
        T = Tb[1].cpu().numpy().reshape(N, 4, 4)
    if wj:
        check_guards(Jb[0], Jb[2], N * 6 * n, dt, entry + " J")
        J = Jb[1].cpu().numpy().reshape(N, 6, n)
    return T, J


def compare(tag, got, want, bar, rows):
    """|got - want| <= bar entry by entry on the given rows; records the largest ratio under tag."""
    err = np.abs(got[rows].astype(np.float64) - want[rows].astype(np.float64))
    ratio = err / bar[rows]
    worst = float(np.nanmax(ratio)) if ratio.size else 0.0
    assert not np.isnan(ratio).any(), (tag, "NaN in a finite row")
    REPORT[tag] = max(REPORT.get(tag, 0.0), worst)
    assert worst <= 1.0, (tag, worst, np.unravel_index(int(np.argmax(ratio)), ratio.shape))


def check_entry(tag, entry, ref, T, J, dt, rows=None):
    N = ref["T"].shape[0]
    rows = np.arange(N) if rows is None else rows
    finite = rows[np.isfinite(ref["T"][rows].astype(np.float64)).all((1, 2))]
    if T is not None:
        assert (T[rows, 3] == np.array([0, 0, 0, 1], dtype=dt)).all(), tag
        pb = R.pose_bar(ref, dt)
        compare(tag + (entry,), T[:, :3], ref["T"][:, :3], pb[:, :3], finite)
    if J is not None:
        want = ref["Je"] if entry.endswith("jacobe") else ref["J0"]
        compare(tag + (entry,), J, want, R.jac_bar(ref, dt), finite)


def run_all(chain, fam, Q, base=None, tool=None, qoff=0, joff=0, entries=ENTRIES):
    """Every entry point on Q; the ones without a base argument get tool only."""
    dt = Q.dtype.type
    ref_b = R.evaluate(chain.desc, Q, base, tool)
    ref_nb = R.evaluate(chain.desc, Q, None, tool) if base is not None else ref_b
    out = {}
    for e in entries:
        takes_base = e.startswith("fkine")
        T, J = call(chain, e, Q, base if takes_base else None, tool, qoff, joff)
        check_entry((np.dtype(dt).name, fam), e, ref_b if takes_base else ref_nb, T, J, dt)
        out[e] = (T, J)
    return out


def rand_q(rng, N, ldq, dt, lo=-math.pi, hi=math.pi):
    return rng.uniform(lo, hi, (N, ldq)).astype(dt)


COUNTS = [1, 2, 31, 32, 33, 63, 65, 127, 129]


# ------------------------------------------------------------------ families x entry points x dtypes
@pytest.mark.parametrize("n", range(1, 11))
def test_dh_like_chains(n):
    """DH-like chains (PROF 1): the lean kernels on the full tiles, the general kernel on the ragged tail, at every
    row count of COUNTS plus ~1000 + r; all five entry points with and without base and tool."""
    rng = np.random.default_rng(n)
    for dt in (np.float64, np.float32):
        for i, tail in enumerate(("ident", "trans", "gen")):
            chain = Chain(R.dh_family(n, rng, tail))
            assert chain.c["dh_like"] and chain.c["dense_jindex"]
            for N in COUNTS[i::3] + [1000 + n + i]:
                Q = rand_q(rng, N, n, dt)
                run_all(chain, "dh-" + tail, Q)
                run_all(chain, "dh-" + tail, Q, BASE, TOOL)
                out = run_all(chain, "dh-" + tail, Q, None, TOOL, entries=("fkine", "fkine_jacob0", "jacob0"))
                # fused T == pose-only T, fused J0 == jacob0, bit for bit, when there is no base
                assert np.array_equal(out["fkine"][0], out["fkine_jacob0"][0])
                assert np.array_equal(out["jacob0"][1], out["fkine_jacob0"][1])


@pytest.mark.parametrize("n", range(1, 11))
def test_near_dh_chains_take_the_generic_profile(n):
    """One breaker of the DH-like rule at every position k: a flipped Rz joint, an Ry-form / Rz-form / general
    constant, a joint offset.  Each must take one launch of the generic (PROF 0) kernel, which the launch count
    asserts, and agree with the reference."""
    rng = np.random.default_rng(20 + n)
    cases = [("flip", k) for k in range(n)] + [(b, k) for k in range(1, n) for b in ("ry", "rz", "gen", "offset")]
    for i, (br, k) in enumerate(cases):
        chain = Chain(R.near_dh_family(n, k, br, rng))
        assert not chain.c["dh_like"]
        dt = (np.float64, np.float32)[i % 2]
        N = COUNTS[i % len(COUNTS)] + 32 * (i % 3)
        run_all(chain, "near-dh", rand_q(rng, N, n, dt), *((BASE, TOOL) if i % 2 else (None, None)))


@pytest.mark.parametrize("n", range(1, 11))
def test_generic_chains(n):
    """All six joint axes, flips, prismatic joints, and constants of every AK_* class x translation bits (spread over
    the n sweep by fkj_ref.generic_family) through both walks."""
    kinds = list(R.ALL_KINDS)
    rng = np.random.default_rng(40 + n)
    for m in range(1, n):  # consume the classes the smaller chains of the sweep took
        R.generic_family(m, np.random.default_rng(0), kinds)
    chain = Chain(R.generic_family(n, rng, kinds))
    assert not chain.c["dh_like"]
    for dt in (np.float64, np.float32):
        for N in (33, 129, 1000 + n):
            Q = rand_q(rng, N, n, dt, -2, 2)
            run_all(chain, "generic", Q)
            run_all(chain, "generic", Q, BASE, TOOL)


@pytest.mark.parametrize("n", range(1, 11))
def test_layouts(n):
    """q rows wider than n (ldq up to 16, both q staging modes), q one element past a 16-byte boundary, non-dense
    jindex, and J 8 but not 16-byte aligned (fp32, odd n): all on the general kernel, one launch each."""
    rng = np.random.default_rng(60 + n)
    chain = Chain(R.dh_family(n, rng, "gen"))
    for dt in (np.float64, np.float32):
        for ldq in sorted({n + 1, 4 * ((n + 4) // 4), 16, min(16, 2 * n + 1)}):
            if ldq < n or ldq > 16:
                continue
            run_all(chain, "layout", rand_q(rng, 65 + ldq, ldq, dt), BASE, TOOL)
        run_all(chain, "layout", rand_q(rng, 97, n, dt), None, TOOL, qoff=1)
        if dt == np.float32 and n % 2:
            run_all(chain, "layout", rand_q(rng, 97, n, dt), BASE, None, joff=8)
    perm = rng.permutation(16)[:n]
    chainp = Chain(R.with_jindex(R.dh_family(n, rng), perm))
    for dt in (np.float64, np.float32):
        run_all(chainp, "jindex", rand_q(rng, 161, 16, dt), BASE, TOOL)


def test_large_batch_many_blocks():
    """~262 147 rows: many blocks and a partial last block, lean + tail and generic; all rows checked for the guards
    and launches, a random subset and both ends against the reference."""
    rng = np.random.default_rng(7)
    N = 262147
    for desc, fam in ((R.dh_family(7, rng, "gen"), "dh-gen"), (R.generic_family(10, rng, []), "generic")):
        chain = Chain(desc)
        for dt in (np.float64, np.float32):
            Q = rand_q(rng, N, chain.n, dt)
            rows = np.unique(np.r_[0:64, N - 64:N, rng.integers(0, N, 2048)])
            ref = R.evaluate(desc, Q[rows], BASE, TOOL)
            refnb = R.evaluate(desc, Q[rows], None, TOOL)
            for e in ("fkine_jacob0", "fkine_jacobe", "jacob0"):
                T, J = call(chain, e, Q, BASE if e.startswith("fkine") else None, TOOL)
                check_entry((np.dtype(dt).name, fam), e, ref if e.startswith("fkine") else refnb,
                            None if T is None else T[rows], J[rows], dt)


# ------------------------------------------------------------------ sincos through the kernels
def _sweep32():
    big = np.float32(105615.0)
    x = np.concatenate([
        np.linspace(-8, 8, 4001), [np.nextafter(np.float32(8), np.float32(0)), -np.nextafter(np.float32(8), np.float32(0)), 8, -8],
        np.geomspace(8, 1e3, 600), -np.geomspace(8, 1e3, 600), np.geomspace(1e3, 105614, 600),
        [np.nextafter(big, np.float32(0)), big, np.nextafter(big, np.float32(1e6)), -big],
        np.geomspace(105616, 1e22, 300), [0.0, -0.0, 1e-45, -1e-45, 1e-39, np.inf, -np.inf, np.nan]])
    return x


TRIG_REPORT = {}


def _trig_errors(x, s, c, dt):
    xr = x.astype(R.LD)
    rs, rc = np.sin(xr), np.cos(xr)
    eps = float(np.finfo(dt).eps)
    ae = np.maximum(np.abs(s.astype(R.LD) - rs), np.abs(c.astype(R.LD) - rc)).astype(np.float64)
    us = (np.abs(s.astype(R.LD) - rs) / np.maximum(np.abs(rs) * eps, R.LD(eps) * eps)).astype(np.float64)
    uc = (np.abs(c.astype(R.LD) - rc) / np.maximum(np.abs(rc) * eps, R.LD(eps) * eps)).astype(np.float64)
    return ae, np.maximum(us, uc)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_sincos_through_the_kernels(dt):
    """Rz(q) with identity constants gives T[0,0] = cos q and T[1,0] = sin q from b2k_sincos_batch<real, 1> (lean
    kernel at N = 32k, general kernel through an ldq = 2 copy); Rx(q) gives T[1,1] and T[2,1] from the scalar
    b2k_sincos of the generic profile.  Pins: on the special-function path the error beyond the rounding of the
    unit's argument (fkj_ref.mufu_arg_error) within 2^-21.4 (measured on H100: 3.1e-7 beyond it, 1.16e-6 in all at
    |x| < 8, where b2k_trig.cuh's |x| 2^-25 argument term would allow 6e-7); on the other paths 2 ulp (fp64) / 2.5 ulp (fp32), with an absolute floor of eps^2, up to |x| = 100
    (b2k_trig.cuh's measured 1.6) and 2 eps absolute at every finite angle; NaN for non-finite angles."""
    x = _sweep32().astype(dt)
    x = np.concatenate([x, np.zeros((-len(x)) % 32, dt)])
    finite = np.isfinite(x)
    ax = np.abs(x.astype(np.float64))
    eps = float(np.finfo(dt).eps)
    rz = Chain(ch.Builder().joint(R.RZ).desc())
    rx = Chain(ch.Builder().joint(R.RX).desc())
    checks = []
    for chain, name, (si, ci) in ((rz, "batch", ((1, 0), (0, 0))), (rx, "scalar", ((2, 1), (1, 1)))):
        for ldq in (1, 2):
            Q = np.stack([x, np.zeros_like(x)], 1)[:, :ldq].copy()
            T, _ = call(chain, "fkine", Q)
            s, c = T[:, si[0], si[1]], T[:, ci[0], ci[1]]
            checks.append((name, ldq, "NaN out for non-finite in", np.isnan(s[~finite]).all() and np.isnan(c[~finite]).all()))
            checks.append((name, ldq, "cos(+-0) == 1, sin(+-0) == 0", (c[x == 0] == 1).all() and (s[x == 0] == 0).all()))
            ae, ulp = _trig_errors(x[finite], s[finite], c[finite], dt)
            path, _ = R.sincos_path(x[finite, None], dt, name == "batch")
            small = ax[finite] < 100
            for p, label in ((R.PATH_MUFU, "mufu"), (R.PATH_POLY, "poly"), (R.PATH_SLOW, "slow")):
                sel = path == p
                if not sel.any():
                    continue
                key = (np.dtype(dt).name, name, "lean" if ldq == 1 else "general", label)
                if p == R.PATH_MUFU:
                    resid = ae[sel] - R.mufu_arg_error(x[finite][sel])
                    TRIG_REPORT[key] = (float(ae[sel].max()), float(resid.max()), float(ulp[sel].max()))
                    checks.append(key + ("unit error", resid.max() <= R.MUFU_ERR))
                else:
                    TRIG_REPORT[key] = (float(ae[sel].max()), float("nan"), float(ulp[sel & small].max(initial=0)))
                    checks.append(key + ("2 eps", ae[sel].max() <= 2 * eps))
                    checks.append(key + ("ulp", ulp[sel & small].max(initial=0) <= (2.0 if dt == np.float64 else 2.5)))
    print("\nsincos through the kernels: (dtype, trig, kernel, path) -> max abs error, max of it beyond the "
          "argument rounding, max ulp (|x| < 100 off the special-function path)")
    for k in sorted(TRIG_REPORT):
        if k[0] == np.dtype(dt).name:
            print(f"  {k}: {TRIG_REPORT[k][0]:.3e}  {TRIG_REPORT[k][1]:.3e}  {TRIG_REPORT[k][2]:.2f}")
    failed = [c[:-1] for c in checks if not c[-1]]
    assert not failed, failed


@pytest.mark.parametrize("n", range(2, 11))
def test_mixed_sincos_paths_in_one_warp(n):
    """fp32 DH-like rows of one warp on three sincos paths: every angle below 8 (special-function unit), exactly one
    angle in [8, 1e3] (the whole row on the polynomial), one angle >= 105615 or non-finite (the whole row on the scalar
    fallback).  Each row within its own path's bar; non-finite rows NaN only in their own outputs."""
    rng = np.random.default_rng(80 + n)
    chain = Chain(R.dh_family(n, rng, "gen"))
    N = 96 + 7
    Q = rand_q(rng, N, n, np.float32, -3, 3)
    kind = np.arange(N) % 3
    j = rng.integers(0, n, N)
    Q[kind == 1, j[kind == 1]] = rng.uniform(8, 1e3, int((kind == 1).sum())).astype(np.float32)
    far = np.array([105615.0, -2e5, 1e22, np.inf, -np.inf, np.nan], np.float32)
    Q[kind == 2, j[kind == 2]] = far[np.arange(int((kind == 2).sum())) % len(far)]
    ref = R.evaluate(chain.desc, Q, BASE, TOOL)
    assert set(ref["path"].tolist()) == {R.PATH_MUFU, R.PATH_POLY, R.PATH_SLOW}
    bad = ~np.isfinite(Q).all(1)
    for e in ENTRIES:
        takes_base = e.startswith("fkine")
        r = ref if takes_base else R.evaluate(chain.desc, Q, None, TOOL)
        T, J = call(chain, e, Q, BASE if takes_base else None, TOOL)
        check_entry(("float32", "dh-mixed-trig"), e, r, T, J, np.float32, np.flatnonzero(~bad))
        for X in (T, J):
            if X is not None:
                assert np.isfinite(X[~bad]).all()


# ------------------------------------------------------------------ row independence, lean vs general
@pytest.mark.parametrize("n", [1, 3, 6, 7, 10])
def test_row_independence(n):
    """Replacing every other row by NaN / +-inf / 1e30 rows, or permuting the rows (full tiles among themselves, the
    ragged tail among itself), leaves every other row's outputs bit-identical; non-finite rows spoil only themselves."""
    rng = np.random.default_rng(90 + n)
    for desc, fam in ((R.dh_family(n, rng, "gen"), "dh"), (R.generic_family(n, rng, []), "generic")):
        chain = Chain(desc)
        for dt in (np.float64, np.float32):
            N = 128 + 13
            Q = rand_q(rng, N, n, dt)
            Qb = Q.copy()
            junk = np.array([np.nan, np.inf, -np.inf, 1e30], dtype=dt)
            Qb[1::2] = junk[(np.arange(N // 2) % 4)][:, None]
            perm = np.r_[rng.permutation(128), 128 + rng.permutation(13)]
            for e in ENTRIES:
                base = BASE if e.startswith("fkine") else None
                a = call(chain, e, Q, base, TOOL)
                b = call(chain, e, Qb, base, TOOL)
                p = call(chain, e, Q[perm].copy(), base, TOOL)
                for X, Y, Z in zip(a, b, p):
                    if X is None:
                        continue
                    assert np.array_equal(X[0::2], Y[0::2]), (fam, e, dt)
                    assert np.array_equal(X[perm], Z), (fam, e, dt)
                    assert np.isfinite(Y[0::2]).all()


@pytest.mark.parametrize("n", range(1, 11))
def test_lean_and_general_kernels_agree(n):
    """The same rows through the lean kernel (ldq = n) and the general kernel (an ldq = n + 1 copy): both within the
    bar; whether they agree bit for bit is reported."""
    rng = np.random.default_rng(110 + n)
    chain = Chain(R.dh_family(n, rng, "gen"))
    for dt in (np.float64, np.float32):
        Q = rand_q(rng, 256, n, dt)
        Qw = np.concatenate([Q, np.full((256, 1), 7.0, dt)], 1)
        for e in ENTRIES:
            base = BASE if e.startswith("fkine") else None
            ref = R.evaluate(chain.desc, Q, base, TOOL)
            lean = call(chain, e, Q, base, TOOL)
            gen = call(chain, e, Qw, base, TOOL)
            check_entry((np.dtype(dt).name, "dh-lean"), e, ref, *lean, dt)
            check_entry((np.dtype(dt).name, "dh-general"), e, ref, *gen, dt)
            same = all(np.array_equal(x, y) for x, y in zip(lean, gen) if x is not None)
            REPORT[(np.dtype(dt).name, "lean==general", e)] = max(REPORT.get((np.dtype(dt).name, "lean==general", e), 0.0),
                                                                 0.0 if same else 1.0)


# ------------------------------------------------------------------ several tiles per warp, measurement variants
def _persistent_tpw(nrows):
    """An upper bound of the grid of variant 4 (launch_impl: as many blocks as fit, each warp a contiguous share) and
    the tiles per warp it gives: at most max-threads-per-SM / 128 blocks of 128 threads per SM."""
    p = torch.cuda.get_device_properties(0)
    g = p.multi_processor_count * (p.max_threads_per_multi_processor // 128)
    ntiles = (nrows + 31) // 32
    return (ntiles + g * 4 - 1) // (g * 4)


@pytest.mark.parametrize("n", [1, 4, 7, 10])
def test_persistent_grid_several_tiles_per_warp(n):
    """set_variant(4) at 1M + 17 rows: every warp walks several consecutive tiles (next-tile q load, L2 prefetch)."""
    N = (1 << 20) + 17
    assert _persistent_tpw(N) > 1
    rng = np.random.default_rng(130 + n)
    rows = np.unique(np.r_[0:64, N - 64:N, rng.integers(0, N, 1024)])
    rtb.set_variant(4)
    try:
        for desc, fam in ((R.dh_family(n, rng, "gen"), "v4-dh"), (R.generic_family(n, rng, []), "v4-generic")):
            chain = Chain(desc)
            for dt in (np.float64, np.float32):
                Q = rand_q(rng, N, n, dt)
                ref = R.evaluate(desc, Q[rows], BASE, TOOL)
                for e in ("fkine_jacob0", "fkine_jacobe", "fkine"):
                    T, J = call(chain, e, Q, BASE, TOOL, variant=4)
                    check_entry((np.dtype(dt).name, fam), e, ref, T[rows], None if J is None else J[rows], dt)
    finally:
        rtb.set_variant(0)


def tpw3_body():
    """Run in a process started with B2K_TPW_POSE=3 B2K_TPW_JAC=3 (read once per process)."""
    rng = np.random.default_rng(5)
    for n in (2, 7, 10):
        for desc, fam in ((R.generic_family(n, rng, []), "tpw3-generic"), (R.dh_family(n, rng, "gen"), "tpw3-tail")):
            chain = Chain(desc)
            for dt in (np.float64, np.float32):
                for N in (32 * 4 * 3 * 5 + 17, 1000 + n):
                    run_all(chain, fam, rand_q(rng, N, n, dt), BASE, TOOL)
    print("TPW3_OK")


def test_three_tiles_per_warp_in_the_default_variant():
    env = dict(os.environ, B2K_TPW_POSE="3", B2K_TPW_JAC="3")
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_fkj_dispatch as t; t.tpw3_body()"
            % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0 and "TPW3_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("n", [6, 7])
def test_warp_per_configuration_variant(n):
    """set_variant(1): the warp-per-configuration walk (b2k_fkw.cu, built for n = 6 and 7 only) on a DH-like chain;
    it calls the scalar sincos."""
    rng = np.random.default_rng(150 + n)
    chain = Chain(R.dh_family(n, rng, "gen"))
    rtb.set_variant(1)
    try:
        for dt in (np.float64, np.float32):
            Q = rand_q(rng, 77, n, dt)
            for e, base in (("fkine", BASE), ("jacob0", None), ("fkine_jacob0", BASE)):
                ref = R.evaluate(chain.desc, Q, base, TOOL, batch_trig=False)
                T, J = call(chain, e, Q, base, TOOL, variant=1)
                check_entry((np.dtype(dt).name, "variant1"), e, ref, T, J, dt)
    finally:
        rtb.set_variant(0)


def test_public_ets_methods():
    """One pass through ETS.eval / jacob0 / jacobe / fkine_jacob0 on device tensors."""
    rng = np.random.default_rng(170)
    AX = ["Rx", "Ry", "Rz", "tx", "ty", "tz"]
    for desc in (R.dh_family(6, rng, "gen"), R.generic_family(8, rng, [])):
        ets = []
        for i in range(len(desc["isjoint"])):
            if desc["isjoint"][i]:
                ets.append(rtb.ET(AX[int(desc["axis"][i])], flip=bool(desc["flip"][i]), jindex=int(desc["jindex"][i])))
            else:
                ets.append(rtb.ET.SE3(desc["T"][i]))
        e = rtb.ETS(ets)
        for dt in (np.float64, np.float32):
            Q = rand_q(rng, 100, e.n, dt)
            qd = torch.from_numpy(Q).cuda()
            ref = R.evaluate(desc, Q, BASE, TOOL)
            refnb = R.evaluate(desc, Q, None, TOOL)
            T, J = (x.cpu().numpy() for x in e.fkine_jacob0(qd, base=BASE, tool=TOOL))
            check_entry((np.dtype(dt).name, "ETS"), "fkine_jacob0", ref, T, J, dt)
            check_entry((np.dtype(dt).name, "ETS"), "fkine", ref, e.eval(qd, base=BASE, tool=TOOL).cpu().numpy(), None, dt)
            check_entry((np.dtype(dt).name, "ETS"), "jacob0", refnb, None, e.jacob0(qd, tool=TOOL).cpu().numpy(), dt)
            check_entry((np.dtype(dt).name, "ETS"), "jacobe", refnb, None, e.jacobe(qd, tool=TOOL).cpu().numpy(), dt)
