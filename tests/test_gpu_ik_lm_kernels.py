"""The batched LM / NR / GN inverse-kinematics kernels (csrc/b2k_ik.cuh: k_ik_lm, k_ik_restarts; STEP = 0 for LM, 1 for
NR / GN) at every joint count, chain profile, step rule, weighting, precision, loop semantics and restart schedule.

a. One step of every variant against the 40-digit reference of tests/ik_lm_ref.py: with Python semantics and
   ilimit = slimit = 1, q_out - q0 is the kernel's step and residual is E(q0).
b. The whole loop (seeded restarts, joint limits on / off, both semantics) against the oracle's sequential loop.
c. The schedule (persistent launch, two phases, split first search, every shape of the restart rounds) changes no
   reported number: restart draws are keyed by (seed, row, search, joint).
d. Edge batch sizes, a grid that must pull more than one problem per lane, targets met at q0, ilimit = slimit = 1 and a
   singular start.
e. Sub-chains and permuted jindex: q0 / q_out / limits are in chain order whatever the jindices.

Every chain asserts the kernel profile it takes (PROF 1 for dh_like chains, PROF 0 otherwise) through the restated host
flags of tests/fkj_ref.py.
"""
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import b2kin as rtb  # noqa: E402
from oracle import chains as ch  # noqa: E402
from oracle import oracle as orc  # noqa: E402

import fkj_ref as FR  # noqa: E402
import ik_lm_ref as R  # noqa: E402

AX = ["Rx", "Ry", "Rz", "tx", "ty", "tz"]
PARITY = 0.97  # the bar of the existing IK parity tests (test_gpu_parity.IK_COUNTER_PARITY)
CPP, PY = rtb._lib.SEM_CPP, rtb._lib.SEM_PYTHON
WEIGHTS = {"unit": None, "mask": np.array([1, 1, 1, 0, 0, 0.0]), "wts": np.array([1, 1, 1, 0.3, 0.3, 0.3])}
# rule -> (reference method, kernel method, lambda / damping)
RULES = {"chan": ("chan", "chan", 1.0), "wampler": ("wampler", "wampler", 0.05), "sugihara": ("sugihara", "sugihara", 0.05),
         "nr": ("nr", rtb._lib.IK_NR, 0.1), "nr0": ("nr", rtb._lib.IK_NR, 0.0), "gn": ("gn", rtb._lib.IK_GN, 0.0)}


def ets_of(desc):
    """A product ETS of a neutral chain description (joints keep the description's jindex and limits)."""
    ets = []
    for i in range(len(desc["isjoint"])):
        if desc["isjoint"][i]:
            ets.append(rtb.ET(AX[int(desc["axis"][i])], flip=bool(desc["flip"][i]), jindex=int(desc["jindex"][i]),
                              qlim=desc["qlim"][i]))
        else:
            ets.append(rtb.ET.SE3(desc["T"][i]))
    return rtb.ETS(ets)


def chain(n, prof, seed):
    rng = np.random.default_rng(seed)
    if prof == "dh":
        desc = FR.dh_family(n, rng)
    else:
        desc = FR.generic_family(n, rng, list(rng.permutation(FR.ALL_KINDS)))
    assert FR.compile_chain(desc)["dh_like"] == (prof == "dh"), (n, prof)
    return desc


def narrowed(desc, lo, hi):
    """The chain with its revolute joints limited to [lo, hi]."""
    d = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in desc.items()}
    for i in np.flatnonzero(d["isjoint"]):
        if d["axis"][i] < 3:
            d["qlim"][i] = (lo, hi)
    return d


def dev(a, dt=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).cuda()


def solve(e, Tep, q0, ilimit, slimit, rule, sem, dt=np.float64, mask=None, jl=False, seed=0, rng_per_row=True,
          tol=1e-6):
    """One b2k_ik_lm call through ETS._ik; (q, success, iterations, searches, residual) on the host."""
    _, code, lam = RULES[rule]
    r = e._ik(dev(Tep, dt), None if q0 is None else dev(q0, dt), ilimit, slimit, tol, mask, jl, lam, code, seed, sem,
              rng_per_row, None)
    torch.cuda.synchronize()
    return tuple(x.cpu().numpy() for x in r[:5])


def oracle(C, Tep, q0, ilimit, slimit, rule, sem, mask=None, jl=False, seed=0, rng_per_row=True, tol=1e-6):
    m, _, lam = RULES[rule]
    return C.ik_lm(Tep, q0, ilimit, slimit, tol, jl, mask, lam, m, seed=seed, semantics=sem, rng_per_row=rng_per_row)


def targets(C, N, rng, far=0.0):
    """(qt, Tep): in-limit configurations and their poses; a fraction `far` of the targets has its translation scaled
    by 10 (unreachable)."""
    lo, hi = C.qlim_l, C.qlim_h
    qt = lo + (hi - lo) * rng.uniform(0.05, 0.95, (N, C.n))
    Tep = C.fkine(qt)
    if far:
        sel = rng.random(N) < far
        Tep[sel, :3, 3] *= 10.0
    return qt, Tep


def same_all(a, b, rows=slice(None)):
    return all(np.array_equal(x[rows], y[rows]) for x, y in zip(a, b))


# ------------------------------------------------------------------ a. one step of every variant
STEP_ROWS = 257  # one full block of 256 lanes and a ragged one
SAMPLE = (0, 1, 2, 31, 32, 128, 254, 255, 256)


@pytest.mark.parametrize("n", range(1, 11))
def test_one_step_every_variant(n):
    """q_out - q0 against the 40-digit step and residual against E(q0), for both profiles, the six step rules and the
    three weightings, in fp64 and fp32.  The inputs are fp32-representable so one reference serves both precisions."""
    rng = np.random.default_rng(1000 + n)
    worst = {}
    for prof in ("dh", "gen"):
        desc = chain(n, prof, 10 * n + (prof == "gen"))
        e, C = ets_of(desc), orc.Chain(desc)
        qt, _ = targets(C, STEP_ROWS, rng)
        q0 = (qt + rng.normal(0.0, 0.25, qt.shape) * (C.qlim_h - C.qlim_l) / 4).astype(np.float32).astype(np.float64)
        Tep = C.fkine(qt).astype(np.float32).astype(np.float64)
        J = C.jacob0(q0)
        for wname, mask in WEIGHTS.items():
            we = np.ones(6) if mask is None else mask
            for rule, (m, _, lam) in RULES.items():
                ref = {r: R.step(C, q0[r], Tep[r], m, lam, we) for r in SAMPLE}
                for dt in (np.float64, np.float32):
                    q, s, it, sr, E = solve(e, Tep, q0, 1, 1, rule, PY, dt, mask=mask, tol=1e-30)
                    tag = f"n={n} {prof} {rule} {wname} {np.dtype(dt).name}"
                    assert (it == 1).all() and (sr == 1).all(), tag
                    assert (s == (E < 1e-30)).all(), tag  # only a row met at q0 (E = 0 under the mask) succeeds
                    dq = q.astype(np.float64) - q0
                    f64 = dt == np.float64
                    for r, (_, Er, dqr) in ref.items():
                        if s[r] or Er < 1e-12:  # E at the rounding level: the step is a ratio of two rounding errors
                            continue
                        # relative, plus the rounding of e itself (|e| eps) where E is tiny
                        bar = (1e-12 * Er + 1e-15 * np.sqrt(Er)) if f64 else (2e-3 * Er + 1e-6 * np.sqrt(Er))
                        assert abs(E[r] - Er) <= bar + 1e-300, (tag, r, E[r], Er)
                        c = R.cond(J[r], Er, m, lam, we)
                        if c < (1e6 if f64 else 1e3):
                            err = np.abs(dq[r] - dqr).max() / max(1.0, np.abs(dqr).max())
                            worst[np.dtype(dt).name] = max(worst.get(np.dtype(dt).name, 0.0), err)
                            assert err <= (1e-9 if f64 else 2e-3), (tag, r, f"cond {c:.1e}", dq[r], dqr)
    print(f"\nn={n}: worst step error / max(1, |dq|):", {k: f"{v:.1e}" for k, v in worst.items()})


# ------------------------------------------------------------------ b. the full loop against the sequential oracle
@pytest.mark.parametrize("n", [1, 3, 5, 6, 8, 10])
def test_full_loop_matches_sequential_oracle(n):
    rng = np.random.default_rng(2000 + n)
    for prof in ("dh", "gen"):
        desc = chain(n, prof, 20 * n + (prof == "gen"))
        e, C = ets_of(desc), orc.Chain(desc)
        _, Tep = targets(C, 300, rng)
        for sem in (CPP, PY):
            for jl in (True, False):
                for rule in ("chan", "wampler", "sugihara", "nr", "nr0", "gn"):
                    tag = f"n={n} {prof} sem={sem} jl={jl} {rule}"
                    want = oracle(C, Tep, None, 30, 8, rule, sem, jl=jl, seed=5)
                    q, s, it, sr, E = solve(e, Tep, None, 30, 8, rule, sem, jl=jl, seed=5)
                    if rule in ("nr0", "gn"):  # chaotic near singular configurations: outcome statistics only
                        assert abs(s.mean() - want[1].mean()) < 0.06, (tag, s.mean(), want[1].mean())
                    else:
                        # a row agrees when its counters and its q do: on redundant chains a trajectory that drifts
                        # apart at the rounding level (Cholesky here, LU / SVD in the oracle) can still end after the
                        # same number of iterations, on another point of the self-motion
                        same = (s == want[1]) & (it == want[2]) & (sr == want[3])
                        close = same & (np.abs(q - want[0]).max(axis=1) <= 1e-6)
                        assert close.mean() >= PARITY, (tag, same.mean(), close.mean())
                    ok = s == 1
                    assert (E[ok] < 1e-6).all(), tag
                    if sem == PY and rule in ("nr0", "gn"):
                        continue  # the Python loop returns q one undamped step past the tested one: no pose bound
                    # the C++ loop returns the q it tested (E < tol); the Python loop returns q after one more step,
                    # which near a singular configuration can move the pose by ~1e-2
                    reproduces(C, desc, q[ok], Tep[ok], 5e-2 if sem == PY else 5e-3, tag)


def reproduces(C, desc, q, Tep, bar, tag):
    """Every row of q reaches its target through the oracle's FK.  Both loops wrap every joint with fmod, prismatic ones
    included (as the reference does), so without joint limits a prismatic coordinate may come back shifted by a multiple
    of 2 pi: such a row must reproduce its target once that shift is undone."""
    err = np.abs(C.fkine(q) - Tep).reshape(len(q), -1).max(axis=1) if len(q) else np.zeros(0)
    pris = np.flatnonzero(desc["axis"][desc["isjoint"] == 1] >= 3)
    shifts = 2 * np.pi * np.array(list(itertools.product(range(-8, 9), repeat=len(pris))), dtype=np.float64)
    for r in np.flatnonzero(err >= bar):
        qq = np.repeat(q[r][None], len(shifts), axis=0)
        qq[:, pris] += shifts.reshape(len(shifts), len(pris))
        best = np.abs(C.fkine(qq) - Tep[r]).reshape(len(qq), -1).max(axis=1).min()
        assert best < bar, (tag, r, err[r], best)


# ------------------------------------------------------------------ c. the schedule changes no reported number
def hard_case(prof, N, seed):
    """A chain with narrowed limits and targets of which 40 % are unreachable: many rows use every search."""
    rng = np.random.default_rng(seed)
    if prof == "dh":
        desc = narrowed(ch.panda_ets(), -1.6, 1.6)
    else:
        desc = narrowed(chain(5, "gen", seed), -1.2, 1.2)
    assert FR.compile_chain(desc)["dh_like"] == (prof == "dh")
    C = orc.Chain(desc)
    _, Tep = targets(C, N, rng, far=0.4)
    return ets_of(desc), C, Tep


def check_hard_rows(C, Tep, got, ilimit, slimit, rule, sem, rows=128):
    """The first `rows` rows against the sequential oracle, failures included (C++: the last draw; Python: the last
    iterate, and the residual with it)."""
    want = oracle(C, Tep[:rows], None, ilimit, slimit, rule, sem, jl=True, seed=3)
    q, s, it, sr, E = (x[:rows] for x in got)
    same = (s == want[1]) & (it == want[2]) & (sr == want[3])
    close = same & (np.abs(q - want[0]).max(axis=1) <= 1e-6) & (np.abs(E - want[4]) <= 1e-6 * np.abs(want[4]) + 1e-9)
    assert close.mean() >= PARITY, (ilimit, slimit, rule, sem, same.mean(), close.mean())
    assert ((s == 0) & close).sum() >= rows // 5  # the unreachable rows are compared too


@pytest.mark.parametrize("prof", ["dh", "gen"])
def test_two_phase_equals_persistent_launch(prof):
    """Rows 0..1022 of a 1024-row batch (two phases) equal the same rows run as a 1023-row batch (one persistent
    launch), bit for bit in fp64."""
    e, C, Tep = hard_case(prof, 1024, 31)
    for sem in (CPP, PY):
        for rule in ("chan", "nr"):
            for dt in (np.float64, np.float32):
                a = solve(e, Tep, None, 30, 100, rule, sem, dt, jl=True, seed=3)
                b = solve(e, Tep[:1023], None, 30, 100, rule, sem, dt, jl=True, seed=3)
                check_same(a, b, slice(0, 1023), dt, (prof, sem, rule))
                if dt == np.float64 and rule == "chan":
                    check_hard_rows(C, Tep, a, 30, 100, rule, sem)


def check_same(a, b, rows, dt, tag):
    if dt == np.float64:
        assert same_all(a, b, rows), tag
    else:
        for k in (1, 2, 3):
            assert np.array_equal(a[k][rows], b[k][rows]), (tag, k)
        np.testing.assert_allclose(a[0][rows], b[0][rows], atol=1e-5, err_msg=str(tag))


def test_shared_draws_equal_chunked_batches():
    """rng_per_row = 0: every row draws the same restarts, so a 3000-row batch equals its rows run in chunks of at
    most 1023 (single persistent launches)."""
    e, C, Tep = hard_case("dh", 3000, 32)
    for sem in (CPP, PY):
        for dt in (np.float64, np.float32):
            a = solve(e, Tep, None, 20, 30, "chan", sem, dt, jl=True, seed=4, rng_per_row=False)
            for s0 in range(0, 3000, 1000):
                b = solve(e, Tep[s0:s0 + 1000], None, 20, 30, "chan", sem, dt, jl=True, seed=4, rng_per_row=False)
                check_same(tuple(x[s0:s0 + 1000] for x in a), b, slice(None), dt, (sem, s0))


@pytest.mark.parametrize("slimit", [2, 5, 6, 13, 14, 100])
def test_every_restart_round_shape(slimit):
    """ilimit 12 (first search in one launch) and 13 (split after 10 evaluations) with every shape of the restart
    rounds (8-lane groups only; 4 then 8; 4, one batch of 8, then 32), against the persistent launch and the oracle."""
    for prof in ("dh", "gen"):
        e, C, Tep = hard_case(prof, 1500, 33 + slimit)
        for ilimit in (12, 13):
            for sem in (CPP, PY):
                for dt in (np.float64, np.float32):
                    a = solve(e, Tep, None, ilimit, slimit, "chan", sem, dt, jl=True, seed=3)
                    b = solve(e, Tep[:1023], None, ilimit, slimit, "chan", sem, dt, jl=True, seed=3)
                    check_same(a, b, slice(0, 1023), dt, (prof, ilimit, slimit, sem))
                    if dt == np.float64:
                        check_hard_rows(C, Tep, a, ilimit, slimit, "chan", sem)


# ------------------------------------------------------------------ d. edge rows and sizes
def test_edge_batch_sizes():
    e = ets_of(ch.panda_ets())
    C = orc.Chain(ch.panda_ets())
    _, Tep = targets(C, 1025, np.random.default_rng(40), far=0.1)
    for sem in (CPP, PY):
        full = solve(e, Tep, None, 30, 5, "chan", sem, jl=True, seed=6)
        want = oracle(C, Tep, None, 30, 5, "chan", sem, jl=True, seed=6)
        same = (full[1] == want[1]) & (full[2] == want[2]) & (full[3] == want[3])
        assert same.mean() >= PARITY, (sem, same.mean())
        np.testing.assert_allclose(full[0][same], want[0][same], atol=1e-6)
        for N in (0, 1, 31, 32, 33, 127, 128, 129, 1023, 1024):
            got = solve(e, Tep[:N], None, 30, 5, "chan", sem, jl=True, seed=6)
            assert all(len(x) == N for x in got)
            assert same_all(got, full, slice(0, N)), (sem, N)


def test_persistent_grid_pulls_many_problems_per_lane():
    """slimit = 1 and 100 001 rows: about two problems per resident lane (132 SMs x 3 blocks x 128 lanes in fp64 on an
    H100 SXM).  With shared draws the last 2000 rows equal the
    same rows run alone, and the oracle."""
    e = ets_of(ch.panda_ets())
    C = orc.Chain(ch.panda_ets())
    _, Tep = targets(C, 100001, np.random.default_rng(41))
    for sem in (CPP, PY):
        big = solve(e, Tep, None, 30, 1, "chan", sem, seed=8, rng_per_row=False)
        assert set(np.unique(big[1])) <= {0, 1} and (big[2] >= 1).all() and big[1].mean() > 0.5
        tail = solve(e, Tep[-2000:], None, 30, 1, "chan", sem, seed=8, rng_per_row=False)
        assert same_all(tail, tuple(x[-2000:] for x in big)), sem
        want = oracle(C, Tep[-2000:], None, 30, 1, "chan", sem, seed=8, rng_per_row=False)
        same = (tail[1] == want[1]) & (tail[2] == want[2]) & (tail[3] == want[3])
        assert same.mean() >= PARITY, (sem, same.mean())


def test_target_met_at_q0_and_single_iteration():
    e = ets_of(ch.panda_ets())
    C = orc.Chain(ch.panda_ets())
    qt, Tep = targets(C, 200, np.random.default_rng(42))
    for rule in ("chan", "sugihara", "nr", "gn"):
        # met at q0: the C++ loop tests before stepping (1 iteration, q0 wrapped), the Python loop steps once first --
        # which for chan (wn = lambda E ~ 0) and undamped GN solves a singular system on this 7-joint arm: the kernel
        # abandons such a search, so those two are left to the C++ loop
        for sem in ((CPP, PY) if rule in ("sugihara", "nr") else (CPP,)):
            q, s, it, sr, E = solve(e, Tep, qt, 30, 3, rule, sem)
            want = oracle(C, Tep, qt, 30, 3, rule, sem)
            assert (s == 1).all() and (it == 1).all() and (sr == 1).all(), (rule, sem)
            for k in (1, 2, 3):
                assert np.array_equal((s, it, sr)[k - 1], want[k])
            np.testing.assert_allclose(q, want[0], atol=1e-12)
            np.testing.assert_allclose(E, want[4], rtol=0, atol=1e-24)
            if sem == CPP:
                np.testing.assert_allclose(q, qt, atol=1e-12)
        # ilimit = slimit = 1 from random starts
        for sem in (CPP, PY):
            got = solve(e, Tep, None, 1, 1, rule, sem, seed=9)
            want = oracle(C, Tep, None, 1, 1, rule, sem, seed=9)
            for k in (1, 2, 3):
                assert np.array_equal(got[k], want[k]), (rule, sem, k)
            np.testing.assert_allclose(got[0], want[0], atol=1e-9)
            np.testing.assert_allclose(got[4], want[4], rtol=1e-12)


def test_singular_start_undamped_gn():
    """Panda at q = 0 has two aligned joint axes: J J^T is singular.  Undamped GN from there either abandons the search
    (q stays q0 under Python semantics) or, where rounding leaves a positive pivot, takes a finite step; it never
    reports success in one iteration and the counters are those of one spent search."""
    e = ets_of(ch.panda_ets())
    C = orc.Chain(ch.panda_ets())
    _, Tep = targets(C, 64, np.random.default_rng(43))
    q0 = np.zeros((64, 7))
    q, s, it, sr, E = solve(e, Tep, q0, 1, 1, "gn", PY, tol=1e-30)
    assert (s == 0).all() and (it == 1).all() and (sr == 1).all()
    abandoned = (q == 0).all(axis=1)
    print(f"\nPanda at q = 0, undamped GN: {abandoned.mean():.2f} of the rows abandoned the search")
    assert abandoned.all(), abandoned.mean()
    # the C++ loop counts its first search from 1 and leaves a fresh draw in q when the searches run out
    q, s, it, sr, E = solve(e, Tep, q0, 1, 1, "gn", CPP, tol=1e-30)
    assert (s == 0).all() and (it == 2).all() and (sr == 2).all()
    np.testing.assert_allclose(q, np.stack([R.rand_q(C.qlim_l, C.qlim_h, 0, r, 1) for r in range(64)]), atol=1e-14)


# ------------------------------------------------------------------ e. sub-chains and permuted jindex
def dense(desc):
    d = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in desc.items()}
    d["jindex"][np.flatnonzero(d["isjoint"])] = np.arange(int(d["isjoint"].sum()), dtype=np.int32)
    return d


def test_sub_chains_and_permuted_jindex():
    panda = rtb.models.Panda()
    L = panda.links
    sub = panda.ets(start=L[4], end=L[-1])
    assert list(sub.jindices) == [4, 5, 6]
    rng = np.random.default_rng(44)
    gen = chain(6, "gen", 44)
    cases = [("panda[4:]", sub, sub.describe()), ("permuted", ets_of(FR.with_jindex(gen, rng.permutation(6))), gen)]
    for name, e, desc in cases:
        dd = dense(desc)
        ed, C = ets_of(dd), orc.Chain(dd)
        _, Tep = targets(C, 1100, rng)
        jind = e.jindices
        for sem in (CPP, PY):
            for rule in ("chan", "nr", "gn"):
                for N in (300, 1100):  # one persistent launch / two phases
                    a = solve(e, Tep[:N], None, 30, 10, rule, sem, jl=True, seed=12)
                    b = solve(ed, Tep[:N], None, 30, 10, rule, sem, jl=True, seed=12)
                    assert same_all(a, b), (name, sem, rule, N)
                want = oracle(C, Tep[:300], None, 30, 10, rule, sem, jl=True, seed=12)
                q, s = a[0][:300], a[1][:300]
                if rule != "gn":
                    same = (s == want[1]) & (a[2][:300] == want[2]) & (a[3][:300] == want[3])
                    assert same.mean() >= PARITY, (name, sem, rule, same.mean())
                    np.testing.assert_allclose(q[same], want[0][same], atol=1e-6)
                ok = s == 1
                Q = np.zeros((ok.sum(), int(jind.max()) + 1))
                Q[:, jind] = q[ok]
                bar = 5e-3 if sem == CPP else 5e-2
                assert np.abs(e.eval(Q) - Tep[:300][ok]).max() < bar, (name, sem, rule)
