#!/usr/bin/env python3
"""Device-timed micro-benchmarks of every hot-path kernel (one JSON line per case).

Each case: W warm-up launches, then K launches bracketed by CUDA events on the launching stream;
inputs rotate over enough distinct batches to exceed the 50 MB L2.  `frac` is algorithmic bytes
(SURVEY 8d) / time / MEASURED_PEAKS hbm_gbs.  Usage:  python scripts/kernel_bench.py [--rows 1000000] [--only substr]
"""
import argparse
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import b2kin as rtb  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1_000_000)
ap.add_argument("--ik-rows", type=int, default=100_000)
ap.add_argument("--steps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=10)
ap.add_argument("--only", default="")
args = ap.parse_args()
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    PEAK = 3350.0  # H100 SXM data sheet
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)


def timeit(fn, nbuf):
    for i in range(args.warmup):
        fn(i % nbuf)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        fn(i % nbuf)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps


def report(name, ms, rows, bytes_per_row, extra=None):
    gbs = bytes_per_row * rows / (ms * 1e-3) / 1e9
    d = {"case": name, "rows": rows, "ms": round(ms, 5), "rows_per_s": rows / (ms * 1e-3), "GBps": round(gbs, 1),
         "frac_of_hbm": round(gbs / PEAK, 4), "bytes_per_row": bytes_per_row}
    if extra:
        d.update(extra)
    print(json.dumps(d), flush=True)


def want(name):
    # `name` is a case name or the prefix of a block of cases ("ik_", "dyn_", "probe_")
    return args.only in name or (name.endswith("_") and args.only.startswith(name))


N = args.rows
rng = np.random.default_rng(0)
if want("probe_"):
    # context only (torch library kernels, not part of the product): what this box's HBM does for a
    # pure-write stream and for a copy of the same footprint as the headline step
    buf = torch.empty(520_000_000 // 8, dtype=torch.float64, device=dev)
    src = torch.empty(260_000_000 // 8, dtype=torch.float64, device=dev)
    report("probe_fill_520MB", timeit(lambda i: buf.fill_(1.0), 1), 1, 520_000_000)
    report("probe_copy_260MB_to_260MB", timeit(lambda i: buf[: src.numel()].copy_(src), 1), 1, 520_000_000)
    del buf, src
tdt = {np.float32: torch.float32, np.float64: torch.float64}

for robot_name, robot in (("panda", rtb.models.Panda()), ("ur10", rtb.models.UR10())):
    ets = robot.ets()
    n = ets.n
    for dt in (np.float64, np.float32):
        es = np.dtype(dt).itemsize
        tag = f"{robot_name}_{'f64' if dt == np.float64 else 'f32'}"
        nbuf = max(2, int(np.ceil(300e6 / (N * n * es))))
        nbuf = min(nbuf, 8)
        qs = [torch.from_numpy(rng.uniform(-np.pi, np.pi, (N, n)).astype(dt)).to(dev) for _ in range(nbuf)]
        T = torch.empty((N, 4, 4), dtype=tdt[dt], device=dev)
        J = torch.empty((N, 6, n), dtype=tdt[dt], device=dev)
        L = rtb._lib.lib()
        ch = ets._chain
        st = torch.cuda.current_stream().cuda_stream
        code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
        if want(f"fkine_{tag}"):
            report(f"fkine_{tag}", timeit(lambda i: L.b2k_fkine(ch, code, qs[i].data_ptr(), N, n, None, None, T.data_ptr(), st), nbuf), N, (n + 16) * es)
        if want(f"fkine_jacob0_{tag}"):
            report(f"fkine_jacob0_{tag}", timeit(lambda i: L.b2k_fkine_jacob0(ch, code, qs[i].data_ptr(), N, n, None, None, T.data_ptr(), J.data_ptr(), st), nbuf), N, (n + 16 + 6 * n) * es)
        if want(f"jacob0_{tag}") and robot_name == "panda":
            report(f"jacob0_{tag}", timeit(lambda i: L.b2k_jacob0(ch, code, qs[i].data_ptr(), N, n, None, J.data_ptr(), st), nbuf), N, (n + 6 * n) * es)
        if want(f"jacobe_{tag}") and robot_name == "panda":
            report(f"jacobe_{tag}", timeit(lambda i: L.b2k_jacobe(ch, code, qs[i].data_ptr(), N, n, None, J.data_ptr(), st), nbuf), N, (n + 6 * n) * es)
        del qs, T, J

# The general kernels (k_fkj_forward / k_fkj_backward), which the cases above do not reach: Panda with q rows one wider
# than the chain (the DH-like profile), and a 7-joint chain with Rx / Ry / prismatic joints (the generic profile).
E = rtb.ET
gen7 = rtb.ETS([E.tz(0.3), E.Rx(), E.ty(0.1), E.Ry(), E.tz(), E.tx(0.2), E.Rz(), E.Ry(), E.tx(), E.tz(0.1), E.Rx(),
                E.tx(0.05)])
rngg = np.random.default_rng(1)
for fam, ets, ldq in (("panda_ldq8", rtb.models.Panda().ets(), 8), ("generic7", gen7, 7)):
    n = ets.n
    for dt in (np.float64, np.float32):
        es = np.dtype(dt).itemsize
        tag = f"{fam}_{'f64' if dt == np.float64 else 'f32'}"
        if not (want(f"fkine_jacob0_{tag}") or want(f"jacobe_{tag}")):
            continue
        nbuf = min(8, max(2, int(np.ceil(300e6 / (N * ldq * es)))))
        qs = [torch.from_numpy(rngg.uniform(-np.pi, np.pi, (N, ldq)).astype(dt)).to(dev) for _ in range(nbuf)]
        T = torch.empty((N, 4, 4), dtype=tdt[dt], device=dev)
        J = torch.empty((N, 6, n), dtype=tdt[dt], device=dev)
        L = rtb._lib.lib()
        ch = ets._chain
        st = torch.cuda.current_stream().cuda_stream
        code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
        if want(f"fkine_jacob0_{tag}"):
            report(f"fkine_jacob0_{tag}", timeit(lambda i: rtb._lib.check(L.b2k_fkine_jacob0(ch, code, qs[i].data_ptr(), N, ldq, None, None, T.data_ptr(), J.data_ptr(), st)), nbuf),
                   N, (ldq + 16 + 6 * n) * es)
        if want(f"jacobe_{tag}"):
            report(f"jacobe_{tag}", timeit(lambda i: rtb._lib.check(L.b2k_jacobe(ch, code, qs[i].data_ptr(), N, ldq, None, J.data_ptr(), st)), nbuf),
                   N, (ldq + 6 * n) * es)
        del qs, T, J

puma = rtb.models.Puma560()
for dt in (np.float64, np.float32):
    tag = "f64" if dt == np.float64 else "f32"
    if not want(f"rne_puma_{tag}"):
        continue
    es = np.dtype(dt).itemsize
    nbuf = 3
    ql = puma.qlim
    bufs = [tuple(torch.from_numpy(a.astype(dt)).to(dev) for a in (rng.uniform(ql[0], ql[1], (N, 6)), rng.normal(size=(N, 6)), rng.normal(size=(N, 6)))) for _ in range(nbuf)]
    tau = torch.empty((N, 6), dtype=tdt[dt], device=dev)
    puma.rne(*bufs[0])  # builds the handle
    L = rtb._lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
    g = np.ascontiguousarray(-puma.gravity)
    for variant, setting in (("", "1"), ("_generic", "0")):  # robot-specialised (NVRTC) kernel vs the pre-compiled generic one
        if variant and not want(f"rne_puma_{tag}{variant}"):
            continue
        os.environ["B2K_RNE_SPEC"] = setting
        report(f"rne_puma_{tag}{variant}", timeit(lambda i: L.b2k_rne(puma._rne_ob, code, bufs[i][0].data_ptr(), bufs[i][1].data_ptr(), bufs[i][2].data_ptr(), N, rtb._lib.dptr(g), None, tau.data_ptr(), st), nbuf), N, 24 * es,
               {"kernel": rtb.rne_kernel_info(puma, "rne", dt)})
    os.environ["B2K_RNE_SPEC"] = "1"
    del bufs, tau

# rne with the base wrench (DHRobot.rne(base_wrench=True)): tau (N,6) and wbase (N,6) from one recursion; bytes per row
# = sizeof(real) (4n + 6), against 4n for plain rne
for dt in (np.float64, np.float32):
    tag = "f64" if dt == np.float64 else "f32"
    if not want(f"rne_wrench_puma_{tag}"):
        continue
    es = np.dtype(dt).itemsize
    nbuf = 3
    ql = puma.qlim
    bufs = [tuple(torch.from_numpy(a.astype(dt)).to(dev) for a in (rng.uniform(ql[0], ql[1], (N, 6)), rng.normal(size=(N, 6)), rng.normal(size=(N, 6)))) for _ in range(nbuf)]
    tau = torch.empty((N, 6), dtype=tdt[dt], device=dev)
    wb = torch.empty((N, 6), dtype=tdt[dt], device=dev)
    puma.rne(*bufs[0])
    L = rtb._lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
    g = np.ascontiguousarray(-puma.gravity)
    for variant, setting in (("", "1"), ("_generic", "0")):
        if variant and not want(f"rne_wrench_puma_{tag}{variant}"):
            continue
        os.environ["B2K_RNE_SPEC"] = setting
        report(f"rne_wrench_puma_{tag}{variant}", timeit(lambda i: L.b2k_rne_wrench(puma._rne_ob, code, bufs[i][0].data_ptr(), bufs[i][1].data_ptr(), bufs[i][2].data_ptr(), N, rtb._lib.dptr(g), None, tau.data_ptr(), wb.data_ptr(), st), nbuf), N, (4 * 6 + 6) * es,
               {"kernel": puma.rne_kernel_info("rne_wrench", dt)})
    os.environ["B2K_RNE_SPEC"] = "1"
    del bufs, tau, wb

# static forces (csrc/b2k_static.cu): one chain walk per row.  Algorithmic bytes per row, sizeof(real) = es:
#   static_gravjac_puma             q (n) in; tau (n) and J0 (6n) out                       = 8n es
#   static_gravload_plus_jacob0     the two launches gravjac replaces: q read by each       = 9n es
#   static_pay_panda                q (n) in, tau (n) out, one wrench for every row         = 2n es
#   static_paycap_puma              q (n) and w (6) in; wmax (n) and joint (4 B) out        = (2n + 6) es + 4
for dt in (np.float64, np.float32):
    tag = "f64" if dt == np.float64 else "f32"
    if not want(f"static_{tag}") and not any(want(f"static_{c}_{tag}") for c in ("gravjac_puma", "gravload_plus_jacob0_puma", "pay_panda", "paycap_puma")):
        continue
    es = np.dtype(dt).itemsize
    code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
    L = rtb._lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    nbuf = 3
    ql = puma.qlim
    qs = [torch.from_numpy(rng.uniform(ql[0], ql[1], (N, 6)).astype(dt)).to(dev) for _ in range(nbuf)]
    tau = torch.empty((N, 6), dtype=tdt[dt], device=dev)
    J = torch.empty((N, 6, 6), dtype=tdt[dt], device=dev)
    pch, mass = puma.ets()._chain, puma._static_mass_table()
    g = np.ascontiguousarray(puma.gravity)
    ng = np.ascontiguousarray(-puma.gravity)
    puma.gravload(qs[0][:64])  # builds the RNE handle (and the specialised kernel)
    if want(f"static_gravjac_puma_{tag}"):
        report(f"static_gravjac_puma_{tag}", timeit(lambda i: L.b2k_gravjac(pch, code, qs[i].data_ptr(), N, 6, rtb._lib.dptr(mass), rtb._lib.dptr(g), tau.data_ptr(), J.data_ptr(), st), nbuf), N, 8 * 6 * es)
    if want(f"static_gravload_plus_jacob0_puma_{tag}"):
        def two(i):
            L.b2k_rne_gravload(puma._rne_ob, code, qs[i].data_ptr(), N, rtb._lib.dptr(ng), tau.data_ptr(), st)
            L.b2k_jacob0(pch, code, qs[i].data_ptr(), N, 6, None, J.data_ptr(), st)
        report(f"static_gravload_plus_jacob0_puma_{tag}", timeit(two, nbuf), N, 9 * 6 * es, {"gravload_kernel": puma.rne_kernel_info("gravload", dt)})
    if want(f"static_paycap_puma_{tag}"):
        tauR = np.ascontiguousarray(np.tile([[100.0, -100.0]], (6, 1)))
        w = torch.tensor([0.0, 0.0, -1.0, 0.0, 0.0, 0.0], dtype=tdt[dt], device=dev)
        jt = torch.empty((N,), dtype=torch.int32, device=dev)
        report(f"static_paycap_puma_{tag}", timeit(lambda i: L.b2k_paycap(pch, code, qs[i].data_ptr(), N, 6, rtb._lib.dptr(mass), rtb._lib.dptr(g), w.data_ptr(), 0, 1, rtb._lib.dptr(tauR), tau.data_ptr(), jt.data_ptr(), st), nbuf), N, (2 * 6 + 6) * es + 4)
    del qs, tau, J
    if want(f"static_pay_panda_{tag}"):
        pe = rtb.models.Panda().ets()
        n = pe.n
        qs = [torch.from_numpy(rng.uniform(-np.pi, np.pi, (N, n)).astype(dt)).to(dev) for _ in range(nbuf)]
        tau = torch.empty((N, n), dtype=tdt[dt], device=dev)
        W = torch.tensor([1.0, -2.0, 3.0, 0.1, 0.2, -0.3], dtype=tdt[dt], device=dev)
        report(f"static_pay_panda_{tag}", timeit(lambda i: L.b2k_pay(pe._chain, code, qs[i].data_ptr(), N, n, W.data_ptr(), 0, 1, tau.data_ptr(), st), nbuf), N, 2 * n * es)
        del qs, tau

# dynamics fan-outs over the RNE recursion (SURVEY 8f-1): Puma560, fp64
if want("dyn_"):
    Nd = max(1, N // 4)
    ql = puma.qlim
    qd_ = torch.from_numpy(rng.uniform(ql[0], ql[1], (Nd, 6))).to(dev)
    v_ = torch.from_numpy(rng.normal(size=(Nd, 6))).to(dev)
    t_ = torch.from_numpy(rng.normal(size=(Nd, 6))).to(dev)
    puma.rne(qd_[:4], v_[:4], v_[:4])
    L = rtb._lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    g = np.ascontiguousarray(-puma.gravity)
    Mo = torch.empty((Nd, 6, 6), dtype=torch.float64, device=dev)
    vo = torch.empty((Nd, 6), dtype=torch.float64, device=dev)
    F = rtb._lib.F64
    h = puma._rne_ob
    cases = [
        ("dyn_inertia_puma_f64", lambda i: L.b2k_rne_inertia(h, F, qd_.data_ptr(), Nd, Mo.data_ptr(), st), (6 + 36) * 8, 6),
        ("dyn_gravload_puma_f64", lambda i: L.b2k_rne_gravload(h, F, qd_.data_ptr(), Nd, rtb._lib.dptr(g), vo.data_ptr(), st), 12 * 8, 1),
        ("dyn_itorque_puma_f64", lambda i: L.b2k_rne_itorque(h, F, qd_.data_ptr(), v_.data_ptr(), Nd, vo.data_ptr(), st), 18 * 8, 1),
        ("dyn_coriolis_puma_f64", lambda i: L.b2k_rne_coriolis(h, F, qd_.data_ptr(), v_.data_ptr(), Nd, Mo.data_ptr(), st), (12 + 36) * 8, 21),
        ("dyn_accel_puma_f64", lambda i: L.b2k_rne_accel(h, F, qd_.data_ptr(), v_.data_ptr(), t_.data_ptr(), Nd, rtb._lib.dptr(g), vo.data_ptr(), st), 24 * 8, 7),
    ]
    for name, fn, bpr, nrec in cases:
        for variant, setting in (("", "1"), ("_generic", "0")):
            if want(name + variant) and (not variant or args.only == "" or "generic" in args.only or args.only.startswith("dyn_")):
                os.environ["B2K_RNE_SPEC"] = setting
                ms = timeit(fn, 1)
                report(name + variant, ms, Nd, bpr, {"recursions_per_row": nrec, "recursions_per_s": nrec * Nd / (ms * 1e-3),
                                                     "kernel": rtb.rne_kernel_info(puma, name.split("_")[1], np.float64)})
    os.environ["B2K_RNE_SPEC"] = "1"

# Robot.rne on a rigid-body tree (generated Featherstone recursion): the Puma560 assembled as an ETS robot from its DH table
if want("tree_"):
    ET, ETS, Link = rtb.ET, rtb.ETS, rtb.Link
    links, prev = [], ETS()
    for j, l in enumerate(puma.links):
        post = ETS()
        for kind, v in (("tz", l.d), ("tx", l.a), ("Rx", l.alpha)):
            if v != 0:
                post = post * getattr(ET, kind)(v)
        Tp = np.eye(4)
        for et in post:
            Tp = Tp @ et.A()
        links.append(Link(prev * ET.Rz(), name=f"l{j}", parent=links[-1] if links else None, m=l.m, r=Tp[:3, :3] @ l.r + Tp[:3, 3]))
        prev = post
    links.append(Link(prev, name="tool", parent=links[-1]))
    trob = rtb.Robot(links)
    for dt in (np.float64, np.float32):
        tag = "f64" if dt == np.float64 else "f32"
        if not want(f"tree_rne_puma_{tag}"):
            continue
        es = np.dtype(dt).itemsize
        bufs = [tuple(torch.from_numpy(a.astype(dt)).to(dev) for a in (rng.uniform(-3, 3, (N, 6)), rng.normal(size=(N, 6)), rng.normal(size=(N, 6)))) for _ in range(3)]
        tau = torch.empty((N, 6), dtype=tdt[dt], device=dev)
        h = trob._tree_handle()
        L = rtb._lib.lib()
        st = torch.cuda.current_stream().cuda_stream
        code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
        ag = np.ascontiguousarray(-trob.gravity)
        report(f"tree_rne_puma_{tag}", timeit(lambda i: L.b2k_tree_rne(h, code, bufs[i][0].data_ptr(), bufs[i][1].data_ptr(), bufs[i][2].data_ptr(), N, rtb._lib.dptr(ag), tau.data_ptr(), st), 3), N, 24 * es,
               {"kernel": trob.rne_kernel_info(dt)})
        if dt == np.float64:  # the DynamicsMixin operations of the same tree robot, 250k rows (like the dyn_ block)
            Nd = 250_000
            for op, nin, nout, recs in (("inertia", 1, 36, 6), ("coriolis", 2, 36, 21), ("accel", 3, 6, 7)):
                if not want(f"tree_{op}_puma_f64"):
                    continue
                out = torch.empty((Nd, nout), dtype=tdt[dt], device=dev)
                ptr = [bufs[0][i].data_ptr() if i < nin else None for i in range(3)]
                opc = trob._DYN_OPS[op]
                report(f"tree_{op}_puma_f64", timeit(lambda i: L.b2k_tree_dyn(h, opc, code, ptr[0], ptr[1], ptr[2], Nd, rtb._lib.dptr(ag), out.data_ptr(), st), 3),
                       Nd, (6 * nin + nout) * es, {"recursions_per_row": recs, "kernel": trob.rne_kernel_info(dt, op=op)})
                del out
        del bufs, tau
    # Exact derivatives of the same tree (generated tangent recursion, b2k_tree_derivatives), N rows.  Algorithmic bytes
    # per row: rne_derivatives (3n + 2n^2) es, accel_derivatives (3n + 3n^2) es.  fd_route is what a user has without
    # them, timed in the same call on the same rows: one-sided differences, 2n + 1 b2k_tree_rne launches (inverse mode) and
    # 3n + 1 b2k_tree_dyn(ACCEL) launches (forward mode: the base point and one perturbation of each q, qd, torque entry).
    # The card's name and power limit are read in the same run.
    TD_CASES = [f"tree_{op}_derivs_puma_{t}" for op in ("rne", "accel") for t in ("f64", "f32")]
    if any(want(c) for c in TD_CASES):
        import subprocess

        try:
            plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                                  text=True, timeout=30).stdout.strip()
        except Exception as e:  # the figure is context, the timing does not depend on it
            plim = f"unavailable ({type(e).__name__})"
        card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
        L = rtb._lib.lib()
        h = trob._tree_handle()
        st = torch.cuda.current_stream().cuda_stream
        ag = np.ascontiguousarray(-trob.gravity)
        n = 6
        rngt = np.random.default_rng(14)
        for dt in (np.float64, np.float32):
            tag = "f64" if dt == np.float64 else "f32"
            c_rne, c_acc = f"tree_rne_derivs_puma_{tag}", f"tree_accel_derivs_puma_{tag}"
            if not (want(c_rne) or want(c_acc)):
                continue
            es = np.dtype(dt).itemsize
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            tt = torch.float64 if dt == np.float64 else torch.float32
            q0, qd0, x0 = (torch.from_numpy(rngt.uniform(-2, 2, (N, n)).astype(dt)).to(dev) for _ in range(3))
            o = [torch.empty((N, n, n), dtype=tt, device=dev) for _ in range(3)]
            hstep = 1e-6 if dt == np.float64 else 1e-2
            for case, op, npert in ((c_rne, 7, 2), (c_acc, 8, 3)):
                if not want(case):
                    continue
                pert = []
                for k in range(n):
                    e = torch.zeros(n, dtype=tt, device=dev)
                    e[k] = hstep
                    pert += [(q0 + e, qd0, x0), (q0, qd0 + e, x0)] + ([(q0, qd0, x0 + e)] if npert == 3 else [])
                pert.append((q0, qd0, x0))
                outs = [torch.empty((N, n), dtype=tt, device=dev) for _ in pert]

                def fd_route(i, op=op, pert=pert, outs=outs):
                    for (a, b, c), t in zip(pert, outs):
                        if op == 7:
                            rtb._lib.check(L.b2k_tree_rne(h, code, a.data_ptr(), b.data_ptr(), c.data_ptr(), N, rtb._lib.dptr(ag), t.data_ptr(), st))
                        else:
                            rtb._lib.check(L.b2k_tree_dyn(h, 5, code, a.data_ptr(), b.data_ptr(), c.data_ptr(), N, rtb._lib.dptr(ag), t.data_ptr(), st))

                # alternate the two routes, so that both see the same clocks
                ms_fd, ms = [], []
                for _ in range(2):
                    ms_fd.append(timeit(fd_route, 1))
                    ms.append(timeit(lambda i, op=op: rtb._lib.check(L.b2k_tree_derivatives(
                        h, op, code, q0.data_ptr(), qd0.data_ptr(), x0.data_ptr(), N, rtb._lib.dptr(ag), o[0].data_ptr(), o[1].data_ptr(),
                        o[2].data_ptr() if op == 8 else None, st)), 1))
                ms_fd, ms = min(ms_fd), min(ms)
                report(case, ms, N, (3 * n + npert * n * n) * es,
                       dict(card, frac_of_3p35TBps=round((3 * n + npert * n * n) * es * N / (ms * 1e-3) / 3.35e12, 4), fd_route_ms=round(ms_fd, 4), fd_route_launches=len(pert), speedup_vs_fd_route=round(ms_fd / ms, 2),
                            kernel=trob.rne_kernel_info(dt, op="rne_derivatives" if op == 7 else "accel_derivatives")))
                del pert, outs
            del q0, qd0, x0, o

# forward-dynamics ensemble: friction-free Puma falling from qn for 0.5 s, rtol 1e-6, one lane per trajectory
if want("fdyn_"):
    nf = puma.nofriction()
    for B_ in (1024, 16384):
        if not want(f"fdyn_puma_f64_ens{B_}"):
            continue
        Q0 = torch.from_numpy(nf.qn + rng.uniform(-0.3, 0.3, (B_, 6))).to(dev)
        nf.fdyn(0.05, Q0[:64], dt=0.01)  # builds the kernel
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = nf.fdyn(0.5, Q0, solver_args=dict(rtol=1e-6, atol=1e-9), dt=0.01)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        print(json.dumps({"case": f"fdyn_puma_f64_ens{B_}", "trajectories": B_, "T": 0.5, "rtol": 1e-6, "ms": round(ms, 3),
                          "trajectory_seconds_per_s": B_ * 0.5 / (ms * 1e-3), "grid_samples": int(out.q.shape[1])}), flush=True)

# The widened rows (SURVEY 8f-2 / f-3) through the public API -- the call a user makes, Python dispatch included (tens of
# microseconds per call, visible only on the shortest ones).  Bytes per row = what the operation must read and write.
if want("extra_"):
    NX = args.rows
    rngx = np.random.default_rng(4)
    pe = rtb.models.Panda().ets()
    Qx = torch.from_numpy(rngx.uniform(-2.5, 2.5, (NX, 7))).to(dev)
    QDx = torch.from_numpy(rngx.normal(size=(NX, 7))).to(dev)
    Jx = pe.jacob0(Qx)
    Tx = pe.eval(Qx)
    Ty = pe.eval(torch.roll(Qx, 1, 0))
    cases = [
        ("extra_hessian0_from_J_f64", lambda i: pe.hessian0(J0=Jx), (42 + 294) * 8),
        ("extra_yoshikawa_from_J_f64", lambda i: pe.manipulability(J=Jx), (42 + 1) * 8),
        ("extra_minsingular_from_J_f64", lambda i: pe.manipulability(J=Jx, method="minsingular"), (42 + 1) * 8),
        ("extra_jacobm_from_J_f64", lambda i: pe.jacobm(J=Jx), (42 + 7) * 8),
        ("extra_jacob0_dot_f64", lambda i: pe.jacob0_dot(qd=QDx, J0=Jx), (42 + 7 + 42) * 8),
        ("extra_jacob0_analytical_rpy_f64", lambda i: pe.jacob0_analytical(Qx), (7 + 42) * 8),
        ("extra_jacob0_analytical_exp_f64", lambda i: pe.jacob0_analytical(Qx, representation="exp"), (7 + 42) * 8),
        ("extra_angle_axis_f64", lambda i: rtb.angle_axis(Tx, Ty), (32 + 6) * 8),
        ("extra_p_servo_rpy_f64", lambda i: rtb.p_servo(Tx, Ty), (32 + 6) * 8 + 1),
        ("extra_jtraj_f64", lambda i: rtb.jtraj(np.zeros(7), np.ones(7), NX, device=True), 21 * 8),
        ("extra_mtraj_trapezoidal_f64", lambda i: rtb.mtraj(rtb.trapezoidal, np.zeros(7), np.ones(7), NX, device=True), 21 * 8),
        ("extra_ctraj_f64", lambda i: rtb.ctraj(Tx[0].cpu().numpy(), Tx[1].cpu().numpy(), NX, device=True), 16 * 8),
        ("extra_fkine_all_panda_f64", lambda i: PD.fkine_all(Qx), (7 + 8 * 16) * 8),
    ]
    PD = rtb.models.DH.Panda()

    for name, fn, bpr in cases:
        if not want(name):
            continue
        try:
            ms = timeit(fn, 1)
            report(name, ms, NX, bpr, {"api": "public Python call on device-resident inputs"})
        except Exception as e:  # keep the table going
            print(json.dumps({"case": name, "error": f"{type(e).__name__}: {e}"[:300]}), flush=True)
    del Qx, QDx, Jx, Tx, Ty

# partial_fkine0 of a given Panda jacob0 (b2k_pfk.cu) through the public call: 131 072 rows is 2.2 GB (order 3) to 15 GB
# (order 4) of fp64 output per call, a steady store stream.  Bytes per row = J read + D written, sizeof(real) (6n + 6n^k).
if want("extra_partial_fkine0_"):
    NP = 131_072
    pe = rtb.models.Panda().ets()
    Jp = pe.jacob0(torch.from_numpy(np.random.default_rng(7).uniform(-2.5, 2.5, (NP, 7))).to(dev))
    for k in (3, 4):
        for dt, sz in ((torch.float64, 8), (torch.float32, 4)):
            name = f"extra_partial_fkine0_o{k}_panda_f{8 * sz}"
            if not want(name):
                continue
            Jk = Jp.to(dt)
            ms = timeit(lambda i: pe.partial_fkine0(J0=Jk, n=k), 1)
            report(name, ms, NP, sz * (42 + 6 * 7 ** k), {"api": "public Python call on a device-resident J"})
    del Jp

# Operational-space dynamics (b2k_opspace): the epilogue alone over staged joint-space inputs -- inverse (Puma560) and
# Jacobi pseudo-inverse (PandaMDH, n = 7) -- and the whole coriolis_x pipeline through the public call.  Bytes per row =
# the arrays the epilogue must read and write.
if want("opspace_"):
    NO = args.rows
    rngo = np.random.default_rng(6)
    Lo = rtb._lib.lib()
    sto = torch.cuda.current_stream().cuda_stream
    for tag, rob, kind in (("puma_inv", rtb.models.Puma560(), rtb._lib.OPS_INV), ("pandamdh_pinv", rtb.models.PandaMDH(), rtb._lib.OPS_PINV)):
        n = rob.n
        qo = torch.from_numpy(rngo.uniform(-2, 2, (NO, n))).to(dev)
        qdo = torch.from_numpy(rngo.normal(size=(NO, n))).to(dev)
        Ja, M, Cm, G = rob.jacob0_analytical(qo), rob.inertia(qo), rob.coriolis(qo, qdo), rob.gravload(qo)
        Jd = rob.jacob0_dot(qo, qdo, representation="rpy/xyz")
        Mx, Cx = (torch.empty((NO, 6, 6), dtype=torch.float64, device=dev) for _ in range(2))
        Gx = torch.empty((NO, 6), dtype=torch.float64, device=dev)
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        for case, ins, outs in ((f"opspace_mx_{tag}_f64", (Ja, M, None, None, None), (Mx, None, None)),
                                (f"opspace_mx_cx_gx_{tag}_f64", (Ja, M, Cm, Jd, G), (Mx, Cx, Gx))):
            if not want(case):
                continue
            a = [p(t) for t in ins]
            o = [p(t) for t in outs]
            bpr = (sum(t[0].numel() for t in ins if t is not None) + sum(t[0].numel() for t in outs if t is not None)) * 8
            report(case, timeit(lambda i: rtb._lib.check(Lo.b2k_opspace(rtb._lib.F64, n, kind, a[0], None, a[1], a[2], a[3], a[4], None,
                                                                        None, None, NO, None, o[0], o[1], o[2], None, None, sto)), 1),
                   NO, bpr, {"api": "C ABI, inputs staged on the device"})
        case = f"opspace_coriolis_x_pipeline_{tag}_f64"
        if want(case):
            pinv = kind == rtb._lib.OPS_PINV
            report(case, timeit(lambda i: rob.coriolis_x(qo, qdo, pinv=pinv), 1), NO, (2 * n + 36) * 8,
                   {"api": "public Python call on device-resident q, qd: jacob0_analytical, jacob0_dot, coriolis, inertia, b2k_opspace"})
        del qo, qdo, Ja, M, Cm, G, Jd, Mx, Cx, Gx

# Closed-form IK (b2k_ikine_6s) of Puma560 on device-resident poses: one configuration, and all eight from one read of T.
# Bytes per row = T in, q and the ok flags out: (16 + 6) reals + 4 for one, 16 reals + 8 (6 reals + 4) for eight.  The
# share is against the data sheet's 3.35 TB/s; where it stays low the kernel is bound by FP64 issue (about a dozen
# transcendental functions per configuration), not by HBM.  The card's name and power limit are read in the same run.
if want("ikine_a_"):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    puma = rtb.models.Puma560()
    NI = args.rows
    Tq = torch.from_numpy(rng.uniform(-np.pi, np.pi, (NI, 6))).to(dev)
    T64 = puma.ets().eval(Tq)
    Li = rtb._lib.lib()
    sti = torch.cuda.current_stream().cuda_stream
    dhi = np.ascontiguousarray([[l.d, l.a, l.alpha, l.offset] for l in puma.links], dtype=np.float64)
    for dt, tag in ((np.float64, "f64"), (np.float32, "f32")):
        Ti = T64 if dt == np.float64 else T64.float()
        sz = np.dtype(dt).itemsize
        for nc, bpr in ((1, (16 + 6) * sz + 4), (8, 16 * sz + 8 * (6 * sz + 4))):
            case = f"ikine_a_puma_{nc}conf_{tag}"
            if not want(case):
                continue
            conf = np.arange(nc, dtype=np.int32)
            qi = torch.empty((NI, nc, 6), dtype=Ti.dtype, device=dev)
            oki = torch.empty((NI, nc), dtype=torch.int32, device=dev)
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            ms = timeit(lambda i: rtb._lib.check(Li.b2k_ikine_6s(code, rtb._lib.dptr(dhi), None, None, Ti.data_ptr(), NI, nc,
                                                                 conf.ctypes.data_as(rtb._lib.ip), qi.data_ptr(), oki.data_ptr(),
                                                                 sti)), 1)
            report(case, ms, NI, bpr, dict(card, api="C ABI, poses on the device", frac_of_3350=round(bpr * NI / (ms * 1e-3) / 3.35e12, 4),
                                           solved=float(oki.float().mean())))
            del qi, oki
    del Tq, T64

# Closed-form IK of UR-type arms (b2k_ikine_ur) of UR10 on device-resident poses, with the bytes per row and the card
# context of the ikine_a_ block above, so that `--only ikine_` times both kernels in one run.
if want("ikine_ur_"):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    ur10 = rtb.models.UR10()
    NI = args.rows
    Tq = torch.from_numpy(rng.uniform(-np.pi, np.pi, (NI, 6))).to(dev)
    T64 = ur10.ets().eval(Tq)
    Li = rtb._lib.lib()
    sti = torch.cuda.current_stream().cuda_stream
    dhi = np.ascontiguousarray([[l.d, l.a, l.alpha, l.offset] for l in ur10.links], dtype=np.float64)
    for dt, tag in ((np.float64, "f64"), (np.float32, "f32")):
        Ti = T64 if dt == np.float64 else T64.float()
        sz = np.dtype(dt).itemsize
        for nc, bpr in ((1, (16 + 6) * sz + 4), (8, 16 * sz + 8 * (6 * sz + 4))):
            case = f"ikine_ur_ur10_{nc}conf_{tag}"
            if not want(case):
                continue
            conf = np.arange(nc, dtype=np.int32)
            qi = torch.empty((NI, nc, 6), dtype=Ti.dtype, device=dev)
            oki = torch.empty((NI, nc), dtype=torch.int32, device=dev)
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            ms = timeit(lambda i: rtb._lib.check(Li.b2k_ikine_ur(code, rtb._lib.dptr(dhi), None, None, Ti.data_ptr(), NI, nc,
                                                                 conf.ctypes.data_as(rtb._lib.ip), qi.data_ptr(), oki.data_ptr(),
                                                                 sti)), 1)
            report(case, ms, NI, bpr, dict(card, api="C ABI, poses on the device", frac_of_3350=round(bpr * NI / (ms * 1e-3) / 3.35e12, 4),
                                           solved=float(oki.float().mean())))
            del qi, oki
    del Tq, T64

# Closed-form IK of Panda-type arms at a given q7 (b2k_ikine_panda) of PandaMDH on device-resident poses and q7, with the
# card context of the blocks above, so that `--only ikine_` times all three kernels in one run.  Bytes per row = T and q7
# in, q and the ok flags out: (16 + 1 + 7k) reals + 4k for k configurations.  For context per solved pose, ik_LM (the
# public call, joint limits on) and ikine_panda with all eight configurations are timed on the same --ik-rows reachable
# targets, ikine_panda at each target's own q7.
if want("ikine_panda_"):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    pmdh = rtb.models.PandaMDH()
    NI = args.rows
    Qp = torch.from_numpy(rng.uniform(-np.pi, np.pi, (NI, 7))).to(dev)
    T64, q764 = pmdh.ets().eval(Qp), Qp[:, 6].contiguous()
    Li = rtb._lib.lib()
    sti = torch.cuda.current_stream().cuda_stream
    dhi = np.ascontiguousarray([[l.d, l.a, l.alpha, l.offset] for l in pmdh.links], dtype=np.float64)
    tl = np.ascontiguousarray(pmdh._tool)
    for dt, tag in ((np.float64, "f64"), (np.float32, "f32")):
        Ti, q7i = (T64, q764) if dt == np.float64 else (T64.float(), q764.float())
        sz = np.dtype(dt).itemsize
        for nc in (1, 8):
            case = f"ikine_panda_pandamdh_{nc}conf_{tag}"
            if not want(case):
                continue
            bpr = (16 + 1 + 7 * nc) * sz + 4 * nc
            conf = np.arange(nc, dtype=np.int32)
            qi = torch.empty((NI, nc, 7), dtype=Ti.dtype, device=dev)
            oki = torch.empty((NI, nc), dtype=torch.int32, device=dev)
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            ms = timeit(lambda i: rtb._lib.check(Li.b2k_ikine_panda(code, rtb._lib.dptr(dhi), None, rtb._lib.dptr(tl), Ti.data_ptr(),
                                                                    q7i.data_ptr(), NI, nc, conf.ctypes.data_as(rtb._lib.ip),
                                                                    qi.data_ptr(), oki.data_ptr(), sti)), 1)
            report(case, ms, NI, bpr, dict(card, api="C ABI, poses and q7 on the device", frac_of_3350=round(bpr * NI / (ms * 1e-3) / 3.35e12, 4),
                                           solved=float(oki.float().mean())))
            del qi, oki
    del Qp, T64, q764
    case = "ikine_panda_vs_ik_lm_pandamdh_f64"
    if want(case):
        M = args.ik_rows
        ql = pmdh.qlim
        Qm = torch.from_numpy(np.random.default_rng(2).uniform(ql[0], ql[1], (M, 7))).to(dev)
        Tm = pmdh.ets().eval(Qm)
        q7m = Qm[:, 6].contiguous()
        eight = ["lun", "run", "ldn", "rdn", "luf", "ruf", "ldf", "rdf"]
        lm_ms = timeit(lambda i: pmdh.ik_LM(Tm), 1)
        okv = pmdh.ik_LM(Tm)[1]
        lm_ok = float((okv.cpu().numpy() if hasattr(okv, "cpu") else np.asarray(okv)).mean())
        cf_ms = timeit(lambda i: pmdh.ikine_panda(Tm, q7m, config=eight), 1)
        cf = pmdh.ikine_panda(Tm, q7m, config=eight)
        cf_ok = float((~torch.isnan(cf.q[:, :, 0])).any(1).float().mean())
        report(case, cf_ms, M, (16 + 1 + 56) * 8 + 32,
               dict(card, api="public Python calls on device-resident targets", ik_lm_ms=round(lm_ms, 4), ik_lm_solved=lm_ok,
                    ik_lm_us_per_solved_pose=round(lm_ms * 1e3 / max(lm_ok * M, 1), 5), ikine_panda_solved=cf_ok,
                    ikine_panda_us_per_solved_pose=round(cf_ms * 1e3 / max(cf_ok * M, 1), 5)))
        del Qm, Tm, q7m, cf

# IK (config 4): reachable targets, chan
if want("ik_"):
    panda = rtb.models.Panda().ets()
    M = args.ik_rows
    qs = np.random.default_rng(2).uniform(-np.pi, np.pi, (M, 7))
    Tep = panda.eval(qs)  # reachable targets: Tep = FK(q*) (SURVEY 8d config 4)
    for dt in (np.float32, np.float64):
        tag = "f64" if dt == np.float64 else "f32"
        Td = torch.from_numpy(Tep.astype(dt)).to(dev)
        for k, jl, meth in ((0.1, False, 0), (1.0, True, 0), (0.1, False, 3), (0.0, False, 4)):
            name = f"ik_lm_panda_{tag}_chan{k}_jl{int(jl)}" if meth == 0 else f"ik_{'nr' if meth == 3 else 'gn'}_panda_{tag}_damp{k}"
            if not want(name):
                continue
            n = 7
            tdtype = torch.float32 if dt == np.float32 else torch.float64
            qo = torch.empty((M, n), dtype=tdtype, device=dev)
            so, io, ro = (torch.empty(M, dtype=torch.int32, device=dev) for _ in range(3))
            Eo = torch.empty(M, dtype=tdtype, device=dev)
            Lb = rtb._lib.lib()
            chn = panda._chain
            stp = torch.cuda.current_stream().cuda_stream
            codei = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32

            def run(i):  # straight through the C ABI: no per-call allocations on the Python side
                rtb._lib.check(Lb.b2k_ik_lm(chn, codei, Td.data_ptr(), M, None, 30, 100, 1e-6, int(jl), None, float(k), meth,
                                            5 + i, 0, 1, qo.data_ptr(), so.data_ptr(), io.data_ptr(), ro.data_ptr(),
                                            Eo.data_ptr(), stp))

            steps, args.steps = args.steps, 10
            wu, args.warmup = args.warmup, 2
            ms = timeit(run, 1 << 30)
            args.steps, args.warmup = steps, wu
            out = {"r": (qo, so, io, ro, Eo)}
            q, s, it, sr, E = out["r"]
            report(name, ms, M, (16 + 7 + 4) * np.dtype(dt).itemsize,
                   {"solves_per_s": M / (ms * 1e-3), "success": float(s.float().mean()), "mean_it": float(it.float().mean()),
                    "max_it": int(it.max()), "mean_searches": float(sr.float().mean()), "max_searches": int(sr.max())})

# IK with the null-space terms (b2k_ikine_null) against the same loop without them: config 4's targets (Panda, reachable,
# seed 2), the Python solver loop (ikine_LM: chan k = 1.0, joint limits checked, restarts shared by all rows), gains 1.0,
# ps = 0, pi = 0.3.  "off" is b2k_ik_lm in the same semantics.  The card's name and power limit are read in the same run.
if want("ikine_null_"):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    panda = rtb.models.Panda().ets()
    M = args.ik_rows
    Tep = panda.eval(np.random.default_rng(2).uniform(-np.pi, np.pi, (M, 7)))
    Lb = rtb._lib.lib()
    chn = panda._chain
    stp = torch.cuda.current_stream().cuda_stream
    pi = np.full(7, 0.3)
    for dt in (np.float32, np.float64):
        tag = "f64" if dt == np.float64 else "f32"
        Td = torch.from_numpy(Tep.astype(dt)).to(dev)
        codei = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
        for var, kq, km in (("off", 0.0, 0.0), ("kq", 1.0, 0.0), ("km", 0.0, 1.0), ("both", 1.0, 1.0)):
            name = f"ikine_null_panda_{tag}_{var}"
            if not want(name):
                continue
            qo = torch.empty((M, 7), dtype=Td.dtype, device=dev)
            so, io, ro = (torch.empty(M, dtype=torch.int32, device=dev) for _ in range(3))
            Eo = torch.empty(M, dtype=Td.dtype, device=dev)

            def run(i):
                if var == "off":
                    rc = Lb.b2k_ik_lm(chn, codei, Td.data_ptr(), M, None, 30, 100, 1e-6, 1, None, 1.0, 0, 5 + i,
                                      rtb._lib.SEM_PYTHON, 0, qo.data_ptr(), so.data_ptr(), io.data_ptr(), ro.data_ptr(),
                                      Eo.data_ptr(), stp)
                else:
                    rc = Lb.b2k_ikine_null(chn, codei, Td.data_ptr(), M, None, 30, 100, 1e-6, 1, None, 1.0, 0, 5 + i, 0,
                                           kq, km, 0.0, rtb._lib.dptr(pi), qo.data_ptr(), so.data_ptr(), io.data_ptr(),
                                           ro.data_ptr(), Eo.data_ptr(), stp)
                rtb._lib.check(rc)

            steps, args.steps = args.steps, 10
            wu, args.warmup = args.warmup, 2
            ms = timeit(run, 1 << 30)
            args.steps, args.warmup = steps, wu
            report(name, ms, M, (16 + 7 + 4) * np.dtype(dt).itemsize,
                   dict(card, solves_per_s=M / (ms * 1e-3), success=float(so.float().mean()), mean_it=float(io.float().mean()),
                        mean_searches=float(ro.float().mean())))
            del qo, so, io, ro, Eo
        del Td

# IK with the quadratic-programming step (b2k_ikine_qp) against the LM loop: config 4's targets (Panda, reachable,
# seed 2), the Python solver loop (joint limits checked, restarts shared by all rows), kj = ks = 1, ps = 0, pi = 0.3,
# kq / km = 1.0 where on.  "lm" is b2k_ik_lm in the same semantics (chan k = 1.0).  The card's name and power limit are
# read in the same run.
if want("ikine_qp_"):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    panda = rtb.models.Panda().ets()
    M = args.ik_rows
    Tep = panda.eval(np.random.default_rng(2).uniform(-np.pi, np.pi, (M, 7)))
    Lb = rtb._lib.lib()
    chn = panda._chain
    stp = torch.cuda.current_stream().cuda_stream
    pi = np.full(7, 0.3)
    for dt in (np.float32, np.float64):
        tag = "f64" if dt == np.float64 else "f32"
        Td = torch.from_numpy(Tep.astype(dt)).to(dev)
        codei = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
        for var, kq, km in (("lm", 0.0, 0.0), ("off", 0.0, 0.0), ("kq", 1.0, 0.0), ("km", 0.0, 1.0), ("both", 1.0, 1.0)):
            name = f"ikine_qp_panda_{tag}_{var}"
            if not want(name):
                continue
            qo = torch.empty((M, 7), dtype=Td.dtype, device=dev)
            so, io, ro = (torch.empty(M, dtype=torch.int32, device=dev) for _ in range(3))
            Eo = torch.empty(M, dtype=Td.dtype, device=dev)

            def run(i):
                if var == "lm":
                    rc = Lb.b2k_ik_lm(chn, codei, Td.data_ptr(), M, None, 30, 100, 1e-6, 1, None, 1.0, 0, 5 + i,
                                      rtb._lib.SEM_PYTHON, 0, qo.data_ptr(), so.data_ptr(), io.data_ptr(), ro.data_ptr(),
                                      Eo.data_ptr(), stp)
                else:
                    rc = Lb.b2k_ikine_qp(chn, codei, Td.data_ptr(), M, None, 30, 100, 1e-6, 1, None, 5 + i, 0, 1.0, 1.0,
                                         kq, km, 0.0, rtb._lib.dptr(pi), qo.data_ptr(), so.data_ptr(), io.data_ptr(),
                                         ro.data_ptr(), Eo.data_ptr(), stp)
                rtb._lib.check(rc)

            steps, args.steps = args.steps, 10
            wu, args.warmup = args.warmup, 2
            ms = timeit(run, 1 << 30)
            args.steps, args.warmup = steps, wu
            report(name, ms, M, (16 + 7 + 4) * np.dtype(dt).itemsize,
                   dict(card, solves_per_s=M / (ms * 1e-3), success=float(so.float().mean()), mean_it=float(io.float().mean()),
                        mean_searches=float(ro.float().mean())))
            del qo, so, io, ro, Eo
        del Td

# Planar chains (b2k_fkine_planar, csrc/b2k_planar.cu) through the C ABI: Planar2 (n = 2) and a 7-joint chain with R,
# tx and ty joints, a flip and constants between joints, 1M rows.  Algorithmic bytes per row, sizeof(real) = es:
# fkine (n + 9) es, jacob0 (n + 3n) es, fkine_jacob0 (n + 9 + 3n) es.  planar_3d_fkine_jacob0 is the 3-D kernel on the
# same (embedded) chain, for context: it writes the 16 + 6n reals of the 3-D pose and Jacobian, and its share is stated
# for the planar call's bytes.  The card's name and power limit are read in the same run.
if want("planar_"):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    E2 = rtb.ET2
    planar7 = rtb.ETS2([E2.R(), E2.tx(0.4), E2.R(), E2.tx(0.3), E2.ty(), E2.R(), E2.tx(0.25), E2.R(flip=True), E2.tx(),
                        E2.R(), E2.tx(0.1), E2.ty(0.05)])
    Lp = rtb._lib.lib()
    stp = torch.cuda.current_stream().cuda_stream
    rngp = np.random.default_rng(8)
    for fam, ets in (("planar2", rtb.models.ETS.Planar2().ets()), ("planar7", planar7)):
        n = ets.n
        for dt in (np.float64, np.float32):
            es = np.dtype(dt).itemsize
            tag = f"{fam}_{'f64' if dt == np.float64 else 'f32'}"
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            nbuf = min(8, max(2, int(np.ceil(300e6 / (N * n * es)))))
            qs = [torch.from_numpy(rngp.uniform(-np.pi, np.pi, (N, n)).astype(dt)).to(dev) for _ in range(nbuf)]
            T = torch.empty((N, 3, 3), dtype=tdt[dt], device=dev)
            J = torch.empty((N, 3, n), dtype=tdt[dt], device=dev)
            ch = ets._chain
            for case, t, j, bpr in ((f"planar_fkine_{tag}", T, None, n + 9), (f"planar_jacob0_{tag}", None, J, 4 * n),
                                    (f"planar_fkine_jacob0_{tag}", T, J, 4 * n + 9)):
                if not want(case):
                    continue
                tp, jp = (None if t is None else t.data_ptr()), (None if j is None else j.data_ptr())
                ms = timeit(lambda i: rtb._lib.check(Lp.b2k_fkine_planar(ch, code, qs[i].data_ptr(), N, n, None, None, 0, tp, jp, stp)), nbuf)
                report(case, ms, N, bpr * es, dict(card, api="C ABI, q on the device", frac_of_3350=round(bpr * es * N / (ms * 1e-3) / 3.35e12, 4)))
            case = f"planar_3d_fkine_jacob0_{tag}"
            if want(case):
                T3 = torch.empty((N, 4, 4), dtype=tdt[dt], device=dev)
                J3 = torch.empty((N, 6, n), dtype=tdt[dt], device=dev)
                ms = timeit(lambda i: rtb._lib.check(Lp.b2k_fkine_jacob0(ch, code, qs[i].data_ptr(), N, n, None, None, T3.data_ptr(), J3.data_ptr(), stp)), nbuf)
                report(case, ms, N, (4 * n + 9) * es, dict(card, api="C ABI, 3-D kernel on the embedded chain", bytes_written_per_row=(16 + 6 * n) * es,
                                                          frac_of_3350=round((4 * n + 9) * es * N / (ms * 1e-3) / 3.35e12, 4)))
                del T3, J3
            del qs, T, J

# Analytical derivatives of the DH recursion (k_rne_deriv, csrc/b2k_rne.cuh) through the C ABI, Puma560, 1M rows.
# Algorithmic bytes per row, sizeof(real) = es: rne_derivatives (3n + 2n^2) es, accel_derivatives (3n + 3n^2) es.  The
# kernel does 2n dual-number recursions per row (plus n + 1 plain ones and an n x n solve for accel_derivatives), so it is
# expected to be compute-bound; frac_of_hbm is stated for context only.  fd_route is what a user has without it: the
# 2n + 1 b2k_rne launches of a one-sided finite difference (q and qd perturbed one joint at a time), timed in the same
# call on the same rows.  The card's name and power limit are read in the same run.
DERIV_CASES = [f"dyn_{op}_derivs_puma_{t}" for op in ("rne", "accel") for t in ("f64", "f32")]
if any(want(c) for c in DERIV_CASES):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    Ld = rtb._lib.lib()
    std = torch.cuda.current_stream().cuda_stream
    pz = rtb.models.Puma560()
    pz.rne(np.zeros(6), np.zeros(6), np.zeros(6))  # creates the handle
    hd, n = pz._rne_ob, 6
    gd = np.ascontiguousarray(-pz.gravity)
    rngd = np.random.default_rng(13)
    for dt in (np.float64, np.float32):
        tag = "f64" if dt == np.float64 else "f32"
        es = np.dtype(dt).itemsize
        code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
        tt = torch.float64 if dt == np.float64 else torch.float32
        q0, qd0, x0 = (torch.from_numpy(rngd.uniform(-2, 2, (N, n)).astype(dt)).to(dev) for _ in range(3))
        o = [torch.empty((N, n, n), dtype=tt, device=dev) for _ in range(3)]
        c_rne, c_acc = f"dyn_rne_derivs_puma_{tag}", f"dyn_accel_derivs_puma_{tag}"
        fd = {}
        if want(c_rne) or want(c_acc):
            hstep = 1e-6 if dt == np.float64 else 1e-2
            pert = []
            for k in range(n):
                e = torch.zeros(n, dtype=tt, device=dev)
                e[k] = hstep
                pert.append((q0 + e, qd0))
                pert.append((q0, qd0 + e))
            pert.append((q0, qd0))
            tau = [torch.empty((N, n), dtype=tt, device=dev) for _ in pert]

            def fd_route(i):
                for (a, b), t in zip(pert, tau):
                    rtb._lib.check(Ld.b2k_rne(hd, code, a.data_ptr(), b.data_ptr(), x0.data_ptr(), N, rtb._lib.dptr(gd), None, t.data_ptr(), std))

            ms_fd = timeit(fd_route, 1)
            fd = {"fd_route_ms": round(ms_fd, 4), "fd_route_launches": 2 * n + 1}
            del pert, tau
        if want(c_rne):
            ms = timeit(lambda i: rtb._lib.check(Ld.b2k_rne_derivatives(hd, code, q0.data_ptr(), qd0.data_ptr(), x0.data_ptr(), N, rtb._lib.dptr(gd),
                                                                       None, o[0].data_ptr(), o[1].data_ptr(), std)), 1)
            report(c_rne, ms, N, (3 * n + 2 * n * n) * es, dict(card, **fd, bound="compute (expected, not measured)",
                                                                 speedup_vs_fd_route=round(fd["fd_route_ms"] / ms, 2)))
        if want(c_acc):
            ms = timeit(lambda i: rtb._lib.check(Ld.b2k_rne_accel_derivatives(hd, code, q0.data_ptr(), qd0.data_ptr(), x0.data_ptr(), N,
                                                                             rtb._lib.dptr(gd), o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), std)), 1)
            report(c_acc, ms, N, (3 * n + 3 * n * n) * es, dict(card, **fd, bound="compute (expected, not measured)",
                                                                 speedup_vs_fd_route=round(fd["fd_route_ms"] / ms, 2)))
        del q0, qd0, x0, o

# The dynamics regressor (DHRobot.rne_regressor, b2k_rne_regressor) and its normal equations (b2k_rne_regressor_gram),
# Puma560 (DH) and PandaMDH, N device rows.  Algorithmic bytes per row of the regressor: (3n + 14n^2) es, against
# 3.35 TB/s.  The gram is compute work: n p^2 / 2 FMAs per row (p = 14n, the upper triangle of p x p per joint row),
# reported in FP64 FLOP/s against the data sheet's 34 TFLOP/s (non-tensor).  unit_route is what a user has without the
# regressor, timed in the same call on the same rows: 14n b2k_rne launches, one per unit link table (tests/regressor_ref.py;
# the m r columns need one more subtraction each, not counted), with both routes alternated.  The card's name and power limit are read in the same run.
REG_CASES = [f"regressor_{r}_{t}" for r in ("puma", "pandamdh") for t in ("f64", "f32")] + \
            [f"regressor_gram_{r}_{t}" for r in ("puma", "pandamdh") for t in ("f64", "f32")]
if any(want(c) for c in REG_CASES):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    Lr = rtb._lib.lib()
    str_ = torch.cuda.current_stream().cuda_stream
    rngr = np.random.default_rng(16)
    for rname, rob in (("puma", rtb.models.Puma560()), ("pandamdh", rtb.models.PandaMDH())):
        n, p = rob.n, 14 * rob.n
        hr = rob._rne_handle()
        gr = rob._kernel_gravity(None)
        for dt in (np.float64, np.float32):
            tag = "f64" if dt == np.float64 else "f32"
            c_reg, c_gram = f"regressor_{rname}_{tag}", f"regressor_gram_{rname}_{tag}"
            if not (want(c_reg) or want(c_gram)):
                continue
            es = np.dtype(dt).itemsize
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            tt = torch.float64 if dt == np.float64 else torch.float32
            q0, qd0, qdd0, tau0 = (torch.from_numpy(rngr.uniform(-2, 2, (N, n)).astype(dt)).to(dev) for _ in range(4))
            if want(c_reg):
                Y = torch.empty((N, n, p), dtype=tt, device=dev)
                units = []
                for i in range(p):  # one rne handle per column; which parameter is 1 does not change an rne launch's time
                    import ctypes
                    T = rob._pack_rne().reshape(-1, 24).copy()
                    T[:, 6:20] = 0.0
                    T[:, 21:24] = 0.0
                    T[i // 14, 6] = 1.0
                    hu = rtb._lib.vp()
                    rtb._lib.check(Lr.b2k_rne_create(n, rob.mdh, rtb._lib.dptr(np.ascontiguousarray(T.ravel())), ctypes.byref(hu)))
                    units.append(hu)
                outs = [torch.empty((N, n), dtype=tt, device=dev) for _ in range(p)]

                def unit_route(i):
                    for hu, t in zip(units, outs):
                        rtb._lib.check(Lr.b2k_rne(hu, code, q0.data_ptr(), qd0.data_ptr(), qdd0.data_ptr(), N, rtb._lib.dptr(gr), None,
                                                  t.data_ptr(), str_))

                ms_u, ms = [], []
                for _ in range(2):  # alternate the two routes, so that both see the same clocks
                    ms_u.append(timeit(unit_route, 1))
                    ms.append(timeit(lambda i: rtb._lib.check(Lr.b2k_rne_regressor(hr, code, q0.data_ptr(), qd0.data_ptr(), qdd0.data_ptr(), N,
                                                                                   rtb._lib.dptr(gr), Y.data_ptr(), str_)), 1))
                ms_u, ms = min(ms_u), min(ms)
                bpr = (3 * n + 14 * n * n) * es
                report(c_reg, ms, N, bpr, dict(card, frac_of_3p35TBps=round(bpr * N / (ms * 1e-3) / 3.35e12, 4), unit_route_ms=round(ms_u, 4),
                                               unit_route_launches=p, speedup_vs_unit_route=round(ms_u / ms, 2),
                                               kernel=rob.rne_kernel_info("rne_regressor", dt)))
                for hu in units:
                    Lr.b2k_rne_destroy(hu)
                del Y, outs
            if want(c_gram):
                G = torch.empty((p, p), dtype=torch.float64, device=dev)
                b = torch.empty(p, dtype=torch.float64, device=dev)
                s = torch.empty(1, dtype=torch.float64, device=dev)
                ms = timeit(lambda i: rtb._lib.check(Lr.b2k_rne_regressor_gram(hr, code, q0.data_ptr(), qd0.data_ptr(), qdd0.data_ptr(), tau0.data_ptr(),
                                                                               N, rtb._lib.dptr(gr), None, G.data_ptr(), b.data_ptr(), s.data_ptr(), str_)), 1)
                flops = 2 * (n * p * p / 2) * N
                report(c_gram, ms, N, 4 * n * es, dict(card, fp64_tflops=round(flops / (ms * 1e-3) / 1e12, 2),
                                                      frac_of_34TFLOPs=round(flops / (ms * 1e-3) / 34e12, 4)))
            del q0, qd0, qdd0, tau0

# The dynamics regressor of a rigid-body tree (Robot.rne_regressor, b2k_tree_regressor) and its normal equations
# (b2k_tree_regressor_gram): the Puma560 assembled as an ETS robot and a branched 16-joint tree, N device rows.
# Algorithmic bytes per row of the regressor: (3n + 10n^2) es, against 3.35 TB/s.  The gram is reported in FP64 FLOP/s
# (n p^2 / 2 FMAs per row, p = 10n).  unit_route is what a user has without the regressor, timed in the same call on the
# same rows with both routes alternated: 10n b2k_tree_rne launches, one per handle whose only nonzero inertia is one unit
# parameter of one group (tests/tree_regressor_ref.py).  The card's name and power limit are read in the same run.
TREG_CASES = [f"tree_regressor_{r}_{t}" for r in ("puma", "tree16") for t in ("f64", "f32")] + \
             [f"tree_regressor_gram_{r}_{t}" for r in ("puma", "tree16") for t in ("f64", "f32")]
if any(want(c) for c in TREG_CASES):
    import ctypes
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import tree_regressor_ref as TRR  # noqa: E402
    from test_gpu_tree import random_robot  # noqa: E402
    from test_gpu_tree_derivs import puma_ets  # noqa: E402

    Lt = rtb._lib.lib()
    stt = torch.cuda.current_stream().cuda_stream
    rngq = np.random.default_rng(18)
    for rname, rob in (("puma", puma_ets(0.0)[0]), ("tree16", random_robot(np.random.default_rng(61), 16, True))):
        n, p = rob.n, 10 * rob.n
        ht = rob._tree_handle()
        ag = rob._kernel_gravity(None)
        desc = rob.tree_description()
        for dt in (np.float64, np.float32):
            tag = "f64" if dt == np.float64 else "f32"
            c_reg, c_gram = f"tree_regressor_{rname}_{tag}", f"tree_regressor_gram_{rname}_{tag}"
            if not (want(c_reg) or want(c_gram)):
                continue
            es = np.dtype(dt).itemsize
            code = rtb._lib.F64 if dt == np.float64 else rtb._lib.F32
            tt = torch.float64 if dt == np.float64 else torch.float32
            q0, qd0, qdd0, tau0 = (torch.from_numpy(rngq.uniform(-2, 2, (N, n)).astype(dt)).to(dev) for _ in range(4))
            if want(c_reg):
                Y = torch.empty((N, n, p), dtype=tt, device=dev)
                units = []
                for k in range(p):
                    I6 = np.zeros((n, 6, 6))
                    I6[k // 10] = TRR.basis(k % 10)
                    i32 = [np.ascontiguousarray(desc[key], dtype=np.int32) for key in ("parent", "axis", "flip", "jindex")]
                    Cm = np.ascontiguousarray(np.asarray(desc["C"], dtype=np.float64)[:, :3, :].reshape(n, 12))
                    hu = rtb._lib.vp()
                    rtb._lib.check(Lt.b2k_tree_create(n, *(a.ctypes.data_as(rtb._lib.ip) for a in i32), rtb._lib.dptr(Cm),
                                                      rtb._lib.dptr(np.ascontiguousarray(I6.reshape(n, 36))), ctypes.byref(hu)))
                    units.append(hu)
                outs = [torch.empty((N, n), dtype=tt, device=dev) for _ in range(p)]

                def unit_route(i):
                    for hu, t in zip(units, outs):
                        rtb._lib.check(Lt.b2k_tree_rne(hu, code, q0.data_ptr(), qd0.data_ptr(), qdd0.data_ptr(), N, rtb._lib.dptr(ag),
                                                       t.data_ptr(), stt))

                ms_u, ms = [], []
                for _ in range(2):  # alternate the two routes, so that both see the same clocks
                    ms_u.append(timeit(unit_route, 1))
                    ms.append(timeit(lambda i: rtb._lib.check(Lt.b2k_tree_regressor(ht, code, q0.data_ptr(), qd0.data_ptr(), qdd0.data_ptr(),
                                                                                    N, rtb._lib.dptr(ag), Y.data_ptr(), stt)), 1))
                ms_u, ms = min(ms_u), min(ms)
                bpr = (3 * n + 10 * n * n) * es
                report(c_reg, ms, N, bpr, dict(card, frac_of_3p35TBps=round(bpr * N / (ms * 1e-3) / 3.35e12, 4), unit_route_ms=round(ms_u, 4),
                                               unit_route_launches=p, speedup_vs_unit_route=round(ms_u / ms, 2),
                                               kernel=rob.rne_kernel_info(dt, op="rne_regressor")))
                for hu in units:
                    Lt.b2k_tree_destroy(hu)
                del Y, outs
            if want(c_gram):
                G = torch.empty((p, p), dtype=torch.float64, device=dev)
                b = torch.empty(p, dtype=torch.float64, device=dev)
                s = torch.empty(1, dtype=torch.float64, device=dev)
                ms = timeit(lambda i: rtb._lib.check(Lt.b2k_tree_regressor_gram(ht, code, q0.data_ptr(), qd0.data_ptr(), qdd0.data_ptr(),
                                                                                tau0.data_ptr(), N, rtb._lib.dptr(ag), None, G.data_ptr(),
                                                                                b.data_ptr(), s.data_ptr(), stt)), 1)
                flops = 2 * (n * p * p / 2) * N
                report(c_gram, ms, N, 4 * n * es, dict(card, fp64_tflops=round(flops / (ms * 1e-3) / 1e12, 2),
                                                      frac_of_34TFLOPs=round(flops / (ms * 1e-3) / 34e12, 4)))
            del q0, qd0, qdd0, tau0

# Fixed-step RK4 rollouts with discrete-time sensitivities (DHRobot.rollout / Robot.rollout: b2k_rne_rollout,
# b2k_tree_rollout): Puma560 and PandaMDH (DH) and the UR10 assembled as an ETS robot (tree), N = 16384 trajectories of
# K = 64 steps, one shared torque sequence.  Bytes per trajectory = what the kernel must write: q and qd, 2n (K + 1) reals,
# plus K 6 n^2 reals of A_k | B_k with sensitivities; reported against 3.35 TB/s.  step_route is what a user has without
# the kernel, timed in the same call with both routes alternated: per step four accel and four accel_derivatives launches
# and the torch composition of the RK4 stages.  The card's name and power limit are read in the same run.
ROLL_CASES = [f"rollout_{r}_{t}_{s}" for r in ("puma", "pandamdh", "ur10tree") for t in ("f64", "f32") for s in ("states", "sens")]
if any(want(c) for c in ROLL_CASES):
    import subprocess

    try:
        plim = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # the figure is context, the timing does not depend on it
        plim = f"unavailable ({type(e).__name__})"
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": plim}
    from oracle import chains as ch  # noqa: E402

    def dh_as_tree(dh):
        """A standard-DH link table as an ETS robot: point masses at the links' centres of mass (Robot.rne's model)."""
        links, prev = [], rtb.ETS()
        for j, l in enumerate(dh):
            post = rtb.ETS()
            for kind, v in (("tz", l["d"]), ("tx", l["a"]), ("Rx", l["alpha"])):
                if v != 0:
                    post = post * getattr(rtb.ET, kind)(v)
            Tpost = np.eye(4)
            for et in post:
                Tpost = Tpost @ et.A()
            r_in = Tpost[:3, :3] @ np.asarray(l["r"], dtype=float) + Tpost[:3, 3]
            links.append(rtb.Link(prev * rtb.ET.Rz(), name=f"l{j}", parent=links[-1] if links else None, m=l["m"], r=r_in))
            prev = post
        links.append(rtb.Link(prev, name="tool", parent=links[-1]))
        return rtb.Robot(links)

    def step_route(rob, q0, qd0, tau, h, sens):
        """RK4 with chained sensitivities from the public accel / accel_derivatives, composed with torch."""
        n = rob.n
        x = torch.cat([q0, qd0], 1)
        N = x.shape[0]
        I = torch.eye(2 * n, dtype=x.dtype, device=x.device)
        qs, As, Bs = [x], [], []
        for k in range(tau.shape[0]):
            t = tau[k].expand(N, n).contiguous()
            ks, dxs, dus = [], [], []
            for c in (0.0, 0.5, 0.5, 1.0):
                xs = x if not ks else x + (c * h) * ks[-1]
                q, qd = xs[:, :n].contiguous(), xs[:, n:].contiguous()
                ks.append(torch.cat([qd, rob.accel(q, qd, t)], 1))
                if sens:
                    aq, aqd, at = rob.accel_derivatives(q, qd, t)
                    J = torch.zeros((N, 2 * n, 2 * n), dtype=x.dtype, device=x.device)
                    J[:, :n, n:] = torch.eye(n, dtype=x.dtype, device=x.device)
                    J[:, n:, :n], J[:, n:, n:] = aq, aqd
                    dxs.append(J if not dxs else J @ (I + (c * h) * dxs[-1]))
                    Mt = torch.cat([torch.zeros_like(at), at], 1)
                    dus.append(Mt if not dus else J @ ((c * h) * dus[-1]) + Mt)
            x = x + (h / 6) * (ks[0] + 2 * ks[1] + 2 * ks[2] + ks[3])
            qs.append(x)
            if sens:
                As.append(I + (h / 6) * (dxs[0] + 2 * dxs[1] + 2 * dxs[2] + dxs[3]))
                Bs.append((h / 6) * (dus[0] + 2 * dus[1] + 2 * dus[2] + dus[3]))
        return qs, As, Bs

    NR, KR, HR = 16384, 64, 0.005
    rngr = np.random.default_rng(19)
    robots = (("puma", rtb.models.Puma560()), ("pandamdh", rtb.models.PandaMDH()), ("ur10tree", dh_as_tree(ch.ur10_links())))
    for rname, rob in robots:
        n = rob.n
        for dt in (np.float64, np.float32):
            tag = "f64" if dt == np.float64 else "f32"
            es = np.dtype(dt).itemsize
            q0 = torch.from_numpy(rngr.uniform(-1.5, 1.5, (NR, n)).astype(dt)).to(dev)
            qd0 = torch.from_numpy(rngr.uniform(-1, 1, (NR, n)).astype(dt)).to(dev)
            tau = torch.from_numpy(rngr.normal(size=(KR, n)).astype(dt)).to(dev)
            for sname, sens in (("states", False), ("sens", True)):
                case = f"rollout_{rname}_{tag}_{sname}"
                if not want(case):
                    continue
                # device memory the first call takes beyond torch's allocator: the module and the local memory the
                # driver reserves for the kernel's per-thread stack (a fresh program per case: dtype / sensitivities)
                torch.cuda.synchronize()
                free0, res0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_reserved()
                rob.rollout(q0, tau, HR, qd0=qd0, sensitivities=sens)
                torch.cuda.synchronize()
                driver_mb = ((free0 - torch.cuda.mem_get_info()[0]) - (torch.cuda.memory_reserved() - res0)) / 2**20
                ms_k, ms_r = [], []
                for _ in range(2):  # alternate the two routes, so that both see the same clocks
                    ms_k.append(timeit(lambda i: rob.rollout(q0, tau, HR, qd0=qd0, sensitivities=sens), 1))
                    ms_r.append(timeit(lambda i: step_route(rob, q0, qd0, tau, HR, sens), 1))
                ms_k, ms_r = min(ms_k), min(ms_r)
                bpt = (2 * n * (KR + 1) + (KR * 6 * n * n if sens else 0)) * es
                report(case, ms_k, NR, bpt, dict(card, steps=KR, bytes_written_per_s=round(bpt * NR / (ms_k * 1e-3), 0),
                                                 frac_of_3p35TBps=round(bpt * NR / (ms_k * 1e-3) / 3.35e12, 4),
                                                 step_route_ms=round(ms_r, 3), step_route_launches=KR * (8 if sens else 4),
                                                 speedup_vs_step_route=round(ms_r / ms_k, 2),
                                                 driver_reserved_MB_first_call=round(driver_mb, 1),
                                                 kernel=rob.rne_kernel_info(dtype=dt, op="rollout").split("\n")[int(sens)]))
            del q0, qd0, tau
