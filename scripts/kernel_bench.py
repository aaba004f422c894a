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
ap.add_argument("--variant", type=int, default=0)
args = ap.parse_args()
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    PEAK = 3350.0  # H100 SXM data sheet
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
if args.variant:
    rtb.set_variant(args.variant)


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
        ("extra_fkine_all_panda_f64_per_frame_launches", lambda i: fkine_all_per_frame(PD, Qx), (7 + 8 * 16) * 8),
    ]
    PD = rtb.models.DH.Panda()

    def fkine_all_per_frame(robot, Q):  # the earlier route: one pose launch per frame over the prefix chains
        rtb.ETS.frames_single_walk = False
        try:
            return robot.fkine_all(Q)
        finally:
            rtb.ETS.frames_single_walk = True

    for name, fn, bpr in cases:
        if not want(name):
            continue
        try:
            ms = timeit(fn, 1)
            report(name, ms, NX, bpr, {"api": "public Python call on device-resident inputs"})
        except Exception as e:  # keep the table going
            print(json.dumps({"case": name, "error": f"{type(e).__name__}: {e}"[:300]}), flush=True)
    del Qx, QDx, Jx, Tx, Ty

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
