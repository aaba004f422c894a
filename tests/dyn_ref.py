"""Long-double reference of the DH / MDH inverse dynamics (b2k_rne) and of the five operations built on it
(b2k_rne_inertia, b2k_rne_gravload, b2k_rne_itorque, b2k_rne_coriolis, b2k_rne_accel), with an error bar per entry.

The Newton-Euler recursion is written from the textbook formulation, batched over rows in 80-bit extended precision:
standard DH in link frames after Luh, Walker and Paul (as in Spong / Corke), modified DH after Craig.  Its inputs are
what b2k_rne takes: the packed 24-double link table [alpha, a, theta, d, sigma, offset, m, r(3), I(9), Jm, G, B, Tc+, Tc-]
and the base acceleration ``grav`` (MINUS the robot's gravity).  Behaviour the library keeps on purpose:
  - a prismatic first joint under modified DH keeps the compiled reference's treatment (its link gets the angular rate
    and acceleration q' z, q'' z, and the base acceleration unrotated, without q'' z);
  - the joint torque adds G^2 Jm q'' + G^2 B q' + |G| Tc+ for q' > 0, |G| Tc- for q' < 0 (nothing at q' = +-0);
  - the fan-outs are the reference's DynamicsMixin definitions: inertia = n unit-acceleration calls without gravity,
    coriolis = the centripetal-plus-pair rule on the friction-free robot, accel = M^-1 (torque - rne(q, qd, 0)) with
    friction kept, solved here by Gaussian elimination with partial pivoting in long double.

Error bars.  The same recursion run on absolute values (|R|, |a| |b| for products, |a| + |b| for sums, |q'|, |q''|,
|g|, |fext|) gives for every output the magnitude its rounding error scales with.  The bar of one recursion output is
    K u (2n + 2) |.|  +  (|.| with every sin / cos widened by its error)  -  |.|  +  2 u |.|
(the second term is the effect of the kernel's sin / cos error, of rounding q + offset and of the specialised kernel
snapping sin / cos alpha within 4e-16 of 0 or +-1; the last one the rounding of the link constants to the kernel's
type, which both kernels do), with K = 4 and a floor of a few subnormals.  The fan-outs propagate these bars through their
combination rules; accel propagates them through |M^-1| with the Gaussian-elimination backward error of the solve.
"""
import numpy as np

import fkj_ref

LD = np.longdouble
assert np.finfo(LD).eps < 1e-18, "tests/dyn_ref.py needs 80-bit x86 extended precision for np.longdouble"

SNAP = 4e-16  # b2k_rne_gen.cpp snap(): sin / cos of constant angles within this of 0 or +-1 become exact
OPS = ("rne", "inertia", "gravload", "itorque", "coriolis", "accel")
# plausible kernel defects the bars must catch (tests/test_dyn_ref_cpu.py)
DEFECTS = ("coulomb_at_zero", "signed_G", "jm_G", "mdh_ps_sign", "coriolis_friction", "accel_nofriction", "loose_snap")


def nofriction(L):
    L = np.array(L, dtype=np.float64).reshape(-1, 24).copy()
    L[:, 21:24] = 0.0
    return L.ravel()


def _consts(L, defect=None):
    L = np.asarray(L, dtype=np.float64).reshape(-1, 24)
    al = L[:, 0].astype(LD)
    sa, ca = np.sin(al), np.cos(al)
    if defect == "loose_snap":  # sin / cos of alpha snapped to 0 / +-1 whenever within 1e-7 of it
        for v in (sa, ca):
            r = np.round(v)
            v[np.abs(v - r) < 1e-7] = r[np.abs(v - r) < 1e-7]
    G = L[:, 20].astype(LD)
    aG = G if defect == "signed_G" else np.abs(G)
    th = L[:, 2].astype(LD)
    return dict(n=len(L), sa=sa, ca=ca, a=L[:, 1].astype(LD), st0=np.sin(th), ct0=np.cos(th), d=L[:, 3].astype(LD),
                pris=L[:, 4] != 0, off=L[:, 5].astype(LD), m=L[:, 6].astype(LD), r=L[:, 7:10].astype(LD),
                I=L[:, 10:19].reshape(-1, 3, 3).transpose(0, 2, 1).astype(LD),  # read column-major, as the kernels do
                jm=(G if defect == "jm_G" else G * G) * L[:, 19].astype(LD), b=G * G * L[:, 21].astype(LD),
                tcp=aG * L[:, 22].astype(LD), tcm=aG * L[:, 23].astype(LD))


def _abs_consts(K):
    return {k: (np.abs(v) if k not in ("n", "pris") else v) for k, v in K.items()}


def _cross(a, b, ab):
    if ab:
        return np.stack([a[1] * b[2] + a[2] * b[1], a[2] * b[0] + a[0] * b[2], a[0] * b[1] + a[1] * b[0]])
    return np.stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def _mv(R, v):  # R v, R (3, 3, N), v (3, N)
    return np.einsum("ijn,jn->in", R, v)


def _tmv(R, v):  # R^T v
    return np.einsum("jin,jn->in", R, v)


def _rot(st, ct, sa, ca, mdh, ab):
    z = np.zeros_like(st)
    s = 1 if ab else -1  # on absolute values every entry is a magnitude
    if mdh:  # Rx(alpha) Rz(theta)
        rows = [[ct, s * st, z], [ca * st, ca * ct, s * sa + z], [sa * st, sa * ct, ca + z]]
    else:  # Rz(theta) Rx(alpha)
        rows = [[ct, s * ca * st, sa * st], [st, ca * ct, s * sa * ct], [z, sa + z, ca + z]]
    return np.array(rows)


def _recursion(K, mdh, q, qd, qdd, grav, fext, ab=False, teps=None, defect=None):
    """tau (N, n) of one batch of rows; with ab=True the magnitude recursion (every input given as |.|), its sin / cos
    widened by teps (N, n) absolute."""
    N, n = q.shape
    z0 = np.zeros(N, LD)
    zero = np.zeros((3, N), LD)
    ez = lambda x: np.stack([z0, z0, x])  # noqa: E731  x along z
    g = np.asarray(grav, LD)[:, None] + zero
    w, wd, acc = zero, zero, zero
    Fm, Nm, Rs, ps_, sc = [], [], [], [], []
    for j in range(n):
        pris = bool(K["pris"][j])
        sa, ca = K["sa"][j], K["ca"][j]
        if pris:
            st, ct = K["st0"][j] + z0, K["ct0"][j] + z0
            dj = q[:, j] + K["off"][j]
        else:
            th = q[:, j] + K["off"][j]
            st, ct = (np.sin(th), np.cos(th)) if not ab else (np.abs(np.sin(th)), np.abs(np.cos(th)))
            dj = K["d"][j] + z0
        if ab and teps is not None:  # the specialised kernel snaps constant sin / cos within SNAP of 0 or +-1
            st, ct = (st + SNAP, ct + SNAP) if pris else (st + teps[:, j], ct + teps[:, j])
            sa, ca = sa + SNAP, ca + SNAP
        R = _rot(st, ct, sa, ca, mdh, ab)
        sgn = -1 if (mdh and defect != "mdh_ps_sign") else 1
        ps = np.stack([K["a"][j] + z0, (sgn if not ab else 1) * dj * sa, dj * ca])
        Rs.append(R); ps_.append(ps); sc.append((sa, ca))
        vq, vqq = ez(qd[:, j]), ez(qdd[:, j])
        if mdh:  # Craig: frame j-1 quantities carried across p*_j, then rotated into frame j
            if pris and j == 0:  # the compiled reference's prismatic first joint under modified DH
                wn, wdn, accn = vq, vqq, g
            else:
                lin = _cross(wd, ps, ab) + _cross(w, _cross(w, ps, ab), ab) + acc if j else g
                accn = _tmv(R, lin)
                wr, wdr = _tmv(R, w), _tmv(R, wd)
                if pris:
                    wn, wdn = wr, wdr
                    accn = accn + 2 * _cross(wn, vq, ab) + vqq
                else:
                    wn = wr + vq
                    wdn = wdr + _cross(wr, vq, ab) + vqq
        else:  # Luh-Walker-Paul in link frames
            base = g if j == 0 else acc
            if pris:
                wn, wdn = _tmv(R, w), _tmv(R, wd)
                accn = (_tmv(R, vqq + base) + _cross(wdn, ps, ab) + 2 * _cross(wn, _tmv(R, vq), ab)
                        + _cross(wn, _cross(wn, ps, ab), ab))
            else:
                wn = _tmv(R, w + vq)
                wdn = _tmv(R, wd + vqq + _cross(w, vq, ab))
                accn = _cross(wdn, ps, ab) + _cross(wn, _cross(wn, ps, ab), ab) + _tmv(R, base)
        w, wd, acc = wn, wdn, accn
        rc = K["r"][j][:, None] + zero
        ac = _cross(wd, rc, ab) + _cross(w, _cross(w, rc, ab), ab) + acc
        Fm.append(K["m"][j] * ac)
        Ic = K["I"][j]
        Nm.append(np.einsum("ij,jn->in", Ic, wd) + _cross(w, np.einsum("ij,jn->in", Ic, w), ab))
    ft = np.asarray(fext[:3], LD)[:, None] + zero
    nt = np.asarray(fext[3:], LD)[:, None] + zero
    f, nn = ft, nt
    tau = np.empty((N, n), LD)
    for j in range(n - 1, -1, -1):
        rc = K["r"][j][:, None] + zero
        Rn = Rs[j + 1] if j + 1 < n else None
        if mdh:
            if Rn is None:
                fj, nj = f + Fm[j], nn + _cross(rc, Fm[j], ab) + Nm[j]
            else:
                Rf = _mv(Rn, f)
                fj = Rf + Fm[j]
                nj = _mv(Rn, nn) + _cross(ps_[j + 1], Rf, ab) + _cross(rc, Fm[j], ab) + Nm[j]
            zax = np.stack([z0, z0, z0 + 1])
        else:
            ps = ps_[j]
            if Rn is None:
                fj = f + Fm[j]
                nj = nn + _cross(ps, f, ab) + _cross(ps + rc, Fm[j], ab) + Nm[j]
            else:
                fj = _mv(Rn, f) + Fm[j]
                nj = _mv(Rn, nn + _cross(_tmv(Rn, ps), f, ab)) + _cross(ps + rc, Fm[j], ab) + Nm[j]
            zax = np.stack([z0, z0 + sc[j][0], z0 + sc[j][1]])  # R_j^T z0
        f, nn = fj, nj
        t = ((fj if K["pris"][j] else nj) * zax).sum(0)
        v, a = qd[:, j], qdd[:, j]
        t = t + K["jm"][j] * a + K["b"][j] * v
        pos = v >= 0 if defect == "coulomb_at_zero" else v > 0
        t = t + np.where(pos, K["tcp"][j], 0) + np.where(v < 0, K["tcm"][j], 0)
        tau[:, j] = t
    return tau


def _ld(x):
    return np.atleast_2d(np.asarray(x)).astype(LD)


def rne3(L, mdh, grav, q, qd, qdd, fext=None, dtype=np.float64, defect=None):
    """(tau, bar) of rne over rows, tau in long double, bar the absolute error bar of a kernel of type dtype.  The
    inputs are taken as given: a caller comparing an fp32 kernel passes the fp32 arrays."""
    q, qd, qdd = _ld(q), _ld(qd), _ld(qdd)
    fext = np.zeros(6) if fext is None else np.asarray(fext, dtype=np.float64)
    K = _consts(L, defect)
    tau = _recursion(K, mdh, q, qd, qdd, grav, fext, defect=defect)
    Ka = _abs_consts(K)
    ga, fa = np.abs(np.asarray(grav, np.float64)), np.abs(fext)
    qa, qda, qdda = np.abs(q), np.abs(qd), np.abs(qdd)
    mag = _recursion(Ka, mdh, qa, qda, qdda, ga, fa, ab=True)
    u = float(np.finfo(dtype).eps) / 2
    th = (q + K["off"]).astype(dtype)  # the angles the kernels hand to sincos
    path, amax = fkj_ref.sincos_path(th, np.dtype(dtype), True)
    teps = (fkj_ref.trig_err(path, amax, dtype)[:, None] + 2 * u * (np.abs(q) + np.abs(K["off"])).astype(np.float64))
    mag_t = _recursion(Ka, mdh, qa, qda, qdda, ga, fa, ab=True, teps=teps.astype(LD))
    n = K["n"]
    bar = (4.0 * (2 * n + 2) + 2) * u * mag + (mag_t - mag) + _floor(n, dtype)
    return tau, bar.astype(np.float64)


def _floor(n, dtype):
    """Results in the subnormal range round absolutely: a few subnormals per step of the recursion."""
    return 8 * (2 * n + 2) * float(np.finfo(dtype).smallest_subnormal)


def _units(n, N, which):
    """Rows of unit (or pair) vectors for every row of a batch: (len(which) * N, n), call-major."""
    E = np.zeros((len(which), n), LD)
    for c, idx in enumerate(which):
        E[c, list(idx)] = 1
    return np.repeat(E, N, axis=0)


def op3(op, L, mdh, grav, q, qd=None, x=None, fext=None, dtype=np.float64, defect=None):
    """(value, bar) of one operation.  x: qdd for rne / itorque, the torque for accel."""
    q = _ld(q)
    N, n = q.shape
    zr = np.zeros_like(q)
    g0 = np.zeros(3)
    if op == "rne":
        return rne3(L, mdh, grav, q, qd, x, fext, dtype, defect)
    if op == "gravload":
        return rne3(L, mdh, grav, q, zr, zr, None, dtype, defect)
    if op == "itorque":
        return rne3(L, mdh, g0, q, zr, x, None, dtype, defect)
    qn = np.tile(q, (n, 1))
    if op == "inertia":
        t, b = rne3(L, mdh, g0, qn, np.zeros_like(qn), _units(n, N, [(i,) for i in range(n)]), None, dtype, defect)
        return t.reshape(n, N, n).transpose(1, 0, 2), b.reshape(n, N, n).transpose(1, 0, 2)  # M[row, i, k]
    if op == "coriolis":
        u = float(np.finfo(dtype).eps) / 2
        Lnf = L if defect == "coriolis_friction" else nofriction(L)
        qd = _ld(qd)
        t1, b1 = rne3(Lnf, mdh, g0, qn, _units(n, N, [(i,) for i in range(n)]), np.zeros_like(qn), None, dtype, defect)
        Csq, Esq = t1.reshape(n, N, n), b1.reshape(n, N, n)  # [i, row, k]
        pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
        C = np.zeros((N, n, n), LD)
        Cm = np.zeros((N, n, n))  # magnitude of the combination (its own rounding)
        E = np.zeros((N, n, n))
        if pairs:
            qp = np.tile(q, (len(pairs), 1))
            t2, b2 = rne3(Lnf, mdh, g0, qp, _units(n, N, pairs), np.zeros_like(qp), None, dtype, defect)
            t2, b2 = t2.reshape(len(pairs), N, n), b2.reshape(len(pairs), N, n)
            for p, (i, j) in enumerate(pairs):
                d = t2[p] - Csq[j] - Csq[i]
                dm = (np.abs(t2[p]) + np.abs(Csq[j]) + np.abs(Csq[i])).astype(np.float64)
                de = b2[p] + Esq[j] + Esq[i]
                for col, other in ((j, i), (i, j)):
                    w = qd[:, other][:, None] / 2
                    C[:, :, col] += d * w
                    aw = np.abs(w).astype(np.float64)
                    Cm[:, :, col] += dm * aw
                    E[:, :, col] += de * aw
        for i in range(n):
            C[:, :, i] += Csq[i] * qd[:, i][:, None]
            aw = np.abs(qd[:, i]).astype(np.float64)[:, None]
            Cm[:, :, i] += np.abs(Csq[i]).astype(np.float64) * aw
            E[:, :, i] += Esq[i] * aw
        return C, E + 2 * n * u * Cm + _floor(n, dtype)
    if op == "accel":
        u = float(np.finfo(dtype).eps) / 2
        M, EM = op3("inertia", L, mdh, grav, q, dtype=dtype, defect=defect)
        Lh = nofriction(L) if defect == "accel_nofriction" else L
        h, Eh = rne3(Lh, mdh, grav, q, qd, zr, None, dtype, defect)
        xq, LU, Minv = solve(M, _ld(x) - h)
        ax = np.abs(xq).astype(np.float64)
        dM = np.sqrt(np.abs(np.einsum("nii->ni", M)).astype(np.float64))
        S = np.maximum(LU, dM[:, :, None] * dM[:, None, :])  # |L||U|, or the Cholesky-type bound of a pivot-free LDL^T
        back = Eh + np.einsum("nij,nj->ni", EM + 3 * n * u * S, ax)
        return xq, np.einsum("nij,nj->ni", np.abs(Minv).astype(np.float64), back) + 2 * u * ax + _floor(n, dtype)
    raise ValueError(op)


def solve(M, b):
    """x = M^-1 b per row by Gaussian elimination with partial pivoting in long double; also |L||U| (float64) and
    M^-1 (long double)."""
    M = np.array(M, dtype=LD)
    N, n, _ = M.shape
    A = np.concatenate([M, b[:, :, None], np.broadcast_to(np.eye(n, dtype=LD), (N, n, n))], axis=2)
    Lf = np.zeros((N, n, n), LD)
    rows = np.arange(N)
    for c in range(n):
        p = c + np.argmax(np.abs(A[:, c:, c]), axis=1)
        A[rows, c], A[rows, p] = A[rows, p].copy(), A[rows, c].copy()
        Lf[rows, c], Lf[rows, p] = Lf[rows, p].copy(), Lf[rows, c].copy()
        f = A[:, c + 1:, c] / A[:, c, c][:, None]
        Lf[:, c + 1:, c] = f
        A[:, c + 1:] -= f[:, :, None] * A[:, c][:, None, :]
    Lf += np.eye(n, dtype=LD)
    U = A[:, :, :n]
    X = np.zeros((N, n, n + 1), LD)
    for r in range(n - 1, -1, -1):
        X[:, r] = (A[:, r, n:] - np.einsum("nk,nkc->nc", U[:, r, r + 1:], X[:, r + 1:])) / U[:, r, r][:, None]
    LU = np.einsum("nik,nkj->nij", np.abs(Lf), np.abs(U)).astype(np.float64)
    return X[:, :, 0], LU, X[:, :, 1:]


def cond(M):
    """Infinity-norm condition number of every M (N, n, n), in long double."""
    _, _, Minv = solve(M, np.zeros(M.shape[:2], LD))
    nrm = lambda A: np.abs(A).sum(2).max(1)  # noqa: E731
    return (nrm(np.asarray(M, LD)) * nrm(Minv)).astype(np.float64)


# ------------------------------------------------------------------ robots and inputs
PROFILES = ("struct", "near", "gen")  # alpha = k pi/2 exactly; within 1e-9 of it; anywhere


def robot(n, mdh, profile, prismatic, friction, seed):
    """A packed link table (24 n doubles).  prismatic: the first joint and about a third of the others translate.
    friction: nonzero Jm, B and asymmetric Tc on most links, G of both signs; else all four zero and G = 1."""
    rng = np.random.default_rng(seed)
    L = np.zeros((n, 24))
    for j in range(n):
        k = rng.integers(-1, 3)
        al = {"struct": k * np.pi / 2, "near": k * np.pi / 2 + rng.choice([-1e-9, 1e-9]),
              "gen": rng.uniform(-np.pi, np.pi)}[profile]
        sigma = 1.0 if prismatic and (j == 0 or rng.random() < 0.3) else 0.0
        L[j, :6] = al, rng.uniform(-0.5, 0.5), rng.uniform(-1, 1), rng.uniform(-0.5, 0.5), sigma, rng.uniform(-1, 1)
        L[j, 6] = rng.uniform(0.2, 5.0)
        L[j, 7:10] = rng.uniform(-0.3, 0.3, 3)
        A = rng.normal(size=(3, 3)) * 0.1
        L[j, 10:19] = (A @ A.T + 0.01 * np.eye(3)).ravel()
        if friction:
            L[j, 19:24] = (rng.choice([0.0, rng.uniform(1e-4, 3e-4)], p=[0.2, 0.8]), rng.choice([-1, 1]) * rng.uniform(20, 120),
                           rng.choice([0.0, rng.uniform(5e-4, 2e-3)], p=[0.2, 0.8]), rng.uniform(0.05, 0.5), -rng.uniform(0.05, 0.5))
        else:
            L[j, 20] = 1.0
    return L.ravel()


def inputs(L, N, dtype, seed):
    """q in [-pi, pi] with a few rows whose revolute angles reach 1e6 (the slow sincos path); qd with exact 0, -0.0 and subnormals of both
    signs; qdd; a torque.  Arrays of `dtype`."""
    rng = np.random.default_rng(seed)
    rev = np.asarray(L).reshape(-1, 24)[:, 4] == 0
    n = len(rev)
    q = rng.uniform(-np.pi, np.pi, (N, n))
    q[5::97] *= np.where(rev, rng.uniform(1, 1e6, q[5::97].shape), 1.0)
    qd = rng.normal(size=(N, n))
    tiny = 1e-310 if dtype == np.float64 else 1e-40
    pick = rng.integers(0, 8, (N, n))
    qd = np.where(pick == 0, 0.0, np.where(pick == 1, -0.0, np.where(pick == 2, tiny * rng.choice([-1, 1], (N, n)), qd)))
    qdd, tq = rng.normal(size=(N, n)), 10 * rng.normal(size=(N, n))
    return [np.ascontiguousarray(x, dtype=dtype) for x in (q, qd, qdd, tq)]
