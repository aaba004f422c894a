"""Long-double reference of the forward-kinematics / Jacobian entry points (b2k_fkj.cuh through b2k_api.cu):
b2k_fkine, b2k_jacob0, b2k_jacobe, b2k_fkine_jacob0 and b2k_fkine_jacobe.

The chain walk is restated batched in 80-bit extended precision from an ``ETS.describe()`` dictionary, evaluated on
exactly the numbers the kernel receives (an fp32 q is widened exactly; the fp64 constants of the description are
folded in long double).  Next to T, J0 and Je it returns, per row, what an error bar for that row needs: L, the sum of
the translation lengths the walk multiplies into (folded constants, base, tool, |prismatic q|), the sincos path the
kernel takes for the row, and the largest angle it feeds to sincos.

It also restates the host-side rules that pick a kernel: ``b2k_classify34``, the ``dh_like`` and ``dense_jindex``
flags of ``b2k_chain_create``, and the lean-kernel condition of ``fkj_launch_n``, plus chain families that reach each
kernel shape (tests/test_fkj_ref_cpu.py pins both against the compiled oracle and against themselves).
"""
import math

import numpy as np

from oracle import chains as ch

LD = np.longdouble
assert np.finfo(LD).eps < 1e-18, "tests/fkj_ref.py needs 80-bit x86 extended precision for np.longdouble"

RX, RY, RZ, TX, TY, TZ = range(6)
AK_IDENT, AK_RX, AK_RY, AK_RZ, AK_GEN, AK_ROTMASK, AK_TX, AK_TY, AK_TZ = 0, 1, 2, 3, 4, 7, 8, 16, 32
MUFU_LIMIT = 8.0  # B2K_MUFU_LIMIT (b2k_trig.cuh)
FAST_LIMIT = 105615.0  # TrigC::fast_limit
PATH_MUFU, PATH_POLY, PATH_SLOW = 0, 1, 2  # special-function unit, Cody-Waite + polynomial, CUDA's sincos


# ------------------------------------------------------------------ host rules of b2k_chain.cu / b2k_common.cuh
def mul34(A, B):
    """b2k_mul34 in fp64, the same left-to-right sums (3x4 row-major affine)."""
    C = np.empty((3, 4))
    for i in range(3):
        for j in range(3):
            C[i, j] = A[i, 0] * B[0, j] + A[i, 1] * B[1, j] + A[i, 2] * B[2, j]
        C[i, 3] = A[i, 0] * B[0, 3] + A[i, 1] * B[1, 3] + A[i, 2] * B[2, 3] + A[i, 3]
    return C


def classify34(A):
    """b2k_classify34: structure class of a 3x4 constant (exact 0 / 1 tests)."""
    A = np.asarray(A, dtype=np.float64).reshape(3, 4)
    row0 = A[0, 0] == 1 and A[0, 1] == 0 and A[0, 2] == 0 and A[1, 0] == 0 and A[2, 0] == 0
    row1 = A[1, 1] == 1 and A[1, 0] == 0 and A[1, 2] == 0 and A[0, 1] == 0 and A[2, 1] == 0
    row2 = A[2, 2] == 1 and A[2, 0] == 0 and A[2, 1] == 0 and A[0, 2] == 0 and A[1, 2] == 0
    k = AK_IDENT if (row0 and row1 and row2) else AK_RX if row0 else AK_RY if row1 else AK_RZ if row2 else AK_GEN
    return k | (AK_TX if A[0, 3] != 0 else 0) | (AK_TY if A[1, 3] != 0 else 0) | (AK_TZ if A[2, 3] != 0 else 0)


def compile_chain(desc):
    """b2k_chain_create's fold in fp64: the n + 1 constants, joint axes / flips / jindex, and its flags."""
    acc = np.eye(4)[:3].copy()
    A, axis, flip, jidx = [], [], [], []
    for i in range(len(desc["isjoint"])):
        if desc["isjoint"][i]:
            A.append(acc)
            acc = np.eye(4)[:3].copy()
            axis.append(int(desc["axis"][i]))
            flip.append(int(desc["flip"][i]))
            jidx.append(int(desc["jindex"][i]))
        else:
            acc = mul34(acc, np.asarray(desc["T"][i], dtype=np.float64)[:3])
    A.append(acc)
    n = len(axis)
    all_rz = all(a == RZ and not f for a, f in zip(axis, flip))
    dh_like = all_rz and all((classify34(A[k]) & AK_ROTMASK) in (AK_IDENT, AK_RX) for k in range(1, n))
    dense = all(j == k for k, j in enumerate(jidx))
    return dict(n=n, A=A, axis=axis, flip=flip, jidx=jidx, dh_like=dh_like, dense_jindex=dense,
                q_width=max(jidx) + 1)


def lean_eligible(c, ldq, q_ptr, nrows, variant=0):
    """fkj_launch_n's condition for the lean kernels (k_fkj_fast / k_fkj_back_fast) on the full tiles of a call."""
    return bool(c["dh_like"] and c["dense_jindex"] and ldq == c["n"] and variant == 0 and q_ptr % 16 == 0
                and nrows >= 32)


def expected_launches(c, ldq, q_ptr, nrows, variant=0):
    """Kernel launches of one fkj call: the lean kernel plus the general kernel on a ragged tail, or one kernel."""
    if nrows == 0:
        return 0
    if lean_eligible(c, ldq, q_ptr, nrows, variant):
        return 1 + (nrows % 32 != 0)
    return 1


# ------------------------------------------------------------------ the long-double walk
def _ld44(M):
    M = np.asarray(M, dtype=np.float64)
    out = np.zeros((4, 4), dtype=LD)
    out[:3] = M[:3].astype(LD)
    out[3, 3] = 1
    return out


def _joint(axis, eta):
    """(N, 4, 4) long-double elementary transform of each row's joint value eta (already sign-flipped)."""
    N = eta.shape[0]
    T = np.zeros((N, 4, 4), dtype=LD)
    T[:, 0, 0] = T[:, 1, 1] = T[:, 2, 2] = T[:, 3, 3] = 1
    if axis < 3:
        with np.errstate(invalid="ignore"):  # +-inf rows: NaN, as on the device
            s, c = np.sin(eta), np.cos(eta)
        a, b = [(1, 2), (2, 0), (0, 1)][axis]
        T[:, a, a] = c
        T[:, b, b] = c
        T[:, a, b] = -s
        T[:, b, a] = s
    else:
        T[:, axis - 3, 3] = eta
    return T


def evaluate(desc, q, base=None, tool=None, batch_trig=None):
    """The five entry points' results on q (N, ldq), fp32 or fp64, exactly as the kernel reads it.

    Returns a dict of long-double arrays T (base @ pose @ tool), Tnb (without base), J0 (base-frame Jacobian, tool
    included, base not: RobotKinematics.py:158), Je (end-effector frame), and per row: L, angle (largest |sincos
    argument|) and path (PATH_*: the sincos branch the kernel takes for the row).  batch_trig: the chain walk evaluates
    its n sincos as one batch (b2k_sincos_batch: the DH-like profile of the FK kernels), default from the chain's
    classification; False for kernels that call the scalar b2k_sincos per joint."""
    c = compile_chain(desc)
    n = c["n"]
    q = np.asarray(q)
    assert q.ndim == 2 and q.dtype in (np.float32, np.float64)
    N = q.shape[0]
    ql = q.astype(LD)
    if batch_trig is None:
        batch_trig = c["dh_like"]
    # constants folded in long double from the description's fp64 matrices
    consts, acc = [], np.eye(4, dtype=LD)
    for i in range(len(desc["isjoint"])):
        if desc["isjoint"][i]:
            consts.append(acc)
            acc = np.eye(4, dtype=LD)
        else:
            acc = acc @ _ld44(desc["T"][i])
    consts.append(acc)
    B = _ld44(base) if base is not None else np.eye(4, dtype=LD)
    Tl = _ld44(tool) if tool is not None else np.eye(4, dtype=LD)
    T = np.broadcast_to(consts[0], (N, 4, 4)).copy()
    z = np.zeros((N, 3, n), dtype=LD)
    p = np.zeros((N, 3, n), dtype=LD)
    L = np.full(N, sum(np.sqrt(np.sum(A[:3, 3] ** 2)) for A in consts) + np.sqrt(np.sum(B[:3, 3] ** 2))
                + np.sqrt(np.sum(Tl[:3, 3] ** 2)), dtype=LD)
    angles = []
    for j in range(n):
        if j > 0:
            T = T @ consts[j]
        ax, sg = c["axis"][j], (-1 if c["flip"][j] else 1)
        eta = sg * ql[:, c["jidx"][j]]
        z[:, :, j] = sg * T[:, :3, ax if ax < 3 else ax - 3]
        p[:, :, j] = T[:, :3, 3]
        if ax < 3:
            angles.append(eta)
        else:
            L = L + np.abs(eta)
        T = T @ _joint(ax, eta)
    T = T @ (consts[n] @ Tl)
    J0 = np.zeros((N, 6, n), dtype=LD)
    for j in range(n):
        if c["axis"][j] < 3:
            J0[:, :3, j] = np.cross(z[:, :, j], T[:, :3, 3] - p[:, :, j])
            J0[:, 3:, j] = z[:, :, j]
        else:
            J0[:, :3, j] = z[:, :, j]
    Rt = np.swapaxes(T[:, :3, :3], 1, 2)
    Je = np.concatenate([Rt @ J0[:, :3], Rt @ J0[:, 3:]], axis=1)
    path, angle = sincos_path(np.stack(angles, 1) if angles else np.zeros((N, 0), LD), q.dtype, batch_trig)
    return dict(T=B @ T, Tnb=T, J0=J0, Je=Je, L=L, path=path, angle=angle, chain=c)


def sincos_path(x, dtype, batch):
    """Per row: the sincos branch the kernel takes for the row's angles x (N, k), and max |x| (inf for non-finite).

    b2k_sincos_batch (batch=True): fp32 rows whose every |angle| < B2K_MUFU_LIMIT go to the special-function unit;
    rows whose every |angle| < fast_limit to the Cody-Waite polynomial; any other row calls the scalar b2k_sincos per
    angle, which takes the polynomial below fast_limit and CUDA's sincos beyond (reported as PATH_SLOW).  The scalar
    b2k_sincos (batch=False) never uses the special-function unit."""
    ax = np.abs(x.astype(np.float64))
    amax = np.where(np.isfinite(ax).all(1), ax.max(1, initial=0.0), np.inf)
    fast = (ax < FAST_LIMIT).all(1)  # NaN compares false: not fast
    path = np.where(fast, PATH_POLY, PATH_SLOW)
    if batch and dtype == np.float32:
        path = np.where((ax < MUFU_LIMIT).all(1), PATH_MUFU, path)
    return path, amax


# ------------------------------------------------------------------ error model
MUFU_ERR = 2.0 ** -21.4  # MUFU.SIN / MUFU.COS on the argument they are given (b2k_trig.cuh)
INV_2PI_F32 = float(np.float32(1 / (2 * math.pi)))


def mufu_arg_error(x):
    """|2 pi t - x| for t = x * fl32(1/(2 pi)) rounded toward zero to fp32: the angle __sinf / __cosf actually take
    (the SASS is FMUL.RZ by 0.15915494 ahead of MUFU.SIN / MUFU.COS).  At most |x| (2^-24.56 + 2^-23) < |x| 2^-22.6."""
    x = np.asarray(x, dtype=np.float32)
    p = x.astype(np.float64) * INV_2PI_F32  # exact: a product of two fp32 fits in fp64
    t = p.astype(np.float32)
    over = np.abs(t.astype(np.float64)) > np.abs(p)
    t[over] = np.nextafter(t[over], np.float32(0))
    return np.abs(2 * np.pi * t.astype(LD) - x.astype(LD)).astype(np.float64)


def trig_err(path, angle, dtype):
    """Absolute error of one sin or cos on the row's path: on the special-function unit the unit's own error plus the
    rounding of its argument (mufu_arg_error), 2 ulp of 1 on the polynomial and on CUDA's sincos."""
    eps = float(np.finfo(dtype).eps)
    mufu = MUFU_ERR + np.where(np.isfinite(angle), angle, 0.0) * 2.0 ** -22.6
    return np.where(path == PATH_MUFU, mufu, 2 * eps)


def bars(ref, dtype, K=4.0):
    """Per-row (rotation / angular, position / linear) absolute error bars: K (n+1) u (+ n trig) for unit-size
    entries, times (1 + L) for lengths, plus the rounding of the constants to the kernel's type (u L)."""
    n = ref["chain"]["n"]
    u = float(np.finfo(dtype).eps) / 2
    L = ref["L"].astype(np.float64)
    rot = K * (n + 1) * u + n * trig_err(ref["path"], ref["angle"], dtype)
    pos = rot * (1 + L) + u * L
    return rot, pos


def pose_bar(ref, dtype, K=4.0):
    rot, pos = bars(ref, dtype, K)
    b = np.zeros((len(rot), 4, 4))
    b[:, :3, :3] = rot[:, None, None]
    b[:, :3, 3] = pos[:, None]
    return b  # the bottom row is exact


def jac_bar(ref, dtype, K=4.0):
    rot, pos = bars(ref, dtype, K)
    n = ref["chain"]["n"]
    b = np.empty((len(rot), 6, n))
    b[:, :3] = pos[:, None, None]
    b[:, 3:] = rot[:, None, None]
    return b


# ------------------------------------------------------------------ chain families
def _rot(kind, rng):
    a = float(rng.uniform(-3, 3))
    if kind == AK_IDENT:
        return np.eye(4)
    if kind == AK_RX:
        return ch.trotx(a)
    if kind == AK_RY:
        return ch.troty(a)
    if kind == AK_RZ:
        return ch.trotz(a)
    return ch.trotx(a) @ ch.troty(float(rng.uniform(0.3, 1.2))) @ ch.trotz(float(rng.uniform(-3, 3)))


def _const(kind, rng):
    """A 4x4 constant of the given AK_* class, translation bits included."""
    M = _rot(kind & AK_ROTMASK, rng)
    for bit, r in ((AK_TX, 0), (AK_TY, 1), (AK_TZ, 2)):
        if kind & bit:
            M[r, 3] = float(rng.choice([-1, 1]) * rng.uniform(0.05, 0.6))
    return M


def dh_family(n, rng, tail="gen", alphas=None):
    """DH-like: unflipped Rz joints, a general first constant, Rx-form constants between joints (random a, d and
    alpha from {0, +-pi/2, pi, random}), and a tail that is absent ("ident"), a pure translation ("trans") or
    general ("gen")."""
    b = ch.Builder()
    b.se3(_const(AK_GEN | AK_TX | AK_TY | AK_TZ, rng))
    choices = [0.0, math.pi / 2, -math.pi / 2, math.pi, None]
    for j in range(n):
        if j > 0:
            al = alphas[j] if alphas is not None else choices[int(rng.integers(0, len(choices)))]
            al = float(rng.uniform(-3, 3)) if al is None else al
            b.se3(ch.transl(float(rng.uniform(-0.5, 0.5)), 0.0, float(rng.uniform(-0.5, 0.5))) @ ch.trotx(al))
        b.joint(RZ)
    if tail == "trans":
        b.se3(ch.transl(*rng.uniform(-0.3, 0.3, 3)))
    elif tail == "gen":
        b.se3(_const(AK_GEN | AK_TX | AK_TY | AK_TZ, rng))
    return b.desc()


def near_dh_family(n, k, breaker, rng):
    """A DH-like chain with one breaker at position k, which must send it to the generic profile:
    "flip" (joint k a flipped Rz, 0 <= k < n), "ry" / "rz" / "gen" (the constant ahead of joint k, 1 <= k < n, of
    that class), or "offset" (standard DH links with a joint offset on link k, 1 <= k < n)."""
    if breaker == "offset":
        links = [dict(d=float(rng.uniform(0, 0.4)), a=float(rng.uniform(-0.5, 0.5)),
                      alpha=float(rng.choice([0, math.pi / 2, -math.pi / 2])), offset=(0.3 if j == k else 0.0))
                 for j in range(n)]
        return ch.dh_to_ets(links)
    b = ch.Builder()
    b.se3(_const(AK_GEN | AK_TZ, rng))
    for j in range(n):
        if j > 0:
            if j == k and breaker in ("ry", "rz", "gen"):
                kind = {"ry": AK_RY, "rz": AK_RZ, "gen": AK_GEN}[breaker]
                b.se3(_const(kind | AK_TX | AK_TZ, rng))
            else:
                b.se3(ch.transl(float(rng.uniform(-0.5, 0.5)), 0.0, 0.2) @ ch.trotx(float(rng.uniform(-3, 3))))
        b.joint(RZ, flip=(breaker == "flip" and j == k))
    b.se3(ch.transl(0.0, 0.0, 0.1))
    return b.desc()


ALL_KINDS = [r | t for r in (AK_IDENT, AK_RX, AK_RY, AK_RZ, AK_GEN) for t in range(0, 64, 8)]


def generic_family(n, rng, kinds):
    """Generic: joints cycle through all six axes with flips; the constants ahead of joints 1..n-1 take the AK_*
    classes of `kinds` in turn (the caller spreads ALL_KINDS over a sweep), first and tail constants are general."""
    b = ch.Builder()
    b.se3(_const(AK_GEN | AK_TX | AK_TY | AK_TZ, rng))
    for j in range(n):
        if j > 0:
            kind = kinds.pop(0) if kinds else int(rng.choice(ALL_KINDS))
            if kind != AK_IDENT:  # an identity constant is no ET at all
                b.se3(_const(kind, rng))
        b.joint(int(rng.integers(0, 6)) if j >= 6 else (j + n) % 6, flip=bool((j + n) % 3 == 0))
    b.se3(_const(AK_GEN | AK_TY, rng))
    return b.desc()


def with_jindex(desc, jidx):
    """The same chain reading joint j from column jidx[j] of q."""
    d = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in desc.items()}
    d["jindex"][np.flatnonzero(d["isjoint"])] = np.asarray(jidx, dtype=np.int32)
    return d
