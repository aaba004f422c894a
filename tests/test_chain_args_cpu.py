"""The argument checks of the C ABI entry points that walk a chain -- b2k_fkine, b2k_fkine_frames, b2k_jacob0,
b2k_jacobe, b2k_fkine_jacob0, b2k_fkine_jacobe, b2k_fkine_planar, b2k_gravjac, b2k_pay, b2k_paycap and the host front
ends b2k_fkine_host and b2k_fkine_jacob0_host -- and of b2k_pay_jacobian and b2k_friction (no GPU needed):

* every rejection names the entry point and the argument;
* the checks run in one order: the chain (handle, dtype, N, q, ldq, q alignment), then the entry point's own scalars
  and host tables, then its device arrays in argument order (NULL, then alignment);
* N = 0 is accepted with NULL arrays;
* no call below launches a kernel: each one returns before its first CUDA call.
"""
import numpy as np
import pytest

import b2kin as rtb

F32, F64 = 0, 1
BUF = np.zeros(1 << 12)
P = (BUF.ctypes.data + 255) & ~255  # 256-byte aligned: stands in for device arrays, never dereferenced
EYE3, EYE4 = np.eye(3), np.eye(4)
BAD4 = np.eye(4); BAD4[3, 0] = 1.0  # noqa: E702
BAD3 = np.eye(3); BAD3[2, 0] = 1.0  # noqa: E702
PANDA = rtb.models.Panda().ets()  # n = 7, q_width 7; kept alive: the table passes its chain handle
PLANAR = rtb.models.ETS.Planar2().ets()  # n = 2
MASS = np.ones((7, 4))
GRAV = np.array([0.0, 0.0, -9.81])
TAUR = np.ones((7, 2))
PARAMS = np.zeros((7, 4))
AFTER = np.array([-1, 0, 3], np.int32)
SLOT = np.array([0, 1, 2], np.int32)
TAILS = np.tile(np.eye(4), (3, 1, 1))

CHAIN = [("c", PANDA._chain), ("dt", F64), ("q", P), ("N", 4), ("ldq", 7)]
FK = [("base", EYE4), ("tool", EYE4)]
# each entry point's arguments in order, with a default that passes every check
SPECS = {
    "b2k_fkine": CHAIN + FK + [("T", P), ("stream", None)],
    "b2k_fkine_frames": CHAIN + [("base", EYE4), ("nframes", 3), ("after", AFTER), ("slot", SLOT), ("tails", TAILS),
                                 ("out", P), ("nslots", 3), ("stream", None)],
    "b2k_jacob0": CHAIN + [("tool", EYE4), ("J", P), ("stream", None)],
    "b2k_jacobe": CHAIN + [("tool", EYE4), ("J", P), ("stream", None)],
    "b2k_fkine_jacob0": CHAIN + FK + [("T", P), ("J", P), ("stream", None)],
    "b2k_fkine_jacobe": CHAIN + FK + [("T", P), ("J", P), ("stream", None)],
    "b2k_fkine_planar": [("c", PLANAR._chain), ("dt", F64), ("q", P), ("N", 4), ("ldq", 2), ("base", EYE3),
                         ("tool", EYE3), ("frame", 0), ("T", P), ("J", P), ("stream", None)],
    "b2k_gravjac": CHAIN + [("mass", MASS), ("grav", GRAV), ("taug", P), ("J0", P), ("stream", None)],
    "b2k_pay": CHAIN + [("W", P), ("w_stride", 6), ("frame", 0), ("tau", P), ("stream", None)],
    "b2k_paycap": CHAIN + [("mass", MASS), ("grav", GRAV), ("w", P), ("w_stride", 6), ("frame", 0), ("tauR", TAUR),
                           ("wmax", P), ("joint", P), ("stream", None)],
    "b2k_fkine_host": CHAIN + FK + [("T", P), ("device", 0)],
    "b2k_fkine_jacob0_host": CHAIN + FK + [("T", P), ("J", P), ("device", 0)],
    "b2k_pay_jacobian": [("dt", F64), ("n", 7), ("J", P), ("W", P), ("w_stride", 6), ("N", 4), ("tau", P), ("stream", None)],
    "b2k_friction": [("dt", F64), ("n", 7), ("params", PARAMS), ("qd", P), ("N", 4), ("tau", P), ("stream", None)],
}
WALKERS = [k for k in SPECS if k not in ("b2k_pay_jacobian", "b2k_friction")]
ON_DEVICE = [k for k in WALKERS if not k.endswith("_host")]
# the device arrays of each entry point, in argument order
ARRAYS = {k: [a for a, d in SPECS[k] if d is P and a != "q"] for k in SPECS}


def _call(name, **over):
    lib = rtb._lib.lib()
    args = []
    for a, d in SPECS[name]:
        v = over.get(a, d)
        if isinstance(v, np.ndarray):
            v = v.ctypes.data_as(rtb._lib.ip if v.dtype == np.int32 else rtb._lib.dp)
        args.append(v)
    n0 = lib.b2k_launch_count()
    rc = getattr(lib, name)(*args)
    assert lib.b2k_launch_count() == n0, name
    return rc, lib.b2k_last_error().decode()


def _nan(a, idx):
    a = a.copy()
    a[idx] = np.nan
    return a


def _tails(k):
    t = TAILS.copy()
    t[k, 3, 0] = 1.0
    return t


CASES = []  # (entry point, argument overrides, what the message says after "<entry point>: "; None: accepted)
for name in WALKERS:
    CASES += [
        (name, dict(c=None), "chain handle is NULL"),
        (name, dict(dt=2), "dtype must be B2K_F32 or B2K_F64"),
        (name, dict(N=-1), "N = -1 is negative"),
        (name, dict(q=None), "q is NULL"),
        (name, dict(ldq=17), "q row width 17 outside"),
        (name, dict(ldq=1), "q row width 1 outside"),
        (name, dict(dt=2, N=-1), "dtype"),
        (name, dict(N=-1, q=None), "N = -1"),
        (name, dict(q=None, ldq=1), "q is NULL"),
    ]
    if name != "b2k_fkine_planar":  # which takes T or J, not neither
        CASES.append((name, dict(N=0, q=None, **{a: None for a in ARRAYS[name]}), None))
for name in ON_DEVICE:
    first = ARRAYS[name][0]
    CASES += [
        (name, dict(q=P + 4), "q must be 8-byte aligned"),
        (name, dict(dt=F32, q=P + 2), "q must be 4-byte aligned"),
        (name, dict(ldq=1, q=P + 4), "q row width"),
        (name, dict(q=P + 4, **{first: None}), "q must be 8-byte aligned"),
        (name, {first: P + 2, "N": 0}, f"{first} must be"),  # alignment is checked at N = 0 too
    ]
for name in ("b2k_fkine", "b2k_jacob0", "b2k_jacobe", "b2k_fkine_jacob0", "b2k_fkine_jacobe"):
    CASES += [
        (name, dict(tool=BAD4), "tool is not an SE(3)/affine matrix"),
        (name, dict(q=P + 4, tool=BAD4), "q must be"),
        (name, dict(tool=BAD4, **{ARRAYS[name][0]: None}), "tool is not"),
    ]
    if "T" in ARRAYS[name]:
        CASES += [
            (name, dict(base=BAD4), "base is not an SE(3)/affine matrix"),
            (name, dict(base=BAD4, tool=BAD4), "base is not"),
            (name, dict(T=None), "T is NULL"),
            (name, dict(T=P + 16), "T must be 32-byte aligned"),
            (name, dict(dt=F32, T=P + 16), "T must be 32-byte aligned"),
        ]
    if "J" in ARRAYS[name]:
        CASES += [
            (name, dict(J=None), "J is NULL"),
            (name, dict(J=P + 8), "J must be 16-byte aligned"),
            (name, dict(dt=F32, J=P + 4), "J must be 8-byte aligned"),  # 6 * 7 fp32 rows: 8-byte pieces
        ]
    if ARRAYS[name] == ["T", "J"]:
        CASES += [(name, dict(T=P + 16, J=None), "T must be"), (name, dict(T=None, J=P + 8), "T is NULL")]
CASES += [
    ("b2k_fkine_planar", dict(frame=2), "frame must be 0 (jacob0) or 1 (jacobe), got 2"),
    ("b2k_fkine_planar", dict(T=None, J=None), "T and J are both NULL"),
    ("b2k_fkine_planar", dict(base=BAD3), "base is not an SE(2) matrix"),
    ("b2k_fkine_planar", dict(tool=np.array([[1, 0.5, 0], [0, 1, 0], [0, 0, 1.0]])), "tool has an in-plane part"),
    ("b2k_fkine_planar", dict(c=PANDA._chain, ldq=7), "the chain is not planar"),
    ("b2k_fkine_planar", dict(T=P + 4), "T must be 8-byte aligned"),  # rows of 9 fp64
    ("b2k_fkine_planar", dict(dt=F32, T=P + 2), "T must be 4-byte aligned"),  # rows of 9 fp32
    ("b2k_fkine_planar", dict(J=P + 8), "J must be 16-byte aligned"),  # rows of 3 * 2 fp64
    ("b2k_fkine_planar", dict(dt=F32, J=P + 4), "J must be 8-byte aligned"),  # rows of 3 * 2 fp32
    ("b2k_fkine_planar", dict(c=PANDA._chain, ldq=2), "q row width 2 outside [7, 16]"),
    ("b2k_fkine_planar", dict(frame=2, T=None, J=None), "frame"),
    ("b2k_fkine_planar", dict(T=None, J=None, base=BAD3), "T and J are both NULL"),
    ("b2k_fkine_planar", dict(base=BAD3, T=P + 4), "base is not"),
    ("b2k_fkine_planar", dict(T=P + 4, J=P + 8), "T must be"),
    ("b2k_fkine_planar", dict(N=0, q=None, T=None), None),
    ("b2k_fkine_frames", dict(base=BAD4), "base is not an SE(3)/affine matrix"),
    ("b2k_fkine_frames", dict(nframes=0), "bad frame table"),
    ("b2k_fkine_frames", dict(after=None), "bad frame table"),
    ("b2k_fkine_frames", dict(nslots=0), "bad frame table"),
    ("b2k_fkine_frames", dict(after=np.array([-1, 3, 2], np.int32)), "after[2] = 2: must be ascending"),
    ("b2k_fkine_frames", dict(after=np.array([-1, 0, 7], np.int32)), "after[2] = 7"),
    ("b2k_fkine_frames", dict(slot=np.array([0, 1, 3], np.int32)), "slot[2] = 3 outside [0, 3)"),
    ("b2k_fkine_frames", dict(tails=_tails(1)), "tail 1 is not an SE(3)/affine matrix"),
    ("b2k_fkine_frames", dict(out=None), "out is NULL"),
    ("b2k_fkine_frames", dict(out=P + 8), "out must be 32-byte aligned"),
    ("b2k_fkine_frames", dict(base=BAD4, nframes=0), "base is not"),
    ("b2k_fkine_frames", dict(nframes=0, out=None), "bad frame table"),
    ("b2k_fkine_frames", dict(tails=_tails(2), out=P + 8), "tail 2"),
    ("b2k_fkine_frames", dict(N=0, base=BAD4, q=None, out=None), "base is not"),
    ("b2k_gravjac", dict(mass=None), "mass table is NULL"),
    ("b2k_gravjac", dict(grav=None), "grav is NULL"),
    ("b2k_gravjac", dict(mass=_nan(MASS, (2, 1))), "mass table entry (2, 1) is not finite"),
    ("b2k_gravjac", dict(taug=None), "taug is NULL"),
    ("b2k_gravjac", dict(taug=P + 4), "taug must be 8-byte aligned"),
    ("b2k_gravjac", dict(J0=None), "J0 is NULL"),
    ("b2k_gravjac", dict(dt=F32, J0=P + 2), "J0 must be 4-byte aligned"),
    ("b2k_gravjac", dict(mass=None, taug=None), "mass table"),
    ("b2k_gravjac", dict(taug=P + 4, J0=None), "taug must be"),
    ("b2k_pay", dict(w_stride=3), "w_stride must be 0 (one wrench) or 6 (one per row)"),
    ("b2k_pay", dict(frame=2), "frame must be 0 (world) or 1 (end effector)"),
    ("b2k_pay", dict(W=None), "W is NULL"),
    ("b2k_pay", dict(dt=F32, W=P + 2), "W must be 4-byte aligned"),
    ("b2k_pay", dict(tau=None), "tau is NULL"),
    ("b2k_pay", dict(tau=P + 4), "tau must be 8-byte aligned"),
    ("b2k_pay", dict(w_stride=3, W=None), "w_stride"),
    ("b2k_pay", dict(frame=2, W=None), "frame"),
    ("b2k_pay", dict(W=P + 4, tau=None), "W must be"),
    ("b2k_pay", dict(N=0, w_stride=0, q=None, W=None, tau=None), None),
    ("b2k_paycap", dict(mass=None), "mass table is NULL"),
    ("b2k_paycap", dict(grav=None), "grav is NULL"),
    ("b2k_paycap", dict(w_stride=1), "w_stride must be"),
    ("b2k_paycap", dict(frame=-1), "frame must be"),
    ("b2k_paycap", dict(tauR=None), "tauR is NULL"),
    ("b2k_paycap", dict(w=None), "w is NULL"),
    ("b2k_paycap", dict(w=P + 4), "w must be 8-byte aligned"),
    ("b2k_paycap", dict(wmax=None), "wmax is NULL"),
    ("b2k_paycap", dict(dt=F32, wmax=P + 2), "wmax must be 4-byte aligned"),
    ("b2k_paycap", dict(joint=None), "joint is NULL"),
    ("b2k_paycap", dict(joint=P + 2), "joint must be 4-byte aligned"),
    ("b2k_paycap", dict(mass=None, w_stride=1), "mass table"),
    ("b2k_paycap", dict(w_stride=1, frame=2), "w_stride"),
    ("b2k_paycap", dict(frame=2, tauR=None), "frame"),
    ("b2k_paycap", dict(tauR=None, w=None), "tauR"),
    ("b2k_paycap", dict(wmax=P + 4, joint=None), "wmax must be"),
    ("b2k_fkine_host", dict(T=None), "T is NULL"),
    ("b2k_fkine_jacob0_host", dict(T=None), "T is NULL"),
    ("b2k_fkine_jacob0_host", dict(J=None), "J is NULL"),
    ("b2k_fkine_jacob0_host", dict(T=None, J=None), "T is NULL"),
    ("b2k_fkine_host", dict(N=0, base=BAD4, tool=BAD4), None),  # the device calls check base and tool per chunk
    ("b2k_fkine_jacob0_host", dict(N=0, base=BAD4, tool=BAD4), None),
    ("b2k_pay_jacobian", dict(dt=2), "dtype must be B2K_F32 or B2K_F64"),
    ("b2k_pay_jacobian", dict(n=0), "n = 0 outside [1, 10]"),
    ("b2k_pay_jacobian", dict(n=11), "n = 11 outside [1, 10]"),
    ("b2k_pay_jacobian", dict(N=-1), "N is negative"),
    ("b2k_pay_jacobian", dict(w_stride=3), "w_stride must be"),
    ("b2k_pay_jacobian", dict(J=None), "J is NULL"),
    ("b2k_pay_jacobian", dict(J=P + 4), "J must be 8-byte aligned"),
    ("b2k_pay_jacobian", dict(W=None), "W is NULL"),
    ("b2k_pay_jacobian", dict(dt=F32, W=P + 2), "W must be 4-byte aligned"),
    ("b2k_pay_jacobian", dict(tau=None), "tau is NULL"),
    ("b2k_pay_jacobian", dict(tau=P + 4), "tau must be 8-byte aligned"),
    ("b2k_pay_jacobian", dict(N=0, J=None, W=None, tau=None), None),
    ("b2k_friction", dict(dt=2), "dtype must be"),
    ("b2k_friction", dict(n=0), "n = 0 outside [1, 10]"),
    ("b2k_friction", dict(params=None), "params is NULL"),
    ("b2k_friction", dict(params=_nan(PARAMS, (1, 1))), "params[5] is not finite"),
    ("b2k_friction", dict(N=-1), "N is negative"),
    ("b2k_friction", dict(qd=None), "qd is NULL"),
    ("b2k_friction", dict(qd=P + 1), "qd must be 8-byte aligned"),
    ("b2k_friction", dict(dt=F32, qd=P + 2), "qd must be 4-byte aligned"),
    ("b2k_friction", dict(tau=None), "tau is NULL"),
    ("b2k_friction", dict(tau=P + 4), "tau must be 8-byte aligned"),
    ("b2k_friction", dict(qd=P + 1, tau=None), "qd must be"),
    ("b2k_friction", dict(N=0, qd=None, tau=None), None),
]


def _id(case):
    def show(v):
        if v is None:
            return "NULL"
        if isinstance(v, np.ndarray):
            return "table"
        if v is PANDA._chain:
            return "panda"
        return f"P+{v - P}" if v >= P else str(v)
    name, over, _ = case
    return "-".join([name[4:]] + [f"{k}={show(v)}" for k, v in over.items()])


@pytest.mark.parametrize("name, over, msg", CASES, ids=[_id(c) for c in CASES])
def test_entry_point_checks(name, over, msg):
    rc, err = _call(name, **over)
    if msg is None:
        assert rc == 0, err
    else:
        assert rc == -1 and err.startswith(f"{name}: ") and msg in err, err

